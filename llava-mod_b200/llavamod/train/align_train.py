"""Mimic-distillation entry point (reference: llavamod/train/align_train.py:20-636; launched by
shells/train/qwen/dense2sparse_distillation.sh:48 with the deepspeed CLI -- here: one process per GPU, torchrun-style env).

    torchrun --nproc-per-node 8 -m llavamod.train.align_train <the reference shell's flags>

Kept: the four argument dataclasses, class dispatch by substring of the model path, ``policy_model_type == 'sparse'`` forcing
MoE, ``moe_finetune`` picking the FineTune class, construction order (build -> initialize_moe_modules ->
initialize_vision_modules), auto-resume from ``output_dir/checkpoint-*``, final save overwriting ``pytorch_model.bin`` with the
full ``state_dict()``.  Replaced: HF Trainer/accelerate/DeepSpeed (see train/trainer_base.py, train/engine.py).  The CPU data
pipeline of the reference (LazySupervisedDataset, preprocess_phi, tokenizer; SURVEY section 8f row N1) lives in ``llavamod/data``;
``--data_path synthetic[:N]`` serves seeded synthetic samples of the named shape without a tokenizer.
"""
import glob
import os
import sys
import types

import torch
import torch.distributed as dist

from ..config.args import AlignArguments, DataArguments, ModelArguments, TrainingArguments, parse_args_into_dataclasses
from ..constants import IGNORE_INDEX, IMAGE_TOKEN_INDEX
from ..model import (LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM, LlavaQwen2Config, LlavaQwen2ForCausalLM,
                     LLaVAMoDQwen1_5Config, LLaVAMoDQwen1_5ForCausalLM, LLaVAMoDQwen1_5ForCausalLMFineTune,
                     LLaVAMoDQwen2Config, LLaVAMoDQwen2ForCausalLM, LLaVAMoDQwen2ForCausalLMFineTune)
from ..model import synthetic as S
from .align_trainer import AlignTrainer


def rank0_print(*a):
    if not dist.is_initialized() or dist.get_rank() == 0:
        print(*a, flush=True)


def pick_classes(name, sparse, moe_finetune):
    """Dispatch by substring of the lower-cased checkpoint path (reference: align_train.py:29-32,54-79,129-182)."""
    n = name.lower()
    if "qwen2" in n or "qwen-2" in n:
        fam = (LlavaQwen2Config, LlavaQwen2ForCausalLM, LLaVAMoDQwen2Config, LLaVAMoDQwen2ForCausalLM, LLaVAMoDQwen2ForCausalLMFineTune)
    elif "qwen1.5" in n or "qwen-1.5" in n:
        fam = (LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM, LLaVAMoDQwen1_5Config, LLaVAMoDQwen1_5ForCausalLM, LLaVAMoDQwen1_5ForCausalLMFineTune)
    else:
        raise NotImplementedError("only the Qwen-1.5 / Qwen-2 families are on the distillation hot path (got %r)" % name)
    if not sparse:
        return fam[0], fam[1]
    return fam[2], (fam[4] if moe_finetune else fam[3])


def _arch_from_name(name):
    n = os.path.basename(name.rstrip("/")).lower()
    for k in S.ARCH:
        if k.replace("qwen1.5-", "") in n and ("1.5" in n or "1_5" in n):
            return S.ARCH[k]
    raise FileNotFoundError(name)


def init_process(seed):
    """One process per GPU (torchrun-style env): joins the NCCL group when WORLD_SIZE > 1, seeds torch; -> this rank's device."""
    if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1 and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    torch.manual_seed(seed)
    return torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))


def create_model_tokenizer(model_args, data_args, training_args, name_or_path, model_type, pretrain_adapter=None, device="cuda"):
    sparse = model_type == "sparse"
    if sparse:
        model_args.moe_enable = True                                  # align_train.py:29-32
    cfg_cls, cls = pick_classes(name_or_path, sparse, training_args.moe_finetune)
    dtype = torch.bfloat16 if training_args.bf16 else torch.float32
    if os.path.isdir(name_or_path) and os.path.exists(os.path.join(name_or_path, "config.json")):
        cfg = cfg_cls.from_pretrained(name_or_path)
        model = cls.from_pretrained(name_or_path, config=cfg, device=device, torch_dtype=dtype)
    elif os.environ.get("LLAVAMOD_ALLOW_RANDOM_INIT", "0") == "1":
        cfg = cfg_cls(**_arch_from_name(name_or_path), use_cache=False)
        model = cls(cfg, device=device, dtype=dtype)
        rank0_print("WARNING: %s not found locally -> random-init weights of that architecture" % name_or_path)
    else:
        raise FileNotFoundError("%s: no local checkpoint (no network); set LLAVAMOD_ALLOW_RANDOM_INIT=1 for synthetic weights" % name_or_path)
    model.config.use_cache = False
    if getattr(model_args, "freeze_backbone", False):                 # align_train.py:255-256
        model.model.requires_grad_(False)
    if getattr(model_args, "tune_llm_ffn_only", False):               # align_train.py:258-266
        for name, param in model.named_parameters():
            if "image_tower" not in name:
                param.requires_grad = any(n in name for n in ("mlp.gate_proj", "mlp.up_proj", "mlp.down_proj"))
    if sparse:
        model.initialize_moe_modules(model_args)
    if model_args.image_tower is not None:
        margs = types.SimpleNamespace(**vars(model_args))
        margs.pretrain_mm_mlp_adapter = pretrain_adapter
        model.get_model().initialize_vision_modules(margs)
        model.config.image_aspect_ratio = data_args.image_aspect_ratio
        model.config.tokenizer_padding_side = "right"
        model.config.tune_mm_mlp_adapter = training_args.tune_mm_mlp_adapter = model_args.tune_mm_mlp_adapter      # align_train.py:473-477
        if model_args.tune_mm_mlp_adapter:
            model.requires_grad_(False)
            for p in model.get_model().mm_projector.parameters():
                p.requires_grad = True
        model.config.freeze_mm_mlp_adapter = training_args.freeze_mm_mlp_adapter                                      # align_train.py:479-482
        if training_args.freeze_mm_mlp_adapter:
            for p in model.get_model().mm_projector.parameters():
                p.requires_grad = False
        model.config.mm_projector_lr = training_args.mm_projector_lr
    return model, None


def prepare_gradient_checkpointing(model, training_args):
    """--gradient_checkpointing on the model being trained (align_train.py:276-281, dpo_train.py:245-247, train.py:278-281); the frozen
    teacher is never differentiated and is left alone.  The trainer switches the decoder's recompute on when training starts."""
    if not training_args.gradient_checkpointing:
        return
    if model.config.use_cache:
        rank0_print("`use_cache=True` is incompatible with gradient checkpointing: use_cache=False while training")
        model.config.use_cache = False
    model.enable_input_require_grads()


class SyntheticMimicDataset(torch.utils.data.Dataset):
    """Seeded samples of the named shape (SURVEY section 8d): one <image>, 40 % instruction mask."""

    def __init__(self, n, text_len, vocab, image_size, seed=0):
        self.n, self.text_len, self.vocab, self.image_size, self.seed = n, text_len, vocab, image_size, seed

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 1000003 + i)
        ids = torch.randint(0, self.vocab, (self.text_len,), generator=g)
        ids[5] = IMAGE_TOKEN_INDEX
        labels = ids.clone()
        labels[: int(0.4 * self.text_len)] = IGNORE_INDEX
        return dict(input_ids=ids, labels=labels, image=torch.randn(3, self.image_size, self.image_size, generator=g).to(torch.bfloat16))


def collate(instances, pad_id=0):
    """Batch layout of DataCollatorForSupervisedDataset (reference: data/dataset.py:187-225)."""
    ids = torch.nn.utils.rnn.pad_sequence([x["input_ids"] for x in instances], batch_first=True, padding_value=pad_id)
    labels = torch.nn.utils.rnn.pad_sequence([x["labels"] for x in instances], batch_first=True, padding_value=IGNORE_INDEX)
    lens = torch.tensor([x["input_ids"].shape[0] for x in instances])
    mask = torch.arange(ids.shape[1])[None] < lens[:, None]
    return dict(input_ids=ids, labels=labels, attention_mask=mask, images=[x["image"] for x in instances])


def load_tokenizer(model_args, training_args, name_or_path):
    """Qwen-1.5 / Qwen-2 branch of the reference (align_train.py:360-369,436-441): slow AutoTokenizer, right padding, `<|extra_0|>` as
    unk, pad = unk, and the conversation template picked by --version."""
    import transformers
    from .. import conversation as conversation_lib
    tok = transformers.AutoTokenizer.from_pretrained(name_or_path, cache_dir=training_args.cache_dir,
                                                     model_max_length=training_args.model_max_length, padding_side="right", use_fast=False)
    tok.add_special_tokens({"unk_token": "<|extra_0|>"})
    tok.pad_token = tok.unk_token
    conversation_lib.set_default_conversation(model_args.version)
    return tok


def make_supervised_data_module(data_args, training_args, model, tokenizer=None):
    path = (data_args.data_path or ["synthetic"])[0]
    if not str(path).startswith("synthetic"):
        # SURVEY 8f row N1: the reference's lazy JSON dataset + collator (llavamod/data/dataset.py)
        from ..data.dataset import make_supervised_data_module as make_json_module
        if tokenizer is None:
            raise ValueError("--data_path %s needs a tokenizer next to the policy checkpoint" % path)
        data_args.image_processor = model.get_image_tower().image_processor
        data_args.is_multimodal = True
        if not hasattr(data_args, "mm_use_im_start_end"):           # set from --mm_use_im_start_end by the entry points (align_train.py:487)
            data_args.mm_use_im_start_end = False
        return make_json_module(tokenizer, data_args)
    n = int(path.split(":")[1]) if ":" in path else 1024
    tower = model.get_image_tower()
    text_len = training_args.model_max_length - tower.num_patches + 1
    ds = SyntheticMimicDataset(n, text_len, model.config.vocab_size, tower.config.image_size, training_args.seed)
    return dict(train_dataset=ds, eval_dataset=None, data_collator=collate)


def train(argv=None):
    model_args, data_args, training_args, align_args = parse_args_into_dataclasses(
        (ModelArguments, DataArguments, TrainingArguments, AlignArguments), argv)
    device = init_process(training_args.seed)
    if training_args.deepspeed:
        rank0_print("note: --deepspeed %s accepted and ignored (plain data parallelism, resident optimizer state)" % training_args.deepspeed)
    model, _ = create_model_tokenizer(model_args, data_args, training_args, align_args.policy_model_name_or_path,
                                      align_args.policy_model_type, align_args.policy_pretrain_mm_mlp_adapter, device)
    prepare_gradient_checkpointing(model, training_args)
    ref_args = types.SimpleNamespace(**vars(model_args))
    ref_model, _ = create_model_tokenizer(ref_args, data_args, training_args, align_args.ref_model_name_or_path,
                                          align_args.ref_model_type, align_args.ref_pretrain_mm_mlp_adapter, device)
    training_args.moe_enable = model_args.moe_enable
    training_args.tune_mm_mlp_adapter = model_args.tune_mm_mlp_adapter
    model.config.mm_use_im_start_end = data_args.mm_use_im_start_end = model_args.mm_use_im_start_end      # align_train.py:487
    path = (data_args.data_path or ["synthetic"])[0]
    tokenizer = None
    if not str(path).startswith("synthetic"):
        tokenizer = load_tokenizer(model_args, training_args, align_args.policy_model_name_or_path)
        model.config.pad_token_id = tokenizer.pad_token_id                               # align_train.py:437
    data_module = make_supervised_data_module(data_args, training_args, model, tokenizer)
    trainer = AlignTrainer(model=model, ref_model=ref_model, args=training_args, loss_type=align_args.loss_type,
                           moe_loss_enable=align_args.moe_loss_enable, ref_fp8=align_args.ref_fp8, tokenizer=tokenizer, **data_module)
    resume = bool(glob.glob(os.path.join(training_args.output_dir, "checkpoint-*")))     # align_train.py:601-604
    trainer.train(resume_from_checkpoint=resume)
    model.config.use_cache = True
    if not dist.is_initialized() or dist.get_rank() == 0:                                # align_train.py:623-631
        model.config.save_pretrained(training_args.output_dir)
        sd = {k.replace("base_model.model.", "").replace("base_model.", ""): v.detach().cpu() for k, v in model.state_dict().items()}
        torch.save(sd, os.path.join(training_args.output_dir, "pytorch_model.bin"))
    return trainer


if __name__ == "__main__":
    train()
