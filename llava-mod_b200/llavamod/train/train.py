"""``python -m llavamod.train.train`` -- the plain-CE stages either side of distillation (SURVEY section 8f row N3).

Reference: llavamod/train/train.py:19-562 with the flags of shells/train/qwen/{pretrain,finetune,finetune_moe}.sh:
  * adaptor pre-training: `--tune_mm_mlp_adapter True --version plain` -- everything frozen except mm_projector (train.py:476-481);
    output = config.json + mm_projector.bin, the file the distillation shells pass as --pretrain_mm_mlp_adapter;
  * dense SFT: all language-model parameters train (tower frozen, `--freeze_mm_mlp_adapter` optional, train.py:483-486);
  * MoE fine-tuning: `--moe_enable True --train_modules ...` -> initialize_moe_modules (train.py:291-333), final pytorch_model.bin is
    the full state dict with the `base_model.` / `model.` wrappers stripped (train.py:549-556).
Kept out: LoRA / 4-8-bit (`--lora_enable`, `--bits`), non-Qwen families, `initialize_vision_tokenizer` extra tokens
(`--mm_use_im_start_end` / `--mm_use_im_patch_token True` resize the embedding matrix; the Qwen shells run with both off)."""
import glob
import os
import types

import torch
import torch.distributed as dist

from ..config.args import DataArguments, ModelArguments, TrainingArguments, parse_args_into_dataclasses
from .align_train import (create_model_tokenizer, init_process, load_tokenizer, make_supervised_data_module,
                          prepare_gradient_checkpointing)
from .llava_trainer import LLaVATrainer
from .train_utils import safe_save_model_for_hf_trainer


def select_trainable(model, model_args, training_args):
    """train.py:476-486 (after initialize_moe_modules has applied --train_modules for the sparse classes)."""
    model.config.tune_mm_mlp_adapter = training_args.tune_mm_mlp_adapter = model_args.tune_mm_mlp_adapter
    if model_args.tune_mm_mlp_adapter:
        model.requires_grad_(False)
        for p in model.get_model().mm_projector.parameters():
            p.requires_grad = True
    elif not model_args.moe_enable:
        for n, p in model.named_parameters():          # dense SFT: the whole language model + projector; the tower stays frozen
            p.requires_grad = "image_tower" not in n
    model.config.freeze_mm_mlp_adapter = training_args.freeze_mm_mlp_adapter
    if training_args.freeze_mm_mlp_adapter:
        for p in model.get_model().mm_projector.parameters():
            p.requires_grad = False


def train(argv=None):
    model_args, data_args, training_args = parse_args_into_dataclasses((ModelArguments, DataArguments, TrainingArguments), argv)
    if training_args.lora_enable or training_args.bits in (4, 8):
        raise NotImplementedError("LoRA / 4-8-bit training is outside the Qwen distillation path")
    if model_args.mm_use_im_start_end:
        raise NotImplementedError("--mm_use_im_start_end adds tokens and resizes the embeddings (initialize_vision_tokenizer); the Qwen shells keep it off")
    device = init_process(training_args.seed)
    model, _ = create_model_tokenizer(model_args, data_args, training_args, model_args.model_name_or_path,
                                      "sparse" if model_args.moe_enable else "dense", model_args.pretrain_mm_mlp_adapter, device)
    training_args.moe_enable = model_args.moe_enable
    model.config.mm_use_im_start_end = data_args.mm_use_im_start_end = model_args.mm_use_im_start_end      # train.py (reference): same assignment
    select_trainable(model, model_args, training_args)
    prepare_gradient_checkpointing(model, training_args)
    path = (data_args.data_path or ["synthetic"])[0]
    tokenizer = None
    if not str(path).startswith("synthetic"):
        tokenizer = load_tokenizer(model_args, training_args, model_args.model_name_or_path)
        model.config.pad_token_id = tokenizer.pad_token_id
    data_module = make_supervised_data_module(data_args, training_args, model, tokenizer)
    trainer = LLaVATrainer(model=model, tokenizer=tokenizer, args=training_args, **data_module)
    trainer.train(resume_from_checkpoint=bool(glob.glob(os.path.join(training_args.output_dir, "checkpoint-*"))))      # train.py:527-530
    model.config.use_cache = True
    safe_save_model_for_hf_trainer(trainer=trainer, output_dir=training_args.output_dir)
    if model_args.moe_enable and (not dist.is_initialized() or dist.get_rank() == 0):                                  # train.py:549-556
        sd = {(k[11:] if k.startswith("base_model.") else k): v.detach().cpu() for k, v in model.state_dict().items()}
        if any(k.startswith("model.model.") for k in sd):
            sd = {(k[6:] if k.startswith("model.") else k): v for k, v in sd.items()}
        torch.save(sd, os.path.join(training_args.output_dir, "pytorch_model.bin"))
        model.config.save_pretrained(training_args.output_dir)
    return trainer


if __name__ == "__main__":
    train()
