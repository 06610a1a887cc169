"""Preference-distillation entry point (reference: llavamod/train/dpo_train.py:470-589; preference_distillation.sh:48).
Same construction as align_train; data = chosen / rejected pairs sharing one image (reference: data/dataset.py:465-501)."""
import glob
import os
import types

import torch
import torch.distributed as dist

from ..config.args import DataArguments, DPOArguments, ModelArguments, TrainingArguments, parse_args_into_dataclasses
from ..constants import IGNORE_INDEX
from .align_train import SyntheticMimicDataset, create_model_tokenizer, init_process, prepare_gradient_checkpointing
from .dpo_trainer import DPOTrainer


class SyntheticDPODataset(SyntheticMimicDataset):
    """chosen / rejected share the first 40 % (instruction + image) and differ in the response (SURVEY section 8d)."""

    def __getitem__(self, i):
        a = super().__getitem__(i)
        g = torch.Generator().manual_seed(self.seed * 7000003 + i)
        rej = a["input_ids"].clone()
        k = int(0.4 * self.text_len)
        rej[k:] = torch.randint(0, self.vocab, (self.text_len - k,), generator=g)
        rl = rej.clone()
        rl[:k] = IGNORE_INDEX
        return dict(chosen_input_ids=a["input_ids"], chosen_labels=a["labels"], rejected_input_ids=rej, rejected_labels=rl, image=a["image"])


def collate_dpo(instances, pad_id=0):
    out = {}
    for side in ("chosen", "rejected"):
        ids = torch.nn.utils.rnn.pad_sequence([x[side + "_input_ids"] for x in instances], batch_first=True, padding_value=pad_id)
        labels = torch.nn.utils.rnn.pad_sequence([x[side + "_labels"] for x in instances], batch_first=True, padding_value=IGNORE_INDEX)
        lens = torch.tensor([x[side + "_input_ids"].shape[0] for x in instances])
        out[side + "_input_ids"], out[side + "_labels"] = ids, labels
        out[side + "_attention_mask"] = torch.arange(ids.shape[1])[None] < lens[:, None]
    out["images"] = [x["image"] for x in instances]
    return out


def train(argv=None):
    model_args, data_args, training_args, dpo_args = parse_args_into_dataclasses(
        (ModelArguments, DataArguments, TrainingArguments, DPOArguments), argv)
    device = init_process(training_args.seed)
    model, _ = create_model_tokenizer(model_args, data_args, training_args, dpo_args.policy_model_name_or_path, dpo_args.policy_model_type, None, device)
    prepare_gradient_checkpointing(model, training_args)
    ref_model, _ = create_model_tokenizer(types.SimpleNamespace(**vars(model_args)), data_args, training_args, dpo_args.ref_model_name_or_path,
                                          dpo_args.ref_model_type, None, device)
    training_args.moe_enable = model_args.moe_enable
    path = (data_args.data_path or ["synthetic"])[0]
    tower = model.get_image_tower()
    if not str(path).startswith("synthetic"):
        # SURVEY 8f row N1: RLAIF-V style preference JSON through the reference's lazy dataset + collator (data/dataset.py:253-517)
        from ..data.dataset import make_dpo_data_module
        from .align_train import load_tokenizer
        tokenizer = load_tokenizer(model_args, training_args, dpo_args.policy_model_name_or_path)
        model.config.pad_token_id = tokenizer.pad_token_id
        data_args.image_processor = tower.image_processor
        data_args.is_multimodal = True
        data_args.mm_use_im_start_end = model.config.mm_use_im_start_end = bool(getattr(model_args, "mm_use_im_start_end", False))   # dpo_train.py: same line as align_train.py:487
        data_module = make_dpo_data_module(tokenizer, data_args)
    else:
        tokenizer = None
        n = int(path.split(":")[1]) if ":" in path else 1024
        ds = SyntheticDPODataset(n, training_args.model_max_length - tower.num_patches + 1, model.config.vocab_size, tower.config.image_size,
                                 training_args.seed)
        data_module = dict(train_dataset=ds, eval_dataset=None, data_collator=collate_dpo)
    trainer = DPOTrainer(model=model, ref_model=ref_model, args=training_args, loss_type=dpo_args.loss_type,
                         moe_loss_enable=dpo_args.moe_loss_enable, ref_fp8=dpo_args.ref_fp8, tokenizer=tokenizer, **data_module)
    trainer.train(resume_from_checkpoint=bool(glob.glob(os.path.join(training_args.output_dir, "checkpoint-*"))))
    if not dist.is_initialized() or dist.get_rank() == 0:
        model.config.save_pretrained(training_args.output_dir)
        torch.save({k: v.detach().cpu() for k, v in model.state_dict().items()}, os.path.join(training_args.output_dir, "pytorch_model.bin"))
    return trainer


if __name__ == "__main__":
    train()
