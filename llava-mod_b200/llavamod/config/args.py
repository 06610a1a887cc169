"""Flag surface of the distillation entry points (reference: llavamod/config/args.py:8-133, as used by
shells/train/qwen/dense2sparse_distillation.sh:48-88 and preference_distillation.sh:48-88).

``TrainingArguments`` restates the subset of ``transformers.TrainingArguments`` the shells set (HF Trainer / accelerate /
DeepSpeed are not on this path); unknown HF flags are accepted and ignored with a warning so the reference's shell
command lines keep working (``--deepspeed <json>`` is accepted and ignored: plain data parallelism replaces ZeRO-2)."""
import argparse
import dataclasses
import sys
import warnings
from dataclasses import dataclass, field
from typing import List, Optional


@dataclass
class ModelArguments:
    model_name_or_path: Optional[str] = "facebook/opt-125m"
    version: Optional[str] = "v0"
    freeze_backbone: bool = False
    tune_llm_ffn_only: bool = False
    tune_mm_mlp_adapter: bool = False
    mm_vision_select_layer: Optional[int] = -1
    pretrain_mm_mlp_adapter: Optional[str] = None
    mm_use_im_start_end: bool = False
    mm_use_im_patch_token: bool = True
    mm_vision_select_feature: Optional[str] = "patch"
    s2: bool = False
    s2_scales: Optional[str] = "336,672"
    image_tower: Optional[str] = None
    video_tower: Optional[str] = None
    image_projector_type: Optional[str] = "linear"
    video_projector_type: Optional[str] = "linear"
    video_global_proj: bool = False
    video_temproal_proj: bool = False
    video_spatial_proj: bool = False
    only_lora_ffn: bool = True
    moe_enable: bool = False
    train_modules: Optional[List[str]] = None
    moe_mode: str = "second_half"
    moe_layers_idx: Optional[List[int]] = None
    ep_size: int = 1
    num_experts: Optional[List[int]] = field(default_factory=lambda: [4])
    top_k_experts: int = 2
    capacity_factor: float = 1.0
    eval_capacity_factor: float = 2.0
    min_capacity: int = 0
    use_residual: bool = False
    router_aux_loss_coef: float = 0.01


@dataclass
class DataArguments:
    lazy_preprocess: bool = False
    is_multimodal: bool = False
    image_aspect_ratio: str = "square"
    data_path: Optional[List[str]] = None
    image_folder: Optional[str] = None
    video_folder: Optional[str] = None
    num_frames: int = 8


@dataclass
class TrainingArguments:
    output_dir: str = "./checkpoints"
    per_device_train_batch_size: int = 1
    per_device_eval_batch_size: int = 1
    gradient_accumulation_steps: int = 1
    learning_rate: float = 5e-5
    weight_decay: float = 0.0
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_epsilon: float = 1e-8
    max_grad_norm: float = 1.0
    num_train_epochs: float = 3.0
    max_steps: int = -1
    lr_scheduler_type: str = "linear"
    warmup_ratio: float = 0.0
    warmup_steps: int = 0
    logging_steps: int = 500
    save_strategy: str = "steps"
    save_steps: int = 500
    save_total_limit: Optional[int] = None
    evaluation_strategy: str = "no"
    seed: int = 42
    bf16: bool = False
    fp16: bool = False
    tf32: Optional[bool] = None
    gradient_checkpointing: bool = False
    dataloader_num_workers: int = 0
    report_to: Optional[str] = "none"
    deepspeed: Optional[str] = None
    local_rank: int = -1
    run_name: Optional[str] = None
    # LLaVA-MoD additions (reference args.py:77-116)
    cache_dir: Optional[str] = None
    optim: str = "adamw_torch"
    remove_unused_columns: bool = False
    freeze_mm_mlp_adapter: bool = False
    mpt_attn_impl: Optional[str] = "triton"
    model_max_length: int = 512
    double_quant: bool = True
    quant_type: str = "nf4"
    bits: int = 16
    lora_enable: bool = False
    lora_r: int = 128
    lora_alpha: int = 256
    lora_dropout: float = 0.05
    lora_weight_path: str = ""
    lora_bias: str = "none"
    mm_projector_lr: Optional[float] = None
    group_by_modality_length: bool = False
    moe_finetune: bool = False
    distill_all_tokens: bool = False
    attn_implementation: str = "flash_attention_2"
    # set by the entry points (reference: align_train.py copies model flags onto training_args)
    moe_enable: bool = False
    tune_mm_mlp_adapter: bool = False


@dataclass
class AlignArguments:
    policy_model_type: str = "sparse"
    ref_model_type: str = "dense"
    loss_type: str = "only_kd"
    policy_model_name_or_path: Optional[str] = None
    policy_pretrain_mm_mlp_adapter: Optional[str] = None
    ref_model_name_or_path: Optional[str] = None
    ref_pretrain_mm_mlp_adapter: Optional[str] = None
    moe_loss_enable: bool = False


@dataclass
class DPOArguments:
    policy_model_type: str = "sparse"
    ref_model_type: str = "dense"
    loss_type: str = "sigmoid"
    policy_model_name_or_path: Optional[str] = None
    ref_model_name_or_path: Optional[str] = None
    moe_loss_enable: bool = False


def _str2bool(v):
    if isinstance(v, bool):
        return v
    if v.lower() in ("yes", "true", "t", "y", "1"):
        return True
    if v.lower() in ("no", "false", "f", "n", "0"):
        return False
    raise argparse.ArgumentTypeError("boolean expected, got %r" % v)


def parse_args_into_dataclasses(dataclass_types, argv=None):
    """HfArgumentParser.parse_args_into_dataclasses equivalent (reference call: align_train.py:519-521)."""
    parser = argparse.ArgumentParser(allow_abbrev=False)
    owners = {}
    for dt in dataclass_types:
        for f in dataclasses.fields(dt):
            if f.name in owners:
                owners[f.name].append(dt)           # same flag shared by two dataclasses (e.g. loss_type)
                continue
            owners[f.name] = [dt]
            tp = str(f.type)
            kw = {}
            if "bool" in tp:
                kw = dict(type=_str2bool, nargs="?", const=True)
            elif "List[int]" in tp:
                kw = dict(type=int, nargs="+")
            elif "List[str]" in tp:
                kw = dict(type=str, nargs="+")
            elif "int" in tp:
                kw = dict(type=int)
            elif "float" in tp:
                kw = dict(type=float)
            else:
                kw = dict(type=str)
            parser.add_argument("--" + f.name, dest=f.name, default=argparse.SUPPRESS, **kw)
    ns, unknown = parser.parse_known_args(argv)
    if unknown:
        warnings.warn("ignoring flags outside the distillation path: %s" % " ".join(unknown))
    given = vars(ns)
    out = []
    for dt in dataclass_types:
        names = {f.name for f in dataclasses.fields(dt)}
        out.append(dt(**{k: v for k, v in given.items() if k in names}))
    return tuple(out)
