"""`load_pretrained_model` for the eval path (SURVEY section 8f row N4; reference llavamod/model/builder.py:57-621).

Qwen-1.5 / Qwen-2 branches only, picked by substrings of `model_name` exactly like the reference (builder.py:370-392): `moe` in the name ->
`EvalLLaVAMoD...ForCausalLM` (experts rebuilt from `config.moe`), else the dense `LlavaQwen...ForCausalLM`.  What the reference wraps
around it and is not carried: `deepspeed.init_inference` (a no-op wrapper at ep_size 1 / no kernel injection), LoRA merging, 4/8-bit
loading, the other LLM families.  Returns `(tokenizer, model, processor, context_len)`."""
import os
import warnings

import torch

from ..constants import DEFAULT_IM_END_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_VID_END_TOKEN, DEFAULT_VID_START_TOKEN
from .language_model.llava_qwen1_5 import LlavaQwen1_5ForCausalLM
from .language_model.llava_qwen1_5_moe import EvalLLaVAMoDQwen1_5ForCausalLM
from .language_model.llava_qwen2 import LlavaQwen2ForCausalLM
from .language_model.llava_qwen2_moe import EvalLLaVAMoDQwen2ForCausalLM

DEFAULT_VIDEO_PATCH_TOKEN = "<im_patch>"


def pick_eval_class(model_name):
    n = model_name.lower()
    if "qwen" not in n:
        raise NotImplementedError("load_pretrained_model: only the Qwen-1.5 / Qwen-2 LLaVA-MoD checkpoints are on this path (got %r)" % model_name)
    if "qwen1.5" in n or "qwen-1.5" in n:
        return EvalLLaVAMoDQwen1_5ForCausalLM if "moe" in n else LlavaQwen1_5ForCausalLM
    if "qwen2" in n or "qwen-2" in n:
        return EvalLLaVAMoDQwen2ForCausalLM if "moe" in n else LlavaQwen2ForCausalLM
    raise NotImplementedError("load_pretrained_model: Qwen-1.0 checkpoints (%r) are outside the distillation path" % model_name)


def load_pretrained_model(model_path, model_base, model_name, load_8bit=False, load_4bit=False, device_map="auto", device="cuda",
                          padding_side="right", merge=False, tokenizer=None, **kwargs):
    if load_8bit or load_4bit:
        raise NotImplementedError("4/8-bit loading is not built; a frozen dense model runs in 8 bits on the H100 as FP8 (e4m3): "
                                  "model.quantize_fp8_() after loading, or --ref_fp8 for the teacher of the distillation recipes")
    if "lora" in model_name.lower() or model_base is not None:
        raise NotImplementedError("LoRA / base+projector loading is not built (the distillation recipes save full state dicts)")
    if "llava" not in model_name.lower():
        warnings.warn("model_name %r does not contain 'llava': the reference would load a plain language model here" % model_name)
    if tokenizer is None:
        import transformers
        tokenizer = transformers.AutoTokenizer.from_pretrained(model_path, use_fast=False, padding_side=padding_side)
    cls = pick_eval_class(model_name)
    model = cls.from_pretrained(model_path, device=device, torch_dtype=kwargs.get("torch_dtype", torch.bfloat16))
    model.config.eos_token_id = tokenizer.eos_token_id                       # builder.py:392
    model.eval()
    processor = {"image": None, "video": None}
    if getattr(model.config, "mm_use_im_patch_token", True):                 # builder.py:581-588
        tokenizer.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN], special_tokens=True)
        tokenizer.add_tokens([DEFAULT_VIDEO_PATCH_TOKEN], special_tokens=True)
    if getattr(model.config, "mm_use_im_start_end", False):
        tokenizer.add_tokens([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN], special_tokens=True)
        tokenizer.add_tokens([DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN], special_tokens=True)
    model.resize_token_embeddings(len(tokenizer))
    if getattr(model.config, "mm_image_tower", None) is not None:
        tower = model.get_image_tower()
        if not tower.is_loaded:
            tower.load_model()
        processor["image"] = tower.image_processor
    context_len = getattr(model.config, "max_sequence_length", 2048)
    return tokenizer, model, processor, context_len
