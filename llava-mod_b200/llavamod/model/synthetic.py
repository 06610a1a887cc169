"""Random-init construction of teacher / student pairs at a named architecture (there are no checkpoints or network in
the build environment; throughput does not depend on weight values).  Follows the reference's construction order:
build -> initialize_moe_modules (freeze by name, wrap MoE) -> initialize_vision_modules (re-enable projector grads)
(llavamod/train/align_train.py:151-157,328,448-451)."""
import types

import torch

from .language_model.llava_qwen1_5 import LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM
from .language_model.llava_qwen1_5_moe import LLaVAMoDQwen1_5Config, LLaVAMoDQwen1_5ForCausalLM

ARCH = {
    "qwen1.5-0.5b": dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=24, num_attention_heads=16,
                         num_key_value_heads=16, vocab_size=151936, rope_theta=1e6, tie_word_embeddings=True),
    "qwen1.5-1.8b": dict(hidden_size=2048, intermediate_size=5504, num_hidden_layers=24, num_attention_heads=16,
                         num_key_value_heads=16, vocab_size=151936, rope_theta=1e6, tie_word_embeddings=False),
    "qwen1.5-7b": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                       num_key_value_heads=32, vocab_size=151936, rope_theta=1e6, tie_word_embeddings=False),
    # config 1 of BASELINE.json (2-layer / 128-d); 2 heads -> head_dim 64, so the wgmma attention kernel is the one that runs
    "tiny": dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2,
                 num_key_value_heads=2, vocab_size=512, rope_theta=1e6, tie_word_embeddings=False),
}
CLIP = {
    "clip-l-336": dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                       image_size=336, patch_size=14),
    "tiny": dict(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=1, image_size=32, patch_size=8),
}

TRAIN_MODULES = ["mlp.gate_proj", "mlp.up_proj", "mlp.down_proj", "wg"]      # dense2sparse_distillation.sh


def vision_args(clip):
    return types.SimpleNamespace(image_tower=dict(clip), video_tower=None, mm_vision_select_layer=-2,
                                 mm_vision_select_feature="patch", pretrain_mm_mlp_adapter=None,
                                 image_projector_type="mlp2x_gelu")


def moe_args(num_experts=4, capacity_factor=1.5, moe_mode="sparse", train_modules=TRAIN_MODULES, aux=0.01, min_capacity=0, top_k=2,
             use_residual=False):
    return types.SimpleNamespace(moe_enable=True, train_modules=list(train_modules) if train_modules else None, moe_mode=moe_mode,
                                 moe_layers_idx=None, ep_size=1, top_k_experts=top_k, capacity_factor=capacity_factor,
                                 eval_capacity_factor=2.0, min_capacity=min_capacity, use_residual=use_residual,
                                 router_aux_loss_coef=aux, num_experts=[num_experts])


def _common_cfg(arch, clip):
    d = dict(ARCH[arch]) if isinstance(arch, str) else dict(arch)
    c = dict(CLIP[clip]) if isinstance(clip, str) else dict(clip)
    d.update(mm_image_tower=c, image_projector_type="mlp2x_gelu", mm_hidden_size=c["hidden_size"],
             mm_vision_select_layer=-2, mm_vision_select_feature="patch", use_cache=False)
    return d, c


def make_teacher(arch="qwen1.5-7b", clip="clip-l-336", device="cuda", dtype=torch.bfloat16, seed=0):
    torch.manual_seed(seed)
    d, c = _common_cfg(arch, clip)
    m = LlavaQwen1_5ForCausalLM(LlavaQwen1_5Config(**d), device=device, dtype=dtype)
    m.get_model().initialize_vision_modules(vision_args(c))
    for p in m.parameters():
        p.requires_grad = False
    return m.eval()


def make_student(arch="qwen1.5-0.5b", clip="clip-l-336", device="cuda", dtype=torch.bfloat16, seed=1, margs=None, share_tower_with=None):
    torch.manual_seed(seed)
    d, c = _common_cfg(arch, clip)
    m = LLaVAMoDQwen1_5ForCausalLM(LLaVAMoDQwen1_5Config(**d), device=device, dtype=dtype)
    m.initialize_moe_modules(margs if margs is not None else moe_args())
    m.get_model().initialize_vision_modules(vision_args(c))
    if share_tower_with is not None:      # both models load the same frozen CLIP checkpoint in every recipe of the reference
        src = share_tower_with.get_image_tower().state_dict()
        m.get_image_tower().load_state_dict(src)
    return m.train()
