"""Cached decoding restated on the oracle's pieces (oracle/restated.py), in any float dtype on the CPU.

Restates the past_key_value branch of Qwen2SdpaAttention.forward (modeling_qwen2.py:652-728: k / v of the new rows concatenated onto the
layer's cache by DynamicCache.update, cache_utils.py, then SDPA of the new queries over every cached key) and the cached step of
MoEQwen1_5Model_forward (llava_qwen1_5_moe.py:223-236, 308-325): the MoE layers route the tokens of this forward only, so a decode step
runs top2gating with S = B and capacity ceil(B/E * cf * 2) raised to min_capacity.  Position of a cached step: the cache length, as
llava_arch.py:162-172 computes it for unpadded prompts."""
import dataclasses

import torch
import torch.nn.functional as F

from oracle import restated as R


def attention_cached(sd, pre, cfg, x, position_ids, cos, sin, past):
    """-> (o_proj output [B,T,H], present (k, v) [B, nkv, P + T, hd])."""
    B, T, _ = x.shape
    nh, nkv, hd = cfg.heads, cfg.kv_heads, cfg.head_dim
    q = F.linear(x, sd[pre + "q_proj.weight"], sd[pre + "q_proj.bias"]).view(B, T, nh, hd).transpose(1, 2)
    k = F.linear(x, sd[pre + "k_proj.weight"], sd[pre + "k_proj.bias"]).view(B, T, nkv, hd).transpose(1, 2)
    v = F.linear(x, sd[pre + "v_proj.weight"], sd[pre + "v_proj.bias"]).view(B, T, nkv, hd).transpose(1, 2)
    q, k = R.apply_rope(q, k, cos, sin, position_ids)
    if past is not None:
        k = torch.cat([past[0], k], dim=2)
        v = torch.cat([past[1], v], dim=2)
    present = (k, v)
    S = k.shape[2]
    if nkv != nh:
        rep = nh // nkv
        k = k[:, :, None].expand(B, nkv, rep, S, hd).reshape(B, nh, S, hd)
        v = v[:, :, None].expand(B, nkv, rep, S, hd).reshape(B, nh, S, hd)
    visible = torch.ones(T, S, dtype=torch.bool).tril(S - T)           # new row t sits at position S - T + t
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=visible)
    o = o.transpose(1, 2).reshape(B, T, nh * hd)
    return F.linear(o, sd[pre + "o_proj.weight"]), present


def lm_forward_cached(sd, cfg, inputs_embeds, past=None, moe_noise=None, record=None, capacity_factor=None):
    """Qwen2Model.forward with a cache on unpadded sequences.  past: per-layer (k, v) or None (prefill).  moe_noise: one [B*T, E] tensor per
    MoE layer.  capacity_factor: the routing capacity factor (eval_capacity_factor in eval).  -> (final-normed hidden, presents, l_aux list)."""
    B, T, _ = inputs_embeds.shape
    P = 0 if past is None else past[0][0].shape[2]
    mcfg = dataclasses.replace(cfg, capacity_factor=capacity_factor) if capacity_factor is not None else cfg
    position_ids = torch.arange(P, P + T).unsqueeze(0).expand(B, T)
    cos, sin = R.rope_cache(cfg.head_dim, P + T, cfg.rope_theta, inputs_embeds.dtype)
    h = inputs_embeds
    presents, l_auxes = [], []
    for i in range(cfg.layers):
        p = f"{R.P_LM}layers.{i}."
        x = R.rmsnorm(h, sd[p + "input_layernorm.weight"], cfg.eps)
        a, present = attention_cached(sd, p + "self_attn.", cfg, x, position_ids, cos, sin, None if past is None else past[i])
        presents.append(present)
        h = h + a
        x = R.rmsnorm(h, sd[p + "post_attention_layernorm.weight"], cfg.eps)
        if i in cfg.moe_layers:
            y, l_aux, _ = R.moe_layer(sd, p + "mlp.deepspeed_moe.", mcfg, x, moe_noise[cfg.moe_layers.index(i)], record)
            l_auxes.append(l_aux)
        else:
            y = R.mlp(sd, p + "mlp.", x)
        h = h + y
    return R.rmsnorm(h, sd[R.P_LM + "norm.weight"], cfg.eps), presents, l_auxes


def llava_decode(sd, cfg, clip_cfg, input_ids, images, tokens):
    """LlavaQwen1_5ForCausalLM with use_cache=True on unpadded prompts (dense): the prefill over the spliced prompt, then one cached step
    per column of tokens [B, N].  -> (fp32 logits [N + 1, B, V]: the prefill's last position, then every step; per-layer (k, v))."""
    w = sd[R.P_LM + "embed_tokens.weight"]
    if images is not None:
        feats = R.encode_images(sd, clip_cfg, cfg.proj_depth, torch.stack(list(images)))
        src, _, _, _, img = R.splice_plan(input_ids, None, None, feats.shape[1])
        emb = R.splice_embed(w, feats, src, img)
    else:
        emb = w[input_ids]
    h, past, _ = lm_forward_cached(sd, cfg, emb)
    logits = [lm_head(sd, cfg, h[:, -1]).float()]
    for t in range(tokens.shape[1]):
        h, past, _ = lm_forward_cached(sd, cfg, w[tokens[:, t:t + 1]], past)
        logits.append(lm_head(sd, cfg, h[:, -1]).float())
    return torch.stack(logits), past


def lm_head(sd, cfg, hidden):
    w = sd[R.P_LM + "embed_tokens.weight"] if cfg.tie and "lm_head.weight" not in sd else sd["lm_head.weight"]
    return F.linear(hidden, w)
