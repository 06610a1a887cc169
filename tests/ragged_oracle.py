"""Cached decoding of a PADDED prompt batch restated on the oracle's pieces (oracle/restated.py), in any float dtype on the CPU: the
function generate() computes for prompts of different lengths (llavamod/model/generation.py).

  * prefill: the padded forward (R.sdpa_mask: each row sees its own real keys, causally; rows with no visible key see every key, as HF
    does), with compact positions 0 .. n_b - 1 over sequence b's real rows (pad rows at 0).  MoE layers route every row, pads included
    (S = B * T, one capacity for the batch), as DeepSpeed routes a batch.
  * cached step s: sequence b's token sits at position n_b + s and attends to its real prefill keys and its earlier steps' keys only.
    MoE layers route the B step tokens (S = B), as in tests/decode_oracle.py.
  * logits: each sequence's last real row.
For a dense model each sequence's result is then the one it has alone (test_ragged_decode_reference checks that in float64)."""
import dataclasses

import torch
import torch.nn.functional as F

from oracle import restated as R


def compact_positions(mask):
    """[B, T] bool -> int64 positions 0 .. n_b - 1 over the real rows, 0 at the pads (what the splice plan gives spliced prompts)."""
    m = mask.long()
    return (m.cumsum(1) - 1) * m


def _attention(sd, pre, cfg, x, position_ids, cos, sin, past, add_mask):
    """-> (o_proj output [B,T,H], present (k, v) [B, nkv, P + T, hd]); add_mask: additive [B, 1, T, P + T] or None (causal)."""
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
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=add_mask, is_causal=add_mask is None and T > 1)
    return F.linear(o.transpose(1, 2).reshape(B, T, nh * hd), sd[pre + "o_proj.weight"]), present


def _layers(sd, cfg, h, position_ids, past, add_mask, moe_noise, record, capacity_factor):
    mcfg = dataclasses.replace(cfg, capacity_factor=capacity_factor) if capacity_factor is not None else cfg
    n = int(position_ids.max()) + 2
    cos, sin = R.rope_cache(cfg.head_dim, n, cfg.rope_theta, h.dtype)
    presents = []
    for i in range(cfg.layers):
        p = f"{R.P_LM}layers.{i}."
        x = R.rmsnorm(h, sd[p + "input_layernorm.weight"], cfg.eps)
        a, present = _attention(sd, p + "self_attn.", cfg, x, position_ids, cos, sin, None if past is None else past[i], add_mask)
        presents.append(present)
        h = h + a
        x = R.rmsnorm(h, sd[p + "post_attention_layernorm.weight"], cfg.eps)
        if i in cfg.moe_layers:
            y, _, _ = R.moe_layer(sd, p + "mlp.deepspeed_moe.", mcfg, x, moe_noise[cfg.moe_layers.index(i)], record)
        else:
            y = R.mlp(sd, p + "mlp.", x)
        h = h + y
    return R.rmsnorm(h, sd[R.P_LM + "norm.weight"], cfg.eps), presents


def prefill(sd, cfg, emb, mask, moe_noise=None, record=None, capacity_factor=None):
    """Padded prefill.  emb [B,T,H], mask [B,T] bool (each row one run of real rows).  -> (hidden [B,T,H], state) where state holds the
    per-layer (k, v) in the padded layout, the key mask and every sequence's length."""
    B, T, _ = emb.shape
    pos = compact_positions(mask)
    h, past = _layers(sd, cfg, emb, pos, None, R.sdpa_mask(mask, B, T, emb.dtype), moe_noise, record, capacity_factor)
    return h, dict(past=past, keys=mask.clone(), lens=mask.sum(1))


def step(sd, cfg, emb, state, moe_noise=None, record=None, capacity_factor=None):
    """One cached step: emb [B,1,H] at positions lens[b]; attends to the sequence's real keys.  -> hidden [B,1,H]; state advanced."""
    B = emb.shape[0]
    keys = torch.cat([state["keys"], torch.ones(B, 1, dtype=torch.bool)], 1)
    add = torch.zeros(B, 1, 1, keys.shape[1], dtype=emb.dtype).masked_fill(~keys[:, None, None, :], torch.finfo(emb.dtype).min)
    h, past = _layers(sd, cfg, emb, state["lens"][:, None], state["past"], add, moe_noise, record, capacity_factor)
    state.update(past=past, keys=keys, lens=state["lens"] + 1)
    return h


def packed_cache(state, b):
    """Sequence b's cache rows [0, n_b) per layer: (k, v) [nkv, n_b, hd], its real keys in order (the layout of KVCache)."""
    return [(k[b][:, state["keys"][b]], v[b][:, state["keys"][b]]) for k, v in state["past"]]


def last_real(h, mask):
    hi = mask.shape[1] - mask.flip(1).long().argmax(1)
    return h[torch.arange(h.shape[0]), hi - 1]


def lm_head(sd, cfg, hidden):
    w = sd[R.P_LM + "embed_tokens.weight"] if cfg.tie and "lm_head.weight" not in sd else sd["lm_head.weight"]
    return F.linear(hidden, w)


def prompt_embeds(sd, cfg, clip_cfg, input_ids, mask, images, padding_side="right"):
    """Spliced prompt embeddings and the spliced mask (text-only prompts: the token embeddings and the mask as given)."""
    w = sd[R.P_LM + "embed_tokens.weight"]
    if images is None:
        return w[input_ids.clamp(min=0)], mask.bool()
    feats = R.encode_images(sd, clip_cfg, cfg.proj_depth, torch.stack(list(images)).to(w.dtype))
    src, _, nm, _, img = R.splice_plan(input_ids, mask, None, feats.shape[1], padding_side)
    return R.splice_embed(w, feats, src, img), nm


def llava_decode(sd, cfg, clip_cfg, input_ids, mask, images, tokens, padding_side="right"):
    """Dense LlavaQwen1_5ForCausalLM, padded prompt batch, prefill + one teacher-forced cached step per column of tokens [B, N].
    -> (logits [N + 1, B, V], final state)."""
    w = sd[R.P_LM + "embed_tokens.weight"]
    emb, m = prompt_embeds(sd, cfg, clip_cfg, input_ids, mask, images, padding_side)
    h, state = prefill(sd, cfg, emb, m)
    logits = [lm_head(sd, cfg, last_real(h, m))]
    for t in range(tokens.shape[1]):
        h = step(sd, cfg, w[tokens[:, t:t + 1]], state)
        logits.append(lm_head(sd, cfg, h[:, 0]))
    return torch.stack(logits), state
