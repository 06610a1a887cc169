"""TEST INFRASTRUCTURE ONLY -- CPU restatement (plain PyTorch) of the LLaVA-MoD distillation step.

This is the parity oracle for the H100 build.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it; the product package
(``llava-mod_b200/llavamod``) must never do so.

Every function cites the reference file:line it restates (paths relative to the reference root).
State is a flat ``dict[str, Tensor]`` that uses the reference's checkpoint key names (SURVEY.md
section 8b), so the same dict loads into the CUDA model.

Pinning status
  * dense path (Qwen1.5 decoder, CLIP tower, projector, multimodal splice, shifted CE): pinned
    against the reference's own code imported through ``oracle/ref_shim.py``
    (``tests/test_oracle_pin.py``; golden vectors in ``tests/golden/dense_*.pt`` made by
    ``tests/golden/make_golden.py``).
  * DeepSpeed-0.9.5 MoE (``deepspeed.moe.sharded_moe.top2gating`` / ``MOELayer`` / ``Experts``):
    third-party, un-vendored, not installable here -> restated from the published algorithm
    (SURVEY.md Appendix A).  **parity unpinned** for this piece; an independent token-by-token
    simulation of the same published algorithm agrees with it on every routing decision
    (``tests/test_gating_semantics.py``), and the CUDA router is bit-exact against it.
  * trainers (``align_trainer.py:455-594``, ``dpo_trainer.py:462-641``): the files cannot be imported
    (accelerate / deepspeed missing), but their loss code is plain torch: the reference's own method
    bodies (get_p / get_logp / compute_align_loss / compute_loss, DPO get_logp / dpo_loss /
    compute_loss) are exec'd from the read-only tree on fake model outputs by
    ``tests/golden/make_loss_golden.py`` and this module reproduces them in all 15 cases (-inf terms,
    0/0 -> NaN, distill_all_tokens, both moe-loss branches incl. the -1.0 sentinel, every DPO loss
    type, label smoothing): **pinned** (``tests/test_trainer_loss_pin.py``); plus analytic known
    answers (uniform logits -> log V; policy==ref -> log 2 / 0.5).
  * optimizer / schedule / clipping (HF Trainer 4.37 + torch AdamW): pinned against the installed
    ``torch.optim.AdamW``, ``transformers.get_cosine_schedule_with_warmup`` and
    ``torch.nn.utils.clip_grad_norm_`` over 40 steps (same test file) -- transformers here is 5.5,
    not the reference's 4.37, whose formulas are the same.
  * data pipeline: the reference's own ``data/`` code runs here -> ``tests/golden/data_pipeline.pt``
    (``tests/test_data_pipeline.py``; the product's data modules are checked, the oracle has no copy).
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

IGNORE_INDEX = -100        # llavamod/constants.py:6
IMAGE_TOKEN_INDEX = -200   # llavamod/constants.py:8
KD_VOCAB = 151936          # align_trainer.py:473,497  (hard-coded slice)


# ----------------------------------------------------------------------------------------------
# configs
# ----------------------------------------------------------------------------------------------
@dataclass
class ClipCfg:
    hidden: int = 1024
    inter: int = 4096
    layers: int = 24
    heads: int = 16
    image: int = 336
    patch: int = 14
    eps: float = 1e-5
    select_layer: int = -2          # --mm_vision_select_layer -2

    @property
    def n_patches(self):
        return (self.image // self.patch) ** 2


@dataclass
class LMCfg:
    hidden: int = 1024
    inter: int = 2816
    layers: int = 24
    heads: int = 16
    kv_heads: int = 16
    vocab: int = 151936
    rope_theta: float = 1e6
    eps: float = 1e-6
    tie: bool = False
    # MoE (student only).  Defaults follow shells/train/qwen/dense2sparse_distillation.sh:26-42
    moe_layers: List[int] = field(default_factory=list)
    num_experts: int = 4
    top_k: int = 2
    capacity_factor: float = 1.5
    min_capacity: int = 0
    aux_coef: float = 0.01
    proj_depth: int = 2             # mlp2x_gelu
    kd_vocab: int = KD_VOCAB        # tests shrink this together with vocab

    @property
    def head_dim(self):
        return self.hidden // self.heads


P_LM = "model."
P_CLIP = "model.image_tower.image_tower.vision_model."
P_PROJ = "model.mm_projector.image_spatial_proj."


# ----------------------------------------------------------------------------------------------
# Qwen2 dense pieces -- llavamod/model/language_model/qwen1_5/modeling_qwen2.py
# ----------------------------------------------------------------------------------------------
def rmsnorm(x, w, eps):
    """Qwen2RMSNorm.forward  modeling_qwen2.py:105-110 (fp32 variance, weight multiply in input dtype)."""
    dt = x.dtype
    h = x.to(torch.float32)
    var = h.pow(2).mean(-1, keepdim=True)
    h = h * torch.rsqrt(var + eps)
    return w * h.to(dt)


def rope_cache(head_dim, seq_len, theta, dtype):
    """Qwen2RotaryEmbedding._set_cos_sin_cache / forward  modeling_qwen2.py:114-148
    (cache built in fp32, cast to the activation dtype on use)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2).float() / head_dim))
    t = torch.arange(seq_len, dtype=inv_freq.dtype)
    freqs = torch.outer(t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rotate_half(x):
    """modeling_qwen2.py:152-156"""
    x1 = x[..., : x.shape[-1] // 2]
    x2 = x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


def apply_rope(q, k, cos, sin, position_ids):
    """apply_rotary_pos_emb  modeling_qwen2.py:159-184 (q,k are [B,nh,T,hd])."""
    cos = cos[position_ids].unsqueeze(1)
    sin = sin[position_ids].unsqueeze(1)
    return (q * cos) + (rotate_half(q) * sin), (k * cos) + (rotate_half(k) * sin)


def sdpa_mask(attention_mask, B, T, dtype):
    """_prepare_4d_causal_attention_mask_for_sdpa as called at modeling_qwen2.py:1035-1040 /
    llava_qwen1_5_moe.py:255-263: returns None (-> is_causal) when the 2-D mask is None or
    all-ones, else an additive [B,1,T,T] mask with fully-masked rows un-masked (HF
    AttentionMaskConverter._unmask_unattended, used for the memory-efficient SDPA path)."""
    if attention_mask is None or bool(attention_mask.all()):
        return None
    neg = torch.finfo(dtype).min
    causal = torch.full((T, T), neg, dtype=dtype).triu(1)
    m = causal[None, None].expand(B, 1, T, T).clone()
    pad = (~attention_mask.bool())[:, None, None, :].expand(B, 1, T, T)
    m = m.masked_fill(pad, neg)
    # rows with no visible key (left padding) attend to everything, as HF does
    fully = (m == neg).all(-1, keepdim=True)
    m = m.masked_fill(fully, 0.0)
    return m


def attention(sd, pre, cfg: LMCfg, x, mask4d, position_ids, cos, sin):
    """Qwen2SdpaAttention.forward  modeling_qwen2.py:652-728 (training path: no cache, dropout 0)."""
    B, T, _ = x.shape
    nh, nkv, hd = cfg.heads, cfg.kv_heads, cfg.head_dim
    q = F.linear(x, sd[pre + "q_proj.weight"], sd[pre + "q_proj.bias"])
    k = F.linear(x, sd[pre + "k_proj.weight"], sd[pre + "k_proj.bias"])
    v = F.linear(x, sd[pre + "v_proj.weight"], sd[pre + "v_proj.bias"])
    q = q.view(B, T, nh, hd).transpose(1, 2)
    k = k.view(B, T, nkv, hd).transpose(1, 2)
    v = v.view(B, T, nkv, hd).transpose(1, 2)
    q, k = apply_rope(q, k, cos, sin, position_ids)
    if nkv != nh:                                       # repeat_kv :204-213
        rep = nh // nkv
        k = k[:, :, None].expand(B, nkv, rep, T, hd).reshape(B, nh, T, hd)
        v = v[:, :, None].expand(B, nkv, rep, T, hd).reshape(B, nh, T, hd)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask4d, dropout_p=0.0,
                                       is_causal=(mask4d is None and T > 1))
    o = o.transpose(1, 2).contiguous().reshape(B, T, nh * hd)
    return F.linear(o, sd[pre + "o_proj.weight"])


def mlp(sd, pre, x):
    """Qwen2MLP.forward  modeling_qwen2.py:199-200"""
    g = F.linear(x, sd[pre + "gate_proj.weight"])
    u = F.linear(x, sd[pre + "up_proj.weight"])
    return F.linear(F.silu(g) * u, sd[pre + "down_proj.weight"])


# ----------------------------------------------------------------------------------------------
# DeepSpeed 0.9.5 MoE (third-party; restated from the published source, SURVEY.md Appendix A)
#   deepspeed/moe/sharded_moe.py: top2gating, TopKGate.forward, MOELayer.forward
#   deepspeed/moe/experts.py: Experts.forward ; call site llava_qwen1_5_moe.py:536-546
# ----------------------------------------------------------------------------------------------
def gumbel_noise(shape, generator=None):
    """deepspeed/moe/sharded_moe.py gumbel_rsample: Gumbel(0,1).rsample.  The build takes the noise
    as an explicit tensor so that routing is reproducible on both sides (SURVEY.md section 7 'Hard parts')."""
    u = torch.rand(shape, generator=generator).clamp_(min=1e-20)
    return -torch.log(-torch.log(u).clamp_(min=1e-20))


def moe_capacity(num_tokens, num_experts, capacity_factor, min_capacity, k=2):
    """_capacity: ceil(S/E * cf * k) as int64, raised to min_capacity (Appendix A step 3)."""
    cap = int(math.ceil((num_tokens / num_experts) * (capacity_factor * k)))
    return max(cap, int(min_capacity))


def top2gating(logits, noise, capacity_factor, min_capacity):
    """top2gating (Appendix A steps 2-8).  logits fp32 [S,E]; noise fp32 [S,E].
    Returns dict with l_aux, combine_weights [S,E,C], dispatch_mask, and the integer routing
    record (idx1, idx2, slot1, slot2, keep1, keep2, g1, g2, capacity, exp_counts)."""
    S, E = logits.shape
    gates = F.softmax(logits, dim=1)
    C = moe_capacity(S, E, capacity_factor, min_capacity, 2)
    idx1 = torch.argmax(gates, dim=1)
    mask1 = F.one_hot(idx1, num_classes=E)
    logits_w_noise = logits + noise
    logits_except1 = logits_w_noise.masked_fill(mask1.bool(), float("-inf"))
    idx2 = torch.argmax(logits_except1, dim=1)
    mask2 = F.one_hot(idx2, num_classes=E)
    loc1 = torch.cumsum(mask1, dim=0) - 1
    loc2 = torch.cumsum(mask2, dim=0) - 1
    loc2 = loc2 + torch.sum(mask1, dim=0, keepdim=True)
    exp_counts = torch.sum(mask1, dim=0).detach()
    me = torch.mean(gates, dim=0)
    ce = torch.mean(mask1.float(), dim=0)
    l_aux = torch.mean(me * ce) * E * E
    mask1 = mask1 * torch.lt(loc1, C)
    mask2 = mask2 * torch.lt(loc2, C)
    slot1 = torch.sum(loc1 * mask1, dim=1)
    slot2 = torch.sum(loc2 * mask2, dim=1)
    m1f, m2f = mask1.float(), mask2.float()
    g1 = torch.einsum("se,se->s", gates, m1f)
    g2 = torch.einsum("se,se->s", gates, m2f)
    den = torch.clamp(g1 + g2, min=torch.finfo(g1.dtype).eps)
    g1 = g1 / den
    g2 = g2 / den
    gates1 = torch.einsum("s,se->se", g1, m1f)
    gates2 = torch.einsum("s,se->se", g2, m2f)
    l1 = F.one_hot(slot1, num_classes=C).float()
    l2 = F.one_hot(slot2, num_classes=C).float()
    combine = torch.einsum("se,sc->sec", gates1, l1) + torch.einsum("se,sc->sec", gates2, l2)
    return dict(l_aux=l_aux, combine=combine, dispatch=combine.bool(), exp_counts=exp_counts,
                idx1=idx1, idx2=idx2, slot1=slot1, slot2=slot2,
                keep1=mask1.sum(1).bool(), keep2=mask2.sum(1).bool(), g1=g1, g2=g2, capacity=C,
                gates=gates)


def moe_layer(sd, pre, cfg: LMCfg, x, noise, record=None):
    """MoE.forward -> MOELayer.forward (Appendix A steps 1, 9-11); ep_size=1 so both all_to_all are
    identity.  ``pre`` = 'model.layers.{i}.mlp.deepspeed_moe.'; returns (out, l_aux, exp_counts)."""
    shp = x.shape
    xs = x.reshape(-1, shp[-1])
    wg = sd[pre + "gate.wg.weight"]
    logits = F.linear(xs.float(), wg.float())            # TopKGate.forward: fp32 gate
    r = top2gating(logits, noise, cfg.capacity_factor, cfg.min_capacity)
    if record is not None:
        record.append({k: v for k, v in r.items() if k not in ("combine", "dispatch")} | {"logits": logits})
    dispatched = torch.einsum("sec,sm->ecm", r["dispatch"].type_as(xs), xs)         # [E,C,M]
    outs = []
    for e in range(cfg.num_experts):                                                 # Experts.forward
        outs.append(mlp(sd, pre + f"experts.deepspeed_experts.{e}.", dispatched[e]))
    expert_out = torch.stack(outs, 0)
    combined = torch.einsum("sec,ecm->sm", r["combine"].type_as(xs), expert_out)
    return combined.reshape(shp), r["l_aux"], r["exp_counts"]


# ----------------------------------------------------------------------------------------------
# CLIP vision tower + projector
# ----------------------------------------------------------------------------------------------
def clip_tower(sd, cfg: ClipCfg, images, pre=P_CLIP):
    """CLIPVisionTower.forward + feature_select  multimodal_encoder/clip_encoder.py:35-57 over
    transformers.CLIPVisionModel (third-party; architecture: patch conv(no bias)+cls+pos-emb,
    pre_layrnorm, pre-LN encoder layers with quick_gelu).  hidden_states[select_layer] with
    select_layer=-2 == output of encoder layer L-1; CLS dropped."""
    B = images.shape[0]
    dt = sd[pre + "embeddings.patch_embedding.weight"].dtype
    x = F.conv2d(images.to(dt), sd[pre + "embeddings.patch_embedding.weight"], stride=cfg.patch)
    x = x.flatten(2).transpose(1, 2)
    cls = sd[pre + "embeddings.class_embedding"].expand(B, 1, -1)
    x = torch.cat([cls, x], dim=1) + sd[pre + "embeddings.position_embedding.weight"][None]
    x = F.layer_norm(x, (cfg.hidden,), sd[pre + "pre_layrnorm.weight"], sd[pre + "pre_layrnorm.bias"], cfg.eps)
    n_run = cfg.layers + 1 + cfg.select_layer if cfg.select_layer < 0 else cfg.select_layer
    hd = cfg.hidden // cfg.heads
    for i in range(n_run):
        p = f"{pre}encoder.layers.{i}."
        r = x
        h = F.layer_norm(x, (cfg.hidden,), sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"], cfg.eps)
        T = h.shape[1]
        q = F.linear(h, sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.q_proj.bias"])
        k = F.linear(h, sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.k_proj.bias"])
        v = F.linear(h, sd[p + "self_attn.v_proj.weight"], sd[p + "self_attn.v_proj.bias"])
        q = q.view(B, T, cfg.heads, hd).transpose(1, 2)
        k = k.view(B, T, cfg.heads, hd).transpose(1, 2)
        v = v.view(B, T, cfg.heads, hd).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k, v)
        o = o.transpose(1, 2).reshape(B, T, cfg.hidden)
        x = r + F.linear(o, sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"])
        r = x
        h = F.layer_norm(x, (cfg.hidden,), sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"], cfg.eps)
        h = F.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])
        h = h * torch.sigmoid(1.702 * h)                # quick_gelu
        x = r + F.linear(h, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    return x[:, 1:].to(images.dtype)


def projector(sd, depth, feats, pre=P_PROJ):
    """mlp{N}x_gelu  multimodal_projector/builder.py:57-61,148-149: Linear (GELU Linear)*(N-1)."""
    x = F.linear(feats, sd[pre + "0.weight"], sd[pre + "0.bias"])
    for j in range(1, depth):
        x = F.gelu(x)
        x = F.linear(x, sd[pre + f"{2 * j}.weight"], sd[pre + f"{2 * j}.bias"])
    return x


def encode_images(sd, clip_cfg, depth, images):
    """LlavaMetaForCausalLM.encode_images  llava_arch.py:143-148"""
    feats = clip_tower(sd, clip_cfg, images)
    return projector(sd, depth, feats.to(sd[P_PROJ + "0.weight"].dtype))


# ----------------------------------------------------------------------------------------------
# multimodal splice -- llava_arch.py:155-334 (image branch only; videos out of scope)
# ----------------------------------------------------------------------------------------------
def splice_plan(input_ids, attention_mask, labels, n_patches, padding_side="right"):
    """Integer part of prepare_inputs_labels_for_multimodal (llava_arch.py:228-320).
    Returns src [B,Tmax] int64 (>=0: token id to embed; -1-k: row k of this sample's image-feature
    stream, image features consumed in order; PAD_SRC for padding), new_labels, new_mask, pos_ids,
    img_index [B,Tmax] (index of the image in the flat image list, -1 if not an image row)."""
    PAD = -(1 << 40)
    B = input_ids.shape[0]
    if attention_mask is None:
        attention_mask = torch.ones_like(input_ids, dtype=torch.bool)
    attention_mask = attention_mask.bool()
    if labels is None:
        labels = torch.full_like(input_ids, IGNORE_INDEX)
    rows, cur_img = [], 0
    for b in range(B):
        ids = input_ids[b][attention_mask[b]].tolist()
        lab = labels[b][attention_mask[b]].tolist()
        src, nl, im = [], [], []
        n_img = sum(1 for t in ids if t == IMAGE_TOKEN_INDEX)
        if n_img == 0:
            src, nl, im = list(ids), list(lab), [-1] * len(ids)
            cur_img += 1                      # llava_arch.py:238-245 consumes one feature entry
        else:
            for t, l in zip(ids, lab):
                if t == IMAGE_TOKEN_INDEX:
                    src += [-1 - j for j in range(n_patches)]
                    nl += [IGNORE_INDEX] * n_patches
                    im += [cur_img] * n_patches
                    cur_img += 1
                else:
                    src.append(t); nl.append(l); im.append(-1)
        rows.append((src, nl, im))
    Tm = max(len(r[0]) for r in rows)
    src_t = torch.full((B, Tm), PAD, dtype=torch.int64)
    lab_t = torch.full((B, Tm), IGNORE_INDEX, dtype=torch.int64)
    msk_t = torch.zeros((B, Tm), dtype=torch.bool)
    pos_t = torch.zeros((B, Tm), dtype=torch.int64)
    img_t = torch.full((B, Tm), -1, dtype=torch.int64)
    for b, (src, nl, im) in enumerate(rows):
        n = len(src)
        if n == 0:
            continue
        sl = slice(Tm - n, Tm) if padding_side == "left" else slice(0, n)
        src_t[b, sl] = torch.tensor(src); lab_t[b, sl] = torch.tensor(nl)
        msk_t[b, sl] = True; pos_t[b, sl] = torch.arange(n); img_t[b, sl] = torch.tensor(im)
    return src_t, lab_t, msk_t, pos_t, img_t


def splice_embed(embed_w, image_features, src, img_index):
    """Float part of the splice: gather token embeddings / image feature rows, zero padding
    (llava_arch.py:256-274,295-320).  Differentiable w.r.t. ``image_features`` (projector grads)."""
    H = embed_w.shape[1]
    tok = src >= 0
    isimg = img_index >= 0
    e_tok = embed_w[src.clamp(min=0)] * tok[..., None].to(embed_w.dtype)
    flat = image_features.reshape(-1, H).to(embed_w.dtype)
    idx = (img_index.clamp(min=0) * image_features.shape[1] + (-1 - src).clamp(min=0, max=image_features.shape[1] - 1))
    e_img = flat[idx] * isimg[..., None].to(embed_w.dtype)
    return e_tok + e_img


# ----------------------------------------------------------------------------------------------
# full model forwards
# ----------------------------------------------------------------------------------------------
def lm_forward(sd, cfg: LMCfg, inputs_embeds, attention_mask, position_ids, moe_noise=None, record=None):
    """Qwen2Model.forward modeling_qwen2.py:963-1107 / MoEQwen1_5Model_forward llava_qwen1_5_moe.py:184-339
    with MoEQwen1_5DecoderLayer_forward :112-181.  Returns (final-normed hidden, [l_aux per MoE layer])."""
    B, T, _ = inputs_embeds.shape
    if position_ids is None:
        position_ids = torch.arange(T).unsqueeze(0)
    position_ids = position_ids.view(-1, T).long()
    cos, sin = rope_cache(cfg.head_dim, max(T, int(position_ids.max()) + 1), cfg.rope_theta, inputs_embeds.dtype)
    mask4d = sdpa_mask(attention_mask, B, T, inputs_embeds.dtype)
    h = inputs_embeds
    l_auxes = []
    for i in range(cfg.layers):
        p = f"{P_LM}layers.{i}."
        r = h
        x = rmsnorm(h, sd[p + "input_layernorm.weight"], cfg.eps)
        h = r + attention(sd, p + "self_attn.", cfg, x, mask4d, position_ids, cos, sin)
        r = h
        x = rmsnorm(h, sd[p + "post_attention_layernorm.weight"], cfg.eps)
        if i in cfg.moe_layers:
            noise = moe_noise[cfg.moe_layers.index(i)]
            y, l_aux, _ = moe_layer(sd, p + "mlp.deepspeed_moe.", cfg, x, noise, record)
            l_auxes.append(l_aux)
        else:
            y = mlp(sd, p + "mlp.", x)
        h = r + y
    return rmsnorm(h, sd[P_LM + "norm.weight"], cfg.eps), l_auxes


def shifted_ce(logits, labels, vocab):
    """modeling_qwen2.py:1196-1204 / llava_qwen1_5_moe.py:413-421"""
    sl = logits[..., :-1, :].contiguous().view(-1, vocab)
    tl = labels[..., 1:].contiguous().view(-1)
    return F.cross_entropy(sl, tl)


def llava_forward(sd, cfg: LMCfg, clip_cfg: ClipCfg, input_ids, attention_mask, labels, images,
                  moe_noise=None, record=None, padding_side="right"):
    """LlavaQwen1_5ForCausalLM.forward llava_qwen1_5.py:71-145 (dense) /
    LLaVAMoDQwen1_5ForCausalLM.forward llava_qwen1_5_moe.py:357-451 (MoE).
    ``images``: list of [3,S,S] tensors.  Returns dict(loss, moe_loss, logits fp32, labels, hidden)."""
    imgs = torch.stack(list(images))
    feats = encode_images(sd, clip_cfg, cfg.proj_depth, imgs)
    src, new_labels, new_mask, pos, img_index = splice_plan(input_ids, attention_mask, labels,
                                                             feats.shape[1], padding_side)
    embeds = splice_embed(sd[P_LM + "embed_tokens.weight"], feats, src, img_index)
    mask_for_lm = new_mask if attention_mask is not None else None
    hidden, l_auxes = lm_forward(sd, cfg, embeds, mask_for_lm, pos, moe_noise, record)
    w_head = sd[P_LM + "embed_tokens.weight"] if cfg.tie and "lm_head.weight" not in sd else sd["lm_head.weight"]
    logits = F.linear(hidden, w_head).float()
    loss = shifted_ce(logits, new_labels, cfg.vocab) if labels is not None else None
    moe_loss = None
    if len(l_auxes) > 0:
        moe_loss = cfg.aux_coef * sum(l_auxes)                 # llava_qwen1_5_moe.py:431
        if loss is not None:
            loss = loss + moe_loss                               # :434
    return dict(loss=loss, moe_loss=moe_loss, logits=logits, labels=new_labels, hidden=hidden,
                l_aux=l_auxes, attention_mask=new_mask)


# ----------------------------------------------------------------------------------------------
# trainers -- llavamod/train/align_trainer.py, dpo_trainer.py
# ----------------------------------------------------------------------------------------------
def get_p(logits, kd_vocab=KD_VOCAB):
    """AlignTrainer.get_p  align_trainer.py:473-475"""
    return F.softmax(logits[:, :, :kd_vocab], dim=-1, dtype=torch.float32)


def get_logp(logits, kd_vocab=KD_VOCAB):
    """AlignTrainer.get_logp  align_trainer.py:497-499"""
    return F.log_softmax(logits[:, :, :kd_vocab], dim=-1, dtype=torch.float32)


def compute_align_loss(policy_logprobs, reference_probs, labels, distill_all_tokens=False):
    """AlignTrainer.compute_align_loss  align_trainer.py:503-528 (un-shifted mask, 0/0 -> NaN kept)."""
    inf_mask = torch.isinf(policy_logprobs)
    prod = torch.masked_fill(reference_probs * policy_logprobs, inf_mask, 0)
    x = torch.sum(prod, dim=-1).view(-1)
    if distill_all_tokens:
        m = torch.ones_like(labels).int()
    else:
        m = (labels != IGNORE_INDEX).int()
    return -torch.sum(x * m.view(-1), dim=0) / torch.sum(m.view(-1), dim=0)


def mimic_compute_loss(student_out, teacher_logits, loss_type="kd_lm", moe_loss_enable=True,
                       distill_all_tokens=False, kd_vocab=KD_VOCAB):
    """AlignTrainer.compute_loss  align_trainer.py:530-594 given the two forwards' outputs.
    Keeps the double-counted moe_loss (:573-577 on top of llava_qwen1_5_moe.py:434) and the -1.0 sentinel."""
    ref_probs = get_p(teacher_logits.detach(), kd_vocab)
    logp = get_logp(student_out["logits"], kd_vocab)
    align = compute_align_loss(logp, ref_probs, student_out["labels"], distill_all_tokens)
    sft = student_out["loss"]
    losses = align if loss_type == "only_kd" else align + sft
    moe = student_out["moe_loss"] if moe_loss_enable else None
    if moe is not None and bool(moe):
        losses = losses + moe
        moe_metric = moe
    else:
        moe_metric = torch.full_like(align, -1.0)
    return losses.mean(), {"loss": losses.mean(), "loss/align": align.mean(),
                           "loss/moe_balance": moe_metric.mean(), "loss/lm": sft.mean()}


def dpo_get_logp(logits, labels, average_log_prob=False):
    """DPOTrainer.get_logp  dpo_trainer.py:483-495 (shift, no vocab slice, gather, masked sum)."""
    labels = labels[:, 1:].clone()
    logits = logits[:, :-1, :]
    m = labels != IGNORE_INDEX
    labels[labels == IGNORE_INDEX] = 0
    tok = torch.gather(logits.log_softmax(-1), dim=2, index=labels.unsqueeze(2)).squeeze(2)
    if average_log_prob:
        return (tok * m).sum(-1) / m.sum(-1)
    return (tok * m).sum(-1)


def dpo_loss(pc, pr, rc, rr, beta=0.1, loss_type="sigmoid", label_smoothing=0.0):
    """DPOTrainer.dpo_loss  dpo_trainer.py:497-562"""
    logits = (pc - pr) - (rc - rr)
    if loss_type == "sigmoid":
        losses = -F.logsigmoid(beta * logits) * (1 - label_smoothing) - F.logsigmoid(-beta * logits) * label_smoothing
    elif loss_type == "hinge":
        losses = torch.relu(1 - beta * logits)
    elif loss_type == "ipo":
        losses = (logits - 1 / (2 * beta)) ** 2
    elif loss_type == "kto_pair":
        chosen_KL = (pc - rc).mean().clamp(min=0)
        rejected_KL = (pr - rr).mean().clamp(min=0)
        losses = torch.cat((1 - torch.sigmoid(beta * ((pc - rc) - rejected_KL)),
                            1 - torch.sigmoid(beta * (chosen_KL - (pr - rr)))), 0)
    else:
        raise ValueError(f"Unknown loss type: {loss_type}. Should be one of ['sigmoid', 'hinge']")
    return losses, beta * (pc - rc).detach(), beta * (pr - rr).detach()


def dpo_compute_loss(pol_c, pol_r, ref_c_logits, ref_c_labels, ref_r_logits, ref_r_labels,
                     beta=0.1, loss_type="sigmoid", moe_loss_enable=True):
    """DPOTrainer.compute_loss  dpo_trainer.py:564-641 given the four forwards."""
    pc = dpo_get_logp(pol_c["logits"], pol_c["labels"])
    pr = dpo_get_logp(pol_r["logits"], pol_r["labels"])
    with torch.no_grad():
        rc = dpo_get_logp(ref_c_logits, ref_c_labels)
        rr = dpo_get_logp(ref_r_logits, ref_r_labels)
    reward_losses, cr, rj = dpo_loss(pc, pr, rc, rr, beta, loss_type)
    mc = pol_c["moe_loss"] if moe_loss_enable else None
    mr = pol_r["moe_loss"] if moe_loss_enable else None
    if mc is not None and mr is not None and bool(mc) and bool(mr):
        moe = mc + mr
        losses = reward_losses + moe
    else:
        moe = torch.full_like(reward_losses, -1.0)
        losses = reward_losses
    metrics = {"loss": losses.mean(), "loss/reward": reward_losses.mean(), "loss/moe_balance": moe.mean(),
               "loss/policy_chosen": pol_c["loss"].detach().mean(), "rewards/chosen": cr.mean(),
               "rewards/rejected": rj.mean(), "rewards/accuracies": (cr > rj).float().mean(),
               "rewards/margins": (cr - rj).mean(), "logps/chosen": pc.detach().mean(),
               "logps/rejected": pr.detach().mean()}
    return losses.mean(), metrics


# ----------------------------------------------------------------------------------------------
# optimizer + schedule (third-party HF Trainer 4.37 / torch.optim.AdamW; parity unpinned)
# ----------------------------------------------------------------------------------------------
def cosine_lr(step, total, base_lr, warmup_ratio=0.03):
    """transformers.get_cosine_schedule_with_warmup with warmup = ceil(ratio*total); ``step`` counts
    completed optimizer steps (LambdaLR semantics: lr used for step s is lambda(s))."""
    warm = math.ceil(warmup_ratio * total)
    if step < warm:
        return base_lr * step / max(1, warm)
    prog = (step - warm) / max(1, total - warm)
    return base_lr * max(0.0, 0.5 * (1.0 + math.cos(math.pi * prog)))


def adamw_step(params, grads, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0):
    """torch.optim.AdamW single step (fp32), step is 1-based."""
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    for p, g, mi, vi in zip(params, grads, m, v):
        p.mul_(1 - lr * wd)
        mi.mul_(beta1).add_(g, alpha=1 - beta1)
        vi.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        denom = (vi.sqrt() / math.sqrt(bc2)).add_(eps)
        p.addcdiv_(mi, denom, value=-lr / bc1)


def clip_grad_norm(grads, max_norm=1.0):
    """torch.nn.utils.clip_grad_norm_ (HF Trainer max_grad_norm=1.0 default)."""
    total = torch.sqrt(sum((g.float() ** 2).sum() for g in grads))
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in grads:
        g.mul_(coef)
    return total


# ----------------------------------------------------------------------------------------------
# random-init state dicts with the reference's key layout (SURVEY.md section 8b)
# ----------------------------------------------------------------------------------------------
def init_clip(cfg: ClipCfg, gen, std=0.02, dtype=torch.float32, pre=P_CLIP):
    def rn(*s): return (torch.randn(*s, generator=gen) * std).to(dtype)
    sd = {}
    n_pos = cfg.n_patches + 1
    sd[pre + "embeddings.class_embedding"] = rn(cfg.hidden)
    sd[pre + "embeddings.patch_embedding.weight"] = rn(cfg.hidden, 3, cfg.patch, cfg.patch)
    sd[pre + "embeddings.position_embedding.weight"] = rn(n_pos, cfg.hidden)
    for nm in ("pre_layrnorm", "post_layernorm"):
        sd[pre + nm + ".weight"] = torch.ones(cfg.hidden, dtype=dtype)
        sd[pre + nm + ".bias"] = torch.zeros(cfg.hidden, dtype=dtype)
    for i in range(cfg.layers):
        p = f"{pre}encoder.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{nm}.weight"] = rn(cfg.hidden, cfg.hidden)
            sd[p + f"self_attn.{nm}.bias"] = rn(cfg.hidden)
        for nm in ("layer_norm1", "layer_norm2"):
            sd[p + nm + ".weight"] = 1 + rn(cfg.hidden)
            sd[p + nm + ".bias"] = rn(cfg.hidden)
        sd[p + "mlp.fc1.weight"] = rn(cfg.inter, cfg.hidden); sd[p + "mlp.fc1.bias"] = rn(cfg.inter)
        sd[p + "mlp.fc2.weight"] = rn(cfg.hidden, cfg.inter); sd[p + "mlp.fc2.bias"] = rn(cfg.hidden)
    return sd


def init_lm(cfg: LMCfg, clip_hidden, gen, std=0.02, dtype=torch.float32):
    def rn(*s): return (torch.randn(*s, generator=gen) * std).to(dtype)
    sd = {}
    H, I, hd = cfg.hidden, cfg.inter, cfg.head_dim
    sd[P_LM + "embed_tokens.weight"] = rn(cfg.vocab, H)
    for i in range(cfg.layers):
        p = f"{P_LM}layers.{i}."
        sd[p + "self_attn.q_proj.weight"] = rn(cfg.heads * hd, H); sd[p + "self_attn.q_proj.bias"] = rn(cfg.heads * hd)
        sd[p + "self_attn.k_proj.weight"] = rn(cfg.kv_heads * hd, H); sd[p + "self_attn.k_proj.bias"] = rn(cfg.kv_heads * hd)
        sd[p + "self_attn.v_proj.weight"] = rn(cfg.kv_heads * hd, H); sd[p + "self_attn.v_proj.bias"] = rn(cfg.kv_heads * hd)
        sd[p + "self_attn.o_proj.weight"] = rn(H, cfg.heads * hd)
        sd[p + "input_layernorm.weight"] = 1 + rn(H)
        sd[p + "post_attention_layernorm.weight"] = 1 + rn(H)
        if i in cfg.moe_layers:
            # sparse up-cycling: every expert is a copy of the dense MLP (llava_qwen1_5_moe.py:534-550)
            g, u, d = rn(I, H), rn(I, H), rn(H, I)
            q = p + "mlp.deepspeed_moe."
            sd[q + "gate.wg.weight"] = (torch.randn(cfg.num_experts, H, generator=gen) * std).float()
            for e in range(cfg.num_experts):
                sd[q + f"experts.deepspeed_experts.{e}.gate_proj.weight"] = g.clone()
                sd[q + f"experts.deepspeed_experts.{e}.up_proj.weight"] = u.clone()
                sd[q + f"experts.deepspeed_experts.{e}.down_proj.weight"] = d.clone()
        else:
            sd[p + "mlp.gate_proj.weight"] = rn(I, H)
            sd[p + "mlp.up_proj.weight"] = rn(I, H)
            sd[p + "mlp.down_proj.weight"] = rn(H, I)
    sd[P_LM + "norm.weight"] = 1 + rn(H)
    sd["lm_head.weight"] = sd[P_LM + "embed_tokens.weight"] if cfg.tie else rn(cfg.vocab, H)
    sd[P_PROJ + "0.weight"] = rn(H, clip_hidden); sd[P_PROJ + "0.bias"] = rn(H)
    for j in range(1, cfg.proj_depth):
        sd[P_PROJ + f"{2 * j}.weight"] = rn(H, H); sd[P_PROJ + f"{2 * j}.bias"] = rn(H)
    return sd


def trainable_keys(sd, train_modules=("mlp.gate_proj", "mlp.up_proj", "mlp.down_proj", "wg")):
    """initialize_moe_modules freeze-by-substring llava_qwen1_5_moe.py:501-506 (applied BEFORE the MoE
    wrap, so expert copies inherit requires_grad from 'mlp.*_proj'; 'wg' is created trainable by
    DeepSpeed afterwards), then initialize_vision_modules re-enables mm_projector llava_arch.py:117-120."""
    keys = []
    for k in sd:
        if "image_tower" in k:
            continue
        pre_wrap = re.sub(r"deepspeed_moe\.experts\.deepspeed_experts\.\d+\.", "", k)
        if "mm_projector" in k or "gate.wg" in k or any(t in pre_wrap for t in train_modules):
            keys.append(k)
    return keys
