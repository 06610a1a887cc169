"""Qwen2 decoder engine for the H100 build (dense and DeepSpeed-style sparse-MoE layers).

Stands in for the reference's vendored ``qwen1_5/modeling_qwen2.py`` (RMSNorm :96-110, RoPE :114-184, MLP :188-200,
SDPA attention :644-728, decoder layer :738-812, model :932-1107) and the patched MoE forwards of
``llava_qwen1_5_moe.py:112-339``.  Parameter modules keep the reference's attribute / checkpoint key names;
the arithmetic is issued through ``llavamod.kernels`` (our CUDA: GEMM, attention, norms, RoPE, MoE, loss heads).

Layout decisions (GPU-first):
  * q|k|v and gate|up weights live in ONE fused buffer each (one GEMM instead of three / two); the per-projection
    ``nn.Parameter``s the reference exposes are views into it, so ``state_dict()`` keeps the reference layout;
  * the E experts of an MoE layer are one [E,2I,H] + one [E,H,I] buffer (batched / grouped GEMM operands);
  * residual adds are fused into the following RMSNorm kernel, RoPE runs in place on the fused QKV output,
    the MoE combine fuses the residual add, the lm_head feeds the fused KL/CE kernel without an fp32 copy.
"""
import json
import math
import os
from typing import List, Optional

import torch
import torch.nn as nn

from ... import kernels as K


# -------------------------------------------------------------------------------------------------
# configuration (HF config.json compatible; no transformers import on the hot path)
# -------------------------------------------------------------------------------------------------
class Qwen2Config:
    model_type = "qwen2"
    architectures_default: List[str] = ["Qwen2ForCausalLM"]

    def __init__(self, vocab_size=151936, hidden_size=4096, intermediate_size=22016, num_hidden_layers=32,
                 num_attention_heads=32, num_key_value_heads=None, hidden_act="silu", max_position_embeddings=32768,
                 initializer_range=0.02, rms_norm_eps=1e-6, use_cache=True, tie_word_embeddings=False,
                 rope_theta=10000.0, use_sliding_window=False, sliding_window=4096, max_window_layers=28,
                 attention_dropout=0.0, **kwargs):
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.intermediate_size = intermediate_size
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.num_key_value_heads = num_key_value_heads if num_key_value_heads is not None else num_attention_heads
        self.hidden_act = hidden_act
        self.max_position_embeddings = max_position_embeddings
        self.initializer_range = initializer_range
        self.rms_norm_eps = rms_norm_eps
        self.use_cache = use_cache
        self.tie_word_embeddings = tie_word_embeddings
        self.rope_theta = rope_theta
        self.use_sliding_window = use_sliding_window
        self.sliding_window = sliding_window
        self.max_window_layers = max_window_layers
        self.attention_dropout = attention_dropout
        kwargs.pop("model_type", None)
        for k, v in kwargs.items():
            setattr(self, k, v)

    def to_dict(self):
        d = {k: v for k, v in self.__dict__.items() if not k.startswith("_")}
        d["model_type"] = self.model_type
        d.setdefault("architectures", list(self.architectures_default))
        return d

    @classmethod
    def from_dict(cls, d):
        d = dict(d)
        return cls(**d)

    def save_pretrained(self, path):
        os.makedirs(path, exist_ok=True)
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump(self.to_dict(), f, indent=2, sort_keys=True, default=str)

    @classmethod
    def from_pretrained(cls, path, **kw):
        with open(os.path.join(path, "config.json")) as f:
            d = json.load(f)
        d.update(kw)
        return cls.from_dict(d)

    def __repr__(self):
        return "%s %s" % (type(self).__name__, json.dumps(self.to_dict(), indent=1, default=str))


# -------------------------------------------------------------------------------------------------
# parameter holders (attribute names == reference checkpoint keys)
# -------------------------------------------------------------------------------------------------
class ParamLinear(nn.Module):
    """Holds ``weight`` [out,in] (+ ``bias``) exactly like nn.Linear; may be a view into a fused buffer."""

    def __init__(self, weight, bias=None):
        super().__init__()
        self.weight = nn.Parameter(weight)
        self.bias = nn.Parameter(bias) if bias is not None else None

    @property
    def out_features(self):
        return self.weight.shape[0]

    @property
    def in_features(self):
        return self.weight.shape[1]


class ParamNorm(nn.Module):
    def __init__(self, weight, bias=None, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(weight)
        self.bias = nn.Parameter(bias) if bias is not None else None
        self.variance_epsilon = eps
        self.is_layernorm = bias is not None      # CLIP nn.LayerNorm (no weight decay in the reference's groups); Qwen2RMSNorm decays


def _new(shape, device, dtype, std=None, ones=False):
    t = torch.empty(shape, device=device, dtype=dtype)
    if ones:
        t.fill_(1.0)
    elif std is not None:
        t.normal_(0.0, std)
    return t


class Qwen2Attention(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        H, nh, nkv = cfg.hidden_size, cfg.num_attention_heads, cfg.num_key_value_heads
        hd = H // nh
        self.num_heads, self.num_key_value_heads, self.head_dim = nh, nkv, hd
        std = cfg.initializer_range
        self.qkv_weight = _new(((nh + 2 * nkv) * hd, H), device, dtype, std)       # fused storage (not a Parameter)
        self.qkv_bias = torch.zeros((nh + 2 * nkv) * hd, device=device, dtype=dtype)
        a, b = nh * hd, (nh + nkv) * hd
        self.q_proj = ParamLinear(self.qkv_weight[:a], self.qkv_bias[:a])
        self.k_proj = ParamLinear(self.qkv_weight[a:b], self.qkv_bias[a:b])
        self.v_proj = ParamLinear(self.qkv_weight[b:], self.qkv_bias[b:])
        self.o_proj = ParamLinear(_new((H, nh * hd), device, dtype, std))


class Qwen2MLP(nn.Module):
    """Dense SwiGLU MLP; gate|up fused as one [2I,H] buffer."""

    def __init__(self, cfg, device, dtype, gu=None, dn=None):
        super().__init__()
        H, I = cfg.hidden_size, cfg.intermediate_size
        std = cfg.initializer_range
        self.gu_weight = gu if gu is not None else _new((2 * I, H), device, dtype, std)
        self.gate_proj = ParamLinear(self.gu_weight[:I])
        self.up_proj = ParamLinear(self.gu_weight[I:])
        self.down_proj = ParamLinear(dn if dn is not None else _new((H, I), device, dtype, std))


class TopKGate(nn.Module):
    """deepspeed.moe.sharded_moe.TopKGate parameter holder: ``wg`` is kept in fp32 (Appendix A step 1)."""

    def __init__(self, H, E, device):
        super().__init__()
        w = torch.empty(E, H, device=device, dtype=torch.float32)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))          # torch.nn.Linear default init
        self.wg = ParamLinear(w)


class Experts(nn.Module):
    def __init__(self, cfg, E, device, dtype, src_mlp: Qwen2MLP):
        super().__init__()
        H, I = cfg.hidden_size, cfg.intermediate_size
        self.gu_weight = torch.empty(E, 2 * I, H, device=device, dtype=dtype)
        self.dn_weight = torch.empty(E, H, I, device=device, dtype=dtype)
        # sparse up-cycling: every expert starts as a copy of the dense MLP (llava_qwen1_5_moe.py:534-550)
        self.gu_weight.copy_(src_mlp.gu_weight.detach()[None].expand(E, -1, -1))
        self.dn_weight.copy_(src_mlp.down_proj.weight.detach()[None].expand(E, -1, -1))
        self.deepspeed_experts = nn.ModuleList(
            [Qwen2MLP(cfg, device, dtype, gu=self.gu_weight[e], dn=self.dn_weight[e]) for e in range(E)])
        rg = src_mlp.gate_proj.weight.requires_grad, src_mlp.up_proj.weight.requires_grad, src_mlp.down_proj.weight.requires_grad
        for m in self.deepspeed_experts:                       # deep copies inherit requires_grad
            m.gate_proj.weight.requires_grad = rg[0]
            m.up_proj.weight.requires_grad = rg[1]
            m.down_proj.weight.requires_grad = rg[2]


class MOELayer(nn.Module):
    def __init__(self, cfg, E, device, dtype, src_mlp):
        super().__init__()
        self.gate = TopKGate(cfg.hidden_size, E, device)
        self.experts = Experts(cfg, E, device, dtype, src_mlp)


class MoE(nn.Module):
    """Parameter layout of deepspeed.moe.layer.MoE (call site llava_qwen1_5_moe.py:536-546): ``deepspeed_moe.gate.wg``
    and ``deepspeed_moe.experts.deepspeed_experts.{e}``.  k = 2 (top2gating, the distillation shells' default) or k = 1 (top1gating
    with random token selection), the two widths DeepSpeed's TopKGate accepts.
    use_residual=True (Residual-MoE): ``mlp`` is the dense module passed in (the very object, not a copy) and ``coefficient`` a bf16
    Linear(H, 2) with a bias; the layer returns bf16(moe*c0) + bf16(mlp*c1), c = softmax(coefficient(x)) (SURVEY.md Appendix A)."""

    def __init__(self, cfg, expert: Qwen2MLP, num_experts=4, ep_size=1, k=2, capacity_factor=1.0,
                 eval_capacity_factor=1.0, min_capacity=4, use_residual=False):
        super().__init__()
        if k not in (1, 2):
            raise ValueError("Only top-1 and top-2 gatings are supported (got k = %r)" % (k,))
        if ep_size != 1:
            raise NotImplementedError("expert parallelism is size 1 in the reference's recipes (SURVEY.md 2.3)")
        dev, dt = expert.down_proj.weight.device, expert.down_proj.weight.dtype
        self.num_experts, self.k = num_experts, k
        self.capacity_factor, self.eval_capacity_factor, self.min_capacity = capacity_factor, eval_capacity_factor, min_capacity
        self.use_residual = bool(use_residual)
        self.deepspeed_moe = MOELayer(cfg, num_experts, dev, dt, expert)
        if self.use_residual:
            # module order = DeepSpeed's (deepspeed_moe, mlp, coefficient), hence the state-dict order; nn.Linear's default init drawn
            # in fp32 and cast, as the bf16 engine cast leaves the coefficient bf16
            H = cfg.hidden_size
            self.mlp = expert
            w = torch.empty(2, H, device=dev, dtype=torch.float32)
            nn.init.kaiming_uniform_(w, a=math.sqrt(5))
            b = torch.empty(2, device=dev, dtype=torch.float32).uniform_(-1.0 / math.sqrt(H), 1.0 / math.sqrt(H))
            self.coefficient = ParamLinear(w.to(dt), b.to(dt))

    def trainable(self):
        """Whether any parameter of the layer trains (the routed path's test, plus the dense MLP and coefficient of a residual layer)."""
        ds = self.deepspeed_moe
        if ds.gate.wg.weight.requires_grad or ds.experts.deepspeed_experts[0].down_proj.weight.requires_grad:
            return True
        if not self.use_residual:
            return False
        return any(p.requires_grad for p in (self.mlp.gate_proj.weight, self.mlp.up_proj.weight, self.mlp.down_proj.weight,
                                             self.coefficient.weight, self.coefficient.bias))

    def run(self, x, stream, noise, cf, gview):
        """The layer on post-norm x [S,H] with the residual stream: -> (new stream, l_aux, routing record or None).  Autograd path when
        anything is differentiated (gradients go to the arena views gview returns), the no-grad path otherwise."""
        ds = self.deepspeed_moe
        wg, gu, dn = ds.gate.wg.weight, ds.experts.gu_weight, ds.experts.dn_weight
        grad = torch.is_grad_enabled() and (x.requires_grad or self.trainable())
        if not self.use_residual:
            if grad:
                grads = dict(wg=gview(wg), w_gu=gview(gu), w_dn=gview(dn))
                return K.MoEFn.apply(x, stream, wg, gu, dn, noise, cf, self.min_capacity, grads, self.k) + (None,)
            return K.moe_forward_nograd(x, stream, wg, gu, dn, noise, cf, self.min_capacity, self.k)
        rm, cw = self.mlp, self.coefficient
        if grad:
            grads = dict(wg=gview(wg), w_gu=gview(gu), w_dn=gview(dn), r_gu=gview(rm.gu_weight), r_dn=gview(rm.down_proj.weight),
                         wc=gview(cw.weight), bc=gview(cw.bias))
            return K.ResidualMoEFn.apply(x, stream, wg, gu, dn, noise, cf, self.min_capacity, rm.gu_weight, rm.down_proj.weight,
                                         cw.weight, cw.bias, grads, self.k) + (None,)
        return K.moe_residual_forward_nograd(x, stream, wg, gu, dn, noise, cf, self.min_capacity, rm.gu_weight, rm.down_proj.weight,
                                             cw.weight, cw.bias, self.k)


class Qwen2DecoderLayer(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        H = cfg.hidden_size
        self.self_attn = Qwen2Attention(cfg, device, dtype)
        self.mlp = Qwen2MLP(cfg, device, dtype)
        self.input_layernorm = ParamNorm(_new((H,), device, dtype, ones=True), eps=cfg.rms_norm_eps)
        self.post_attention_layernorm = ParamNorm(_new((H,), device, dtype, ones=True), eps=cfg.rms_norm_eps)


class ParamEmbedding(nn.Module):
    def __init__(self, weight):
        super().__init__()
        self.weight = nn.Parameter(weight)


def rope_tables(head_dim, max_pos, theta, dtype, device):
    """Qwen2RotaryEmbedding._set_cos_sin_cache (modeling_qwen2.py:127-136): built in fp32 on the host exactly as the
    reference does at construction, cast to the activation dtype, then moved to the device."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2).float() / head_dim))
    t = torch.arange(max_pos, dtype=inv_freq.dtype)
    freqs = torch.outer(t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(dtype).to(device).contiguous(), emb.sin().to(dtype).to(device).contiguous()


class Qwen2Model(nn.Module):
    """embed_tokens + layers + norm.  ``forward`` takes ``inputs_embeds`` (the LLaVA wrappers always splice first)."""

    def __init__(self, cfg, device="cuda", dtype=torch.bfloat16):
        super().__init__()
        self.config = cfg
        std = cfg.initializer_range
        self.embed_tokens = ParamEmbedding(_new((cfg.vocab_size, cfg.hidden_size), device, dtype, std))
        self.layers = nn.ModuleList([Qwen2DecoderLayer(cfg, device, dtype) for _ in range(cfg.num_hidden_layers)])
        self.norm = ParamNorm(_new((cfg.hidden_size,), device, dtype, ones=True), eps=cfg.rms_norm_eps)
        self._rope = None
        self.grad_views = {}          # id(storage tensor) -> grad view (set by TrainState)
        self.gradient_checkpointing = False

    # -- helpers -------------------------------------------------------------------------------------
    def rope(self, need, device, dtype):
        if self._rope is None or self._rope[0].shape[0] < need or self._rope[0].device != torch.device(device):
            n = max(need, min(self.config.max_position_embeddings, 8192))
            hd = self.config.hidden_size // self.config.num_attention_heads
            self._rope = rope_tables(hd, n, self.config.rope_theta, dtype, device)
        return self._rope

    def gview(self, t):
        return self.grad_views.get(id(t))

    def quantize_fp8_(self):
        """Turn the decoder linears of every (dense, frozen) layer into e4m3 weights with one fp32 scale per output channel
        (K.quant_rows on the device; the fused q|k|v and gate|up buffers as the single buffers they are) and release the bf16 copies:
        ``qkv_weight`` / ``gu_weight`` become K.Fp8Rows, o_proj / down_proj are held as ``o_fp8`` / ``down_fp8``, and the per-projection
        ``weight`` Parameters are gone.  Biases, norms, embeddings stay bf16.  The callers (quantize_fp8_ of the causal-LM classes) have
        checked that nothing here trains."""
        for layer in self.layers:
            at, mlp = layer.self_attn, layer.mlp
            at.o_fp8, mlp.down_fp8 = K.quant_rows(at.o_proj.weight.detach()), K.quant_rows(mlp.down_proj.weight.detach())
            at.qkv_weight, mlp.gu_weight = K.quant_rows(at.qkv_weight), K.quant_rows(mlp.gu_weight)
            for lin in (at.q_proj, at.k_proj, at.v_proj, at.o_proj, mlp.gate_proj, mlp.up_proj, mlp.down_proj):
                lin.weight = None

    # -- forward -------------------------------------------------------------------------------------
    def forward(self, inputs_embeds, attention_mask=None, position_ids=None, moe_noise=None, training_moe=True, cache=None):
        """inputs_embeds [B,T,H] bf16; attention_mask [B,T] bool or None; position_ids [B,T] int64 or None.
        cache: a KVCache.  Empty: the prefill -- this forward, plus the K / V of every layer appended to the cache.  Holding a prefix: one
        cached step of T tokens per sequence at positions len .. len + T - 1 (modeling_qwen2.py:652-728 with past_key_value), attention
        over the cached keys; T > 1 for dense models only.
        A padded prefill (attention_mask with zeros; real tokens contiguous, either side) is this same padded forward, with positions
        0 .. n_b - 1 over sequence b's real rows when position_ids is None; only the real rows go to the cache, packed at [0, n_b).
        Returns (final-normed hidden [B,T,H], [l_aux per MoE layer], routing records)."""
        if cache is not None and cache.length > 0:
            return self._decode_step(inputs_embeds, moe_noise, training_moe, cache)
        B, T, H = inputs_embeds.shape
        dev = inputs_embeds.device
        padded = attention_mask is not None and not bool(attention_mask.all())      # MaskInfo answers on the host (no sync)
        host_lengths = getattr(attention_mask, "lengths", None)
        if hasattr(attention_mask, "mask"):
            attention_mask = attention_mask.mask
        pad = K.pad_ranges(attention_mask) if padded else None       # per-row real key range; the attention kernels mask from it
        ragged = cache is not None and padded
        if ragged:
            lengths = host_lengths
            if lengths is None:          # a raw mask: its real tokens must be one run per row, which is what pad_ranges assumes
                span, real = torch.stack([pad[1] - pad[0], attention_mask.to(torch.int32).sum(1, dtype=torch.int32)]).tolist()
                if span != real:
                    raise ValueError("KV-cache prefill: every row's real tokens must be contiguous (left or right padding)")
                lengths = span
            lengths = [int(n) for n in lengths]
            if min(lengths) <= 0:
                raise ValueError("KV-cache prefill: sequence %d has no real token" % lengths.index(min(lengths)))
            cache.check(B, lengths)
            if position_ids is None:                        # compact positions (the splice plan gives them for spliced prompts)
                m = attention_mask.to(torch.int64)
                position_ids = (m.cumsum(1) - 1) * m
        elif cache is not None:
            cache.check(B, T)
        if position_ids is None:
            position_ids = torch.arange(T, device=dev, dtype=torch.int64).unsqueeze(0).expand(B, T)
        pos = position_ids.reshape(-1).to(torch.int64).contiguous()
        cos, sin = self.rope(T, dev, inputs_embeds.dtype)
        if moe_noise is None:
            # DeepSpeed draws fresh Gumbel noise (top-2) or uniforms (top-1's token selection) in every MoE layer; one draw for all layers
            # of this forward is the same distribution with 5 launches instead of 5 per layer
            moes = [l.mlp for l in self.layers if isinstance(l.mlp, MoE)]
            if moes and len({(m.num_experts, m.k) for m in moes}) == 1:
                moe_noise = moe_draw((len(moes), B * T, moes[0].num_experts), moes[0].k, dev).unbind(0)

        def attend(li, qkv, nh, nkv, hd):
            if ragged:
                K.kv_append_rows(qkv, B, T, nh, nkv, hd, cache.k[li], cache.v[li], pad[0], pad[1], cache.prefix_len)
            elif cache is not None:
                K.kv_append(qkv, B, T, nh, nkv, hd, cache.k[li], cache.v[li], cache.prefix_len)
            return K.attention(qkv, B, T, nh, nkv, hd, True, None, pad)

        checkpoint = cache is None and self.gradient_checkpointing and self.training and torch.is_grad_enabled()
        out, l_auxes, records = self._layers(inputs_embeds.reshape(B * T, H), cos, sin, pos, attend, moe_noise, training_moe, checkpoint)
        if ragged:
            cache.prefilled(pad[1] - pad[0], lengths)
        elif cache is not None:
            cache.prefilled(T, T)
        return out.view(B, T, H), l_auxes, records

    @torch.no_grad()
    def _decode_step(self, inputs_embeds, moe_noise, training_moe, cache):
        """One cached step: each sequence's new token sits at position len[b] (the reference's rule for a cached step,
        llava_arch.py:162-172, on unpadded prompts; for a padded prompt len[b] = n_b + s counts its real rows only), its k / v are appended
        at row len[b], and its query attends to rows [0, len[b] + 1).
        T > 1 tokens per sequence (the verify step of assisted decoding): token t sits at position len[b] + t, the T rows are appended at
        once and token t attends to rows [0, len[b] + t + 1) (lmod_attn_decode_chunk).  Every kernel of the step works row by row, and
        the chunked attention gives each row the bytes of the single-query kernel, so for a dense model this is T one-token steps, bit for
        bit.
        Everything the step reads about the position is on the device, so the step can be captured once and replayed.  MoE layers route
        the B new tokens alone (top2gating / top1gating with S = B, as MoEQwen1_5Model_forward does with a cache,
        llava_qwen1_5_moe.py:223-236).
        The step builds no autograd graph, whatever the caller's grad mode: decode attention has no backward, and the cached path is for
        decoding (it takes no labels)."""
        B, T, H = inputs_embeds.shape
        if T != 1 and any(isinstance(l.mlp, MoE) for l in self.layers):
            raise NotImplementedError("a cached step of the sparse model decodes one token per sequence (got %d): a step of T tokens would "
                                      "route its B*T tokens together (top2gating with S = B*T), which is not what T one-token steps "
                                      "compute" % T)
        if T != 1 and cache.shared:
            raise NotImplementedError("a shared KVCache decodes one token per sequence (got %d)" % T)
        cache.check(B, T)
        dev = inputs_embeds.device
        cos, sin = cache.rope
        torch.add(cache.len, T, out=cache.end)
        if cache.shared:
            torch.sub(cache.len, cache.prefix_rows, out=cache.suffix_len)
        if T == 1:
            pos = cache.pos
            pos.copy_(cache.len)
        else:
            pos = (cache.len.to(torch.int64)[:, None] + torch.arange(T, device=dev, dtype=torch.int64)[None, :]).reshape(B * T)
            ws = cache.chunk_workspace(T)

        def attend(li, qkv, nh, nkv, hd):
            if cache.shared:                            # the new row goes to the copy's suffix; the prompt's rows are read once per CTA
                K.kv_append(qkv, B, 1, nh, nkv, hd, cache.ks[li], cache.vs[li], cache.suffix_len)
                return K.attn_decode_shared(qkv, cache.share, nh, nkv, hd, cache.k[li], cache.v[li], cache.prefix_len, cache.ks[li],
                                            cache.vs[li], cache.end, cache.max_len, cache.ws)[0]
            K.kv_append(qkv, B, T, nh, nkv, hd, cache.k[li], cache.v[li], cache.len)
            if T == 1:
                return K.attn_decode(qkv, nh, nkv, hd, cache.k[li], cache.v[li], cache.end, cache.ws)[0]
            return K.attn_decode_chunk(qkv, B, T, nh, nkv, hd, cache.k[li], cache.v[li], cache.end, ws)[0]

        out, l_auxes, records = self._layers(inputs_embeds.reshape(B * T, H), cos, sin, pos, attend, moe_noise, training_moe)
        cache.len.copy_(cache.end)
        cache.advance(T)
        return out.view(B, T, H), l_auxes, records

    def _layers(self, stream, cos, sin, pos, attend, moe_noise, training_moe, checkpoint=False):
        """The decoder layers and the final norm on the residual stream [S,H]: -> (final-normed hidden [S,H], [l_aux per MoE layer],
        routing records).  attend(li, qkv, nh, nkv, hd) -> attn is layer li's attention on its RoPE'd q|k|v rows, the one part in which
        forward and the cached step differ.  moe_noise: one tensor per MoE layer, or None to draw each layer's noise for its S tokens.
        checkpoint: every layer with something to differentiate runs as one checkpointed segment (K.checkpoint): its activations are
        recomputed in the backward instead of kept."""
        eps = self.config.rms_norm_eps
        branch = None                                   # pending residual-branch output (added inside the next norm)
        l_auxes, records = [], []
        moe_i = 0
        for li, layer in enumerate(self.layers):
            mlp = layer.mlp
            noise = None
            if isinstance(mlp, MoE):
                # drawn before the layer runs, so a checkpointed layer's recompute routes with the noise of its first forward
                noise = moe_noise[moe_i] if moe_noise is not None else moe_draw((stream.shape[0], mlp.num_experts), mlp.k, stream.device)
                moe_i += 1
            inputs = (stream,) if branch is None else (branch, stream)
            if checkpoint and (any(t.requires_grad for t in inputs) or any(p.requires_grad for p in layer.parameters())):
                def run(*xs, li=li, layer=layer, noise=noise):
                    return self._layer(li, layer, xs, cos, sin, pos, attend, noise, training_moe)[:2]
                branch_or_stream, out = K.checkpoint(run, *inputs)
                rec = None
            else:
                branch_or_stream, out, rec = self._layer(li, layer, inputs, cos, sin, pos, attend, noise, training_moe)
            if not isinstance(mlp, MoE):
                branch, stream = branch_or_stream, out
            else:
                branch, stream = None, branch_or_stream
                l_auxes.append(out)
                if rec is not None:
                    records.append(rec)
        x, res = (stream, None) if branch is None else (branch, stream)
        out, _ = K.rmsnorm(x, self.norm.weight, eps, res=res, wgrad=self.gview(self.norm.weight))
        return out, l_auxes, records

    def _layer(self, li, layer, inputs, cos, sin, pos, attend, noise, training_moe):
        """Decoder layer li on its inputs: (stream,) or (pending branch, stream) -> (branch, stream, None) for a dense layer, (stream, l_aux,
        routing record or None) for an MoE layer.  noise: the MoE layer's router noise."""
        eps = self.config.rms_norm_eps
        at = layer.self_attn
        nh, nkv, hd = at.num_heads, at.num_key_value_heads, at.head_dim
        fp8 = isinstance(at.qkv_weight, K.Fp8Rows)      # a layer of quantize_fp8_: the norms hand e4m3 rows to e4m3 projections
        x, res = inputs if len(inputs) == 2 else (inputs[0], None)
        if fp8:
            x, stream = K.rmsnorm_quant(x, layer.input_layernorm.weight, eps, res=res)
            qkv = K.qkv_rope_fp8(x, at.qkv_weight, at.qkv_bias, cos, sin, pos, nh, nkv, hd)
        else:
            x, stream = K.rmsnorm(x, layer.input_layernorm.weight, eps, res=res, wgrad=self.gview(layer.input_layernorm.weight))
            qkv = K.qkv_rope(x, at.qkv_weight, at.qkv_bias, cos, sin, pos, nh, nkv, hd, self.gview(at.qkv_weight), self.gview(at.qkv_bias))
        attn = attend(li, qkv, nh, nkv, hd)
        if fp8:
            branch = K.linear_fp8(attn, at.o_fp8)
            x, stream = K.rmsnorm_quant(branch, layer.post_attention_layernorm.weight, eps, res=stream)
        else:
            branch = K.linear(attn, at.o_proj.weight, None, self.gview(at.o_proj.weight), None)
            x, stream = K.rmsnorm(branch, layer.post_attention_layernorm.weight, eps, res=stream,
                                  wgrad=self.gview(layer.post_attention_layernorm.weight))
        mlp = layer.mlp
        if isinstance(mlp, MoE):
            cf = mlp.capacity_factor if training_moe else mlp.eval_capacity_factor
            return mlp.run(x, stream, noise, cf, self.gview)
        if fp8:
            return K.mlp_fp8(x, mlp.gu_weight, mlp.down_fp8), stream, None
        return K.mlp(x, mlp.gu_weight, mlp.down_proj.weight, self.gview(mlp.gu_weight), self.gview(mlp.down_proj.weight)), stream, None


class KVCache:
    """Decoding cache of a Qwen2Model for B sequences of up to max_len positions each.

    Per layer one K and one V buffer [B, nkv, max_len, hp] bf16 (HF's legacy layout; hp = the head width the attention kernels run,
    head dims below 64 zero-padded), the valid length of every sequence on the device (``len`` int32 [B], which the kernels read, so a
    captured decode step serves every position and every mix of lengths) and its host mirror ``lengths`` (``length`` is their maximum):
    the host always knows how many rows a forward adds, so every append is bounds-checked without a sync.  Sequence b holds its rows
    packed at [0, lengths[b]), whatever padding its prompt had.  ``cache[i]`` gives layer i's (k, v) views [B, nkv, length, hd], the legacy
    tuple layout llava_arch.py:165 indexes; rows at or past a sequence's own length are unspecified.  The RoPE tables cover max_len at
    allocation, so nothing is rebuilt inside a captured step.

    Shared form (share = n > 1, generate's num_return_sequences on a dense model): `batch` prompts, each decoded as n sequences (row b*n + j
    is copy j of prompt b; ``batch``, ``len`` and ``lengths`` count the B*n rows).  The prefill writes each prompt's rows once into ``k`` / ``v``
    [B, nkv, max_len, hp] (``prefix_len`` int32 [B] on the device, ``prefixes`` its host mirror); each copy's later rows go to its own
    ``ks`` / ``vs`` [B*n, nkv, suffix, hp], suffix row i - prefix_len[b] for key i, and the cached step attends with
    lmod_attn_decode_shared.  max_len bounds every row's total length and sets the attention splits, so each row's attention has the bytes
    of a plain cache of max_len rows.  It has no legacy tuple view: ``cache[i]`` raises, and forward(past_key_values=...) takes the plain
    form only."""

    def __init__(self, model, batch, max_len, share=1, suffix=None):
        cfg = model.config
        w = model.embed_tokens.weight
        dev, dt = w.device, w.dtype
        nh, nkv = cfg.num_attention_heads, cfg.num_key_value_heads
        self.head_dim = cfg.hidden_size // nh
        hp = K.attn_head_dim(self.head_dim)
        self.share, self.prompts = int(share), int(batch)
        if self.share < 1:
            raise ValueError("KVCache: share must be >= 1, got %r" % (share,))
        self.batch, self.max_len = int(batch) * self.share, int(max_len)
        self.k = [torch.empty(batch, nkv, max_len, hp, device=dev, dtype=dt) for _ in model.layers]
        self.v = [torch.empty(batch, nkv, max_len, hp, device=dev, dtype=dt) for _ in model.layers]
        self.len = torch.zeros(self.batch, dtype=torch.int32, device=dev)
        self.end = torch.zeros(self.batch, dtype=torch.int32, device=dev)     # len + 1 during a decode step
        self.pos = torch.zeros(self.batch, dtype=torch.int64, device=dev)     # RoPE positions of a decode step
        if self.share > 1:
            self.suffix = int(suffix) if suffix is not None else self.max_len
            self.ks = [torch.empty(self.batch, nkv, self.suffix, hp, device=dev, dtype=dt) for _ in model.layers]
            self.vs = [torch.empty(self.batch, nkv, self.suffix, hp, device=dev, dtype=dt) for _ in model.layers]
            self.prefix_len = torch.zeros(batch, dtype=torch.int32, device=dev)
            self.prefix_rows = torch.zeros(self.batch, dtype=torch.int32, device=dev)     # prefix_len of every row
            self.suffix_len = torch.zeros(self.batch, dtype=torch.int32, device=dev)      # len - prefix_len: a step's suffix append row
            self.ws = torch.empty(max(1, K.attn_decode_shared_ws_elems(batch, self.share, nh, nkv, self.head_dim, max_len)),
                                  dtype=torch.float32, device=dev)
        else:
            self.prefix_len = self.len                                        # the prefill appends at len
            self.ws = torch.empty(max(1, K.attn_decode_ws_elems(batch, nh, nkv, self.head_dim, max_len)), dtype=torch.float32, device=dev)
        self._chunk_ws = {}                                                   # T -> workspace of a T-token step
        self._shape = (nh, nkv)
        self.rope = model.rope(max_len, dev, dt)
        self.lengths = [0] * self.batch
        self.prefixes = [0] * self.prompts

    @property
    def shared(self):
        return self.share > 1

    @property
    def length(self):
        return max(self.lengths)

    @property
    def nbytes(self):
        """Bytes of the K / V buffers."""
        bufs = self.k + self.v + (self.ks + self.vs if self.shared else [])
        return sum(t.numel() * t.element_size() for t in bufs)

    def _per_seq(self, n_new, rows=None):
        rows = self.batch if rows is None else rows
        return [int(n) for n in n_new] if isinstance(n_new, (list, tuple)) else [int(n_new)] * rows

    def check(self, batch, n_new):
        """n_new: positions each sequence adds (an int for all, or one per sequence).  The prefill of a shared cache (empty) takes one row
        per prompt."""
        if self.shared and self.length == 0:
            if batch != self.prompts:
                raise ValueError("shared KVCache holds %d prompts, got a prefill of %d" % (self.prompts, batch))
            for b, a in enumerate(self._per_seq(n_new, self.prompts)):
                if a > self.max_len:
                    raise ValueError("KVCache is full: prompt %d has %d positions > max_len %d" % (b, a, self.max_len))
            return
        if batch != self.batch:
            raise ValueError("KVCache holds %d sequences, got a batch of %d" % (self.batch, batch))
        for b, (n, a) in enumerate(zip(self.lengths, self._per_seq(n_new))):
            if n + a > self.max_len:
                raise ValueError("KVCache is full: sequence %d has %d cached + %d new positions > max_len %d" % (b, n, a, self.max_len))
            if self.shared and n + a - self.prefixes[b // self.share] > self.suffix:
                raise ValueError("shared KVCache is full: sequence %d has %d rows past its prompt + %d new > suffix %d"
                                 % (b, n - self.prefixes[b // self.share], a, self.suffix))

    def prefilled(self, n_dev, n_new):
        """After the prefill appended n_dev (int32 [prompts] on the device, or an int) rows per prompt at prefix_len; n_new: the same on the
        host (an int for all, or one per prompt).  A shared cache hands every copy its prompt's length."""
        self.prefix_len.add_(n_dev)
        if not self.shared:
            self.advance(n_new)
            return
        self.prefixes = self._per_seq(n_new, self.prompts)
        self.prefix_rows.copy_(self.prefix_len.repeat_interleave(self.share))
        self.len.copy_(self.prefix_rows)
        self.advance([n for n in self.prefixes for _ in range(self.share)])

    def advance(self, n_new):
        self.lengths = [n + a for n, a in zip(self.lengths, self._per_seq(n_new))]

    def reset(self):
        self.len.zero_()
        self.lengths = [0] * self.batch
        if self.shared:
            self.prefix_len.zero_()
            self.prefixes = [0] * self.prompts

    def rollback(self, n_drop):
        """Forget the last n_drop[b] rows of every sequence (an int for all, or one per sequence) in the host mirror ``lengths``; the caller
        has applied the same rollback to the device ``len`` (lmod_spec_accept does it on the device)."""
        if self.shared:
            raise NotImplementedError("a shared KVCache is not rolled back (assisted decoding takes num_return_sequences = 1)")
        drop = self._per_seq(n_drop)
        if any(d < 0 or d > n for d, n in zip(drop, self.lengths)):
            raise ValueError("KVCache.rollback: cannot drop %s rows from lengths %s" % (drop, self.lengths))
        self.lengths = [n - d for n, d in zip(self.lengths, drop)]

    def reorder_beams(self, parent, n):
        """Beam search's cache reorder (HF _reorder_cache), in place by lmod_kv_beam_reorder: sequence b*n + j takes the rows of sequence
        b*n + parent[b*n + j] (host ints in [0, n)).  The beams of a prompt advance together, so they hold the same number of rows.  A
        shared cache (share == n) moves the rows past the prompt only; a plain cache of prompts*n sequences moves every row."""
        if self.shared and n != self.share:
            raise ValueError("KVCache.reorder_beams: a shared cache of %d sequences per prompt, got n = %d" % (self.share, n))
        if self.batch % n:
            raise ValueError("KVCache.reorder_beams: %d sequences are not prompts of %d beams" % (self.batch, n))
        rows = []
        for b in range(self.batch // n):
            r = set(self.lengths[b * n:(b + 1) * n])
            if len(r) != 1:
                raise ValueError("KVCache.reorder_beams: the beams of prompt %d have lengths %s" % (b, self.lengths[b * n:(b + 1) * n]))
            rows.append(r.pop() - (self.prefixes[b] if self.shared else 0))
        if any(rows):
            K.kv_beam_reorder(self.ks + self.vs if self.shared else self.k + self.v, n, self.head_dim, rows, parent)

    def chunk_workspace(self, T):
        """The decode-attention workspace of a step of T tokens per sequence (kept, so a captured step keeps its address)."""
        ws = self._chunk_ws.get(T)
        if ws is None:
            nh, nkv = self._shape
            n = K.attn_decode_chunk_ws_elems(self.batch, T, nh, nkv, self.head_dim, self.max_len)
            ws = self._chunk_ws[T] = torch.empty(max(1, n), dtype=torch.float32, device=self.len.device)
        return ws

    def get_seq_length(self, layer_idx=0):
        return self.length

    def __len__(self):
        return len(self.k)

    def __getitem__(self, i):
        if self.shared:
            raise TypeError("a shared KVCache has no [B, nkv, length, hd] view: its copies keep their prompt's rows once")
        n, hd = self.length, self.head_dim
        return self.k[i][:, :, :n, :hd], self.v[i][:, :, :n, :hd]


def gumbel_noise(shape, device):
    """deepspeed gumbel_rsample (Gumbel(0,1) via -log(-log U)); Philox stream of the current device generator."""
    u = torch.rand(shape, device=device, dtype=torch.float32).clamp_(min=1e-20, max=1.0 - 1e-7)
    return -torch.log(-torch.log(u))


def moe_draw(shape, k, device):
    """The random input of a k-wide MoE layer: Gumbel noise for top-2's second choice, Uniform(0, 1) for top-1's random token selection
    (top1gating draws it on every call, training and eval alike)."""
    if k == 1:
        return torch.rand(shape, device=device, dtype=torch.float32)
    return gumbel_noise(shape, device)
