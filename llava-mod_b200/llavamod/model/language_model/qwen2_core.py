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
    and ``deepspeed_moe.experts.deepspeed_experts.{e}``.  k=2 only (the distillation shells use top-2)."""

    def __init__(self, cfg, expert: Qwen2MLP, num_experts=4, ep_size=1, k=2, capacity_factor=1.0,
                 eval_capacity_factor=1.0, min_capacity=4, use_residual=False):
        super().__init__()
        if k != 2:
            raise NotImplementedError("only top-2 gating is built (the reference's distillation recipes use --top_k_experts 2)")
        if ep_size != 1:
            raise NotImplementedError("expert parallelism is size 1 in the reference's recipes (SURVEY.md 2.3)")
        if use_residual:
            raise NotImplementedError("use_residual=True (Residual-MoE) is not on the hot path")
        dev, dt = expert.down_proj.weight.device, expert.down_proj.weight.dtype
        self.num_experts, self.k = num_experts, k
        self.capacity_factor, self.eval_capacity_factor, self.min_capacity = capacity_factor, eval_capacity_factor, min_capacity
        self.deepspeed_moe = MOELayer(cfg, num_experts, dev, dt, expert)


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

    # -- forward -------------------------------------------------------------------------------------
    def forward(self, inputs_embeds, attention_mask=None, position_ids=None, moe_noise=None, training_moe=True, cache=None):
        """inputs_embeds [B,T,H] bf16; attention_mask [B,T] bool or None; position_ids [B,T] int64 or None.
        cache: a KVCache.  Empty: the prefill -- this forward, plus the K / V of every layer appended to the cache.  Holding a prefix and
        T == 1: one decode step at position len (modeling_qwen2.py:652-728 with past_key_value), attention over the cached keys.
        Returns (final-normed hidden [B,T,H], [l_aux per MoE layer], routing records)."""
        if cache is not None and cache.length > 0:
            return self._decode_step(inputs_embeds, moe_noise, training_moe, cache)
        cfg = self.config
        B, T, H = inputs_embeds.shape
        dev = inputs_embeds.device
        if cache is not None:
            if attention_mask is not None and not bool(attention_mask.all()):
                raise NotImplementedError("KV-cache prefill of padded prompts: decode equal-length, unpadded prompts")
            cache.check(B, T)
        if position_ids is None:
            position_ids = torch.arange(T, device=dev, dtype=torch.int64).unsqueeze(0).expand(B, T)
        pos = position_ids.reshape(-1).to(torch.int64).contiguous()
        cos, sin = self.rope(T, dev, inputs_embeds.dtype)
        padded = attention_mask is not None and not bool(attention_mask.all())      # MaskInfo answers on the host (no sync)
        if hasattr(attention_mask, "mask"):
            attention_mask = attention_mask.mask
        pad = K.pad_ranges(attention_mask) if padded else None       # per-row real key range; the attention kernels mask from it

        stream = inputs_embeds.reshape(B * T, H)
        branch = None                                   # pending residual-branch output (added inside the next norm)
        l_auxes, records = [], []
        moe_i = 0
        if moe_noise is None:
            # DeepSpeed draws fresh Gumbel noise in every MoE layer; one draw for all layers of this forward is the same distribution
            # with 5 launches instead of 5 per layer
            moes = [l.mlp for l in self.layers if isinstance(l.mlp, MoE)]
            if moes and len({m.num_experts for m in moes}) == 1:
                moe_noise = gumbel_noise((len(moes), B * T, moes[0].num_experts), dev).unbind(0)
        for li, layer in enumerate(self.layers):
            at = layer.self_attn
            nh, nkv, hd = at.num_heads, at.num_key_value_heads, at.head_dim
            if branch is None:
                x, stream = K.rmsnorm(stream, layer.input_layernorm.weight, cfg.rms_norm_eps, wgrad=self.gview(layer.input_layernorm.weight))
            else:
                x, stream = K.rmsnorm(branch, layer.input_layernorm.weight, cfg.rms_norm_eps, res=stream, wgrad=self.gview(layer.input_layernorm.weight))
            qkv = K.qkv_rope(x, at.qkv_weight, at.qkv_bias, cos, sin, pos, nh, nkv, hd, self.gview(at.qkv_weight), self.gview(at.qkv_bias))
            if cache is not None:
                K.kv_append(qkv, B, T, nh, nkv, hd, cache.k[li], cache.v[li], cache.len)
            attn = K.attention(qkv, B, T, nh, nkv, hd, True, None, pad)
            if K.residual_fusable(attn, stream, self.gview(at.o_proj.weight), self.gview(layer.post_attention_layernorm.weight)):
                # frozen / no-grad forward: o_proj's epilogue writes residual + branch (modeling_qwen2.py:796), the norm reads one tensor
                stream = K.gemm_residual(attn, at.o_proj.weight, None, stream)
                x, stream = K.rmsnorm(stream, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
            else:
                branch = K.linear(attn, at.o_proj.weight, None, self.gview(at.o_proj.weight), None)
                x, stream = K.rmsnorm(branch, layer.post_attention_layernorm.weight, cfg.rms_norm_eps, res=stream,
                                      wgrad=self.gview(layer.post_attention_layernorm.weight))
            mlp = layer.mlp
            if isinstance(mlp, MoE):
                ds = mlp.deepspeed_moe
                E = mlp.num_experts
                noise = moe_noise[moe_i] if moe_noise is not None else gumbel_noise((B * T, E), dev)
                moe_i += 1
                cf = mlp.capacity_factor if training_moe else mlp.eval_capacity_factor
                wg = ds.gate.wg.weight
                if torch.is_grad_enabled() and (x.requires_grad or wg.requires_grad or ds.experts.deepspeed_experts[0].down_proj.weight.requires_grad):
                    grads = dict(wg=self.gview(wg), w_gu=self.gview(ds.experts.gu_weight), w_dn=self.gview(ds.experts.dn_weight))
                    stream, l_aux = K.MoEFn.apply(x, stream, wg, ds.experts.gu_weight, ds.experts.dn_weight, noise, cf,
                                                  mlp.min_capacity, grads)
                else:
                    stream, l_aux, rec = K.moe_forward_nograd(x, stream, wg, ds.experts.gu_weight, ds.experts.dn_weight, noise,
                                                              cf, mlp.min_capacity)
                    records.append(rec)
                l_auxes.append(l_aux)
                branch = None
            elif K.residual_fusable(x, stream, self.gview(mlp.gu_weight), self.gview(mlp.down_proj.weight)):
                stream = K.mlp(x, mlp.gu_weight, mlp.down_proj.weight, res=stream)      # down_proj epilogue adds the stream (:808)
                branch = None
            else:
                branch = K.mlp(x, mlp.gu_weight, mlp.down_proj.weight, self.gview(mlp.gu_weight), self.gview(mlp.down_proj.weight))
        if branch is None:
            out, _ = K.rmsnorm(stream, self.norm.weight, cfg.rms_norm_eps, wgrad=self.gview(self.norm.weight))
        else:
            out, _ = K.rmsnorm(branch, self.norm.weight, cfg.rms_norm_eps, res=stream, wgrad=self.gview(self.norm.weight))
        if cache is not None:
            cache.len.add_(T)
            cache.length += T
        return out.view(B, T, H), l_auxes, records

    def _decode_step(self, inputs_embeds, moe_noise, training_moe, cache):
        """One cached step: each sequence's new token sits at position len[b] (the reference's rule for a cached step,
        llava_arch.py:162-172, on unpadded prompts), its k / v are appended at row len[b], and its query attends to rows [0, len[b] + 1).
        Everything the step reads about the position is on the device, so the step can be captured once and replayed.  MoE layers route
        the B new tokens alone (top2gating with S = B, as MoEQwen1_5Model_forward does with a cache, llava_qwen1_5_moe.py:223-236).
        The layer body is forward's no-grad layer body with the attention swapped for append + decode attention: the same norm and
        residual-fusion choices, the same MoE call and final norm.  A change to one loop must be made to the other;
        tests/test_decode_gpu.py checks that the two give the same K / V, bit for bit."""
        cfg = self.config
        B, T, H = inputs_embeds.shape
        if T != 1:
            raise NotImplementedError("a cached step decodes one token per sequence (got %d)" % T)
        cache.check(B, 1)
        dev = inputs_embeds.device
        cos, sin = cache.rope
        torch.add(cache.len, 1, out=cache.end)
        cache.pos.copy_(cache.len)
        stream = inputs_embeds.reshape(B, H)
        branch = None
        l_auxes, records = [], []
        moe_i = 0
        for li, layer in enumerate(self.layers):
            at = layer.self_attn
            nh, nkv, hd = at.num_heads, at.num_key_value_heads, at.head_dim
            if branch is None:
                x, stream = K.rmsnorm(stream, layer.input_layernorm.weight, cfg.rms_norm_eps)
            else:
                x, stream = K.rmsnorm(branch, layer.input_layernorm.weight, cfg.rms_norm_eps, res=stream)
            qkv = K.qkv_rope(x, at.qkv_weight, at.qkv_bias, cos, sin, cache.pos, nh, nkv, hd)
            K.kv_append(qkv, B, 1, nh, nkv, hd, cache.k[li], cache.v[li], cache.len)
            attn, _ = K.attn_decode(qkv, nh, nkv, hd, cache.k[li], cache.v[li], cache.end, cache.ws)
            if K.residual_fusable(attn, stream):
                stream = K.gemm_residual(attn, at.o_proj.weight, None, stream)
                x, stream = K.rmsnorm(stream, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
            else:
                branch = K.linear(attn, at.o_proj.weight)
                x, stream = K.rmsnorm(branch, layer.post_attention_layernorm.weight, cfg.rms_norm_eps, res=stream)
            mlp = layer.mlp
            if isinstance(mlp, MoE):
                ds = mlp.deepspeed_moe
                noise = moe_noise[moe_i] if moe_noise is not None else gumbel_noise((B, mlp.num_experts), dev)
                moe_i += 1
                cf = mlp.capacity_factor if training_moe else mlp.eval_capacity_factor
                stream, l_aux, rec = K.moe_forward_nograd(x, stream, ds.gate.wg.weight, ds.experts.gu_weight, ds.experts.dn_weight, noise,
                                                          cf, mlp.min_capacity)
                records.append(rec)
                l_auxes.append(l_aux)
                branch = None
            elif K.residual_fusable(x, stream):
                stream = K.mlp(x, mlp.gu_weight, mlp.down_proj.weight, res=stream)
                branch = None
            else:
                branch = K.mlp(x, mlp.gu_weight, mlp.down_proj.weight)
        if branch is None:
            out, _ = K.rmsnorm(stream, self.norm.weight, cfg.rms_norm_eps)
        else:
            out, _ = K.rmsnorm(branch, self.norm.weight, cfg.rms_norm_eps, res=stream)
        cache.len.copy_(cache.end)
        cache.length += 1
        return out.view(B, 1, H), l_auxes, records


class KVCache:
    """Decoding cache of a Qwen2Model for B equal-length sequences of up to max_len positions.

    Per layer one K and one V buffer [B, nkv, max_len, hp] bf16 (HF's legacy layout; hp = the head width the attention kernels run,
    head dims below 64 zero-padded), the valid length of every sequence on the device (``len`` int32 [B], which the kernels read, so a
    captured decode step serves every position) and its host mirror ``length``: the host always knows how many rows a forward adds, so
    every append is bounds-checked without a sync.  ``cache[i]`` gives layer i's (k, v) views [B, nkv, length, hd], the legacy tuple layout
    llava_arch.py:165 indexes.  The RoPE tables cover max_len at allocation, so nothing is rebuilt inside a captured step."""

    def __init__(self, model, batch, max_len):
        cfg = model.config
        w = model.embed_tokens.weight
        dev, dt = w.device, w.dtype
        nh, nkv = cfg.num_attention_heads, cfg.num_key_value_heads
        self.head_dim = cfg.hidden_size // nh
        hp = K.attn_head_dim(self.head_dim)
        self.batch, self.max_len = int(batch), int(max_len)
        self.k = [torch.empty(batch, nkv, max_len, hp, device=dev, dtype=dt) for _ in model.layers]
        self.v = [torch.empty(batch, nkv, max_len, hp, device=dev, dtype=dt) for _ in model.layers]
        self.len = torch.zeros(batch, dtype=torch.int32, device=dev)
        self.end = torch.zeros(batch, dtype=torch.int32, device=dev)          # len + 1 during a decode step
        self.pos = torch.zeros(batch, dtype=torch.int64, device=dev)          # RoPE positions of a decode step
        self.ws = torch.empty(max(1, K.attn_decode_ws_elems(batch, nh, nkv, self.head_dim, max_len)), dtype=torch.float32, device=dev)
        self.rope = model.rope(max_len, dev, dt)
        self.length = 0

    def check(self, batch, n_new):
        if batch != self.batch:
            raise ValueError("KVCache holds %d sequences, got a batch of %d" % (self.batch, batch))
        if self.length + n_new > self.max_len:
            raise ValueError("KVCache is full: %d cached + %d new positions > max_len %d" % (self.length, n_new, self.max_len))

    def get_seq_length(self, layer_idx=0):
        return self.length

    def __len__(self):
        return len(self.k)

    def __getitem__(self, i):
        n, hd = self.length, self.head_dim
        return self.k[i][:, :, :n, :hd], self.v[i][:, :, :n, :hd]


def gumbel_noise(shape, device):
    """deepspeed gumbel_rsample (Gumbel(0,1) via -log(-log U)); Philox stream of the current device generator."""
    u = torch.rand(shape, device=device, dtype=torch.float32).clamp_(min=1e-20, max=1.0 - 1e-7)
    return -torch.log(-torch.log(u))
