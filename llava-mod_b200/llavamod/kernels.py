"""Torch-facing wrappers (``torch.autograd.Function``) around the C ABI of liblmod_b200.so.

Each wrapper cites the reference call site it stands in for.  Tensors are bf16 CUDA, contiguous; fp32 only
where the reference keeps fp32 (router gate, loss scalars, optimizer state).  No CPU fallback.
"""
import collections

import torch
from torch.autograd import Function

from . import _C
from ._C import call, ptr

BF16 = torch.bfloat16

import contextlib
import os as _os

NVTX = bool(int(_os.environ.get("LLAVAMOD_NVTX", "0")))


@contextlib.contextmanager
def nvtx(name):
    """Named range for nsys / ncu timelines (LLAVAMOD_NVTX=1); a no-op otherwise (and inside CUDA-graph capture the ranges mark the
    capture pass only, which is what identifies the kernels of a phase in `ncu --nvtx`)."""
    if not NVTX:
        yield
        return
    torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        torch.cuda.nvtx.range_pop()


def _c(t):
    return t if t is None or t.is_contiguous() else t.contiguous()


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _C.LmodError("llavamod kernels need CUDA tensors (no CPU fallback); got a %s tensor" % t.device)


# ---------------------------------------------------------------------------------------------------
# GEMM plumbing.  Every dense contraction of the path (forward, dgrad, wgrad, grouped expert forms) runs on the hand-written wgmma /
# TMA GEMM of csrc/gemm.cu through lmod_gemm_bf16 / lmod_grouped_gemm_bf16; no library GEMM is called.
# ---------------------------------------------------------------------------------------------------
def _rows(t):
    t2 = t.reshape(-1, t.shape[-1])
    return t2 if t2.is_contiguous() else t2.contiguous()


def mm_nt(x, w, bias=None):
    """y[..,N] = x[..,K] @ w[N,K]^T (+bias) -- nn.Linear forward on the wgmma GEMM."""
    y = gemm(_rows(x), w, bias=bias)
    return y if x.dim() == 2 else y.view(*x.shape[:-1], w.shape[0])     # no view object for the 2-D case (RoPE writes in place)


def mm_nn(dy, w, m_dev=None):
    """dx[M,K] = dy[M,N] @ w[N,K] -- nn.Linear dgrad: B operand = w as stored (MN-major), no transpose copy.
    Few output tiles + a very long reduction (lm_head dgrad: K = vocab) -> split-K with fp32 atomics."""
    dy2 = _rows(dy)
    M, N = dy2.shape
    Kout = w.shape[1]
    tiles = ((M + 127) // 128) * ((Kout + 255) // 256)
    if tiles < 100 and N >= 16384:
        split = max(2, min(16, torch.cuda.get_device_properties(dy.device).multi_processor_count // max(1, tiles)))
        acc = torch.zeros(M, Kout, dtype=torch.float32, device=dy.device)
        gemm(dy2, w, b_mn=True, out_f32=acc, split_k=split, m_dev=m_dev)
        return acc.to(dy.dtype)
    if m_dev is not None:
        out = torch.zeros(M, Kout, dtype=dy.dtype, device=dy.device)         # rows past the extent's last 128-row tile stay zero
        return gemm(dy2, w, b_mn=True, out=out, m_dev=m_dev)
    return gemm(dy2, w, b_mn=True)


def mm_tn_acc(dy, x, grad, k_dev=None):
    """grad[N,K] += dy[M,N]^T @ x[M,K] -- nn.Linear wgrad accumulated in place into the flat grad buffer (both operands MN-major)."""
    dy2, x2 = _rows(dy), _rows(x)
    if grad.dtype == torch.float32:
        gemm(dy2, x2, a_mn=True, b_mn=True, out_f32=grad, k_dev=k_dev)
    else:
        gemm(dy2, x2, a_mn=True, b_mn=True, out=grad, accumulate=True, k_dev=k_dev)


# ---- active-row compaction of the loss head (csrc/rows.cu) ---------------------------------------------------------------------
ROW_PAD = 256            # GEMM tile height: gathered buffers are zero-filled up to the next multiple so partial tiles stay exact zeros


def active_rows(labels_flat, seq_len, distill_all=False):
    """-> (perm int32 [N], count int32 [1]) on the device; no host sync."""
    _need_cuda(labels_flat)
    n = labels_flat.numel()
    perm = torch.empty(n, dtype=torch.int32, device=labels_flat.device)
    count = torch.empty(1, dtype=torch.int32, device=labels_flat.device)
    call("lmod_active_rows", ptr(labels_flat), n, seq_len, 1 if distill_all else 0, ptr(perm), ptr(count))
    return perm, count


def gather_rows(x2, perm, count, out=None):
    """Compact copy [round_up(N, ROW_PAD), H] of the rows perm[:count] of x2 (perm None: the first count rows); pad rows zeroed."""
    n, h = x2.shape
    if out is None:
        out = torch.empty((n + ROW_PAD - 1) // ROW_PAD * ROW_PAD, h, dtype=x2.dtype, device=x2.device)
    call("lmod_gather_rows", ptr(x2), x2.stride(0), ptr(perm), ptr(count), out.shape[0], h, ROW_PAD,
         ptr(out), out.stride(0))
    return out


def scatter_rows(xc, perm, count, n):
    out = torch.zeros(n, xc.shape[1], dtype=xc.dtype, device=xc.device)
    call("lmod_scatter_rows", ptr(xc), xc.stride(0), ptr(perm), ptr(count), min(xc.shape[0], n), xc.shape[1], ptr(out), out.stride(0))
    return out


def gemm(a, b, a_mn=False, b_mn=False, bias=None, out=None, accumulate=False, out_f32=None, split_k=1, m_dev=None, k_dev=None):
    """Hand-written wgmma/TMA GEMM (lmod_gemm_bf16).  D[M,N] (+)= A * B^T with
       a_mn=False: a is [M,K] ; True: a is [K,M]     b_mn=False: b is [N,K] ; True: b is [K,N].
       m_dev / k_dev: int32 device scalars bounding the rows of D / the reduction (lmod_gemm_bf16_dyn; active-row loss head)."""
    _need_cuda(a, b)
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N = b.shape[1] if b_mn else b.shape[0]
    if out_f32 is not None:                 # fp32 D32 += acc, split-K in epilogue bits 8..; no bf16 D, no bias
        D, ldd, bias, epilogue = None, out_f32.stride(0), None, (int(split_k) << 8) if split_k > 1 else 0
    else:
        D = out if out is not None else torch.empty(M, N, dtype=a.dtype, device=a.device)
        ldd, epilogue = D.stride(0), 1 if accumulate else 0
    call("lmod_gemm_bf16_dyn", ptr(a), a.stride(0), int(a_mn), ptr(b), b.stride(0), int(b_mn), ptr(D), ldd, M, N, K, ptr(bias), epilogue,
         ptr(out_f32), ptr(m_dev), ptr(k_dev))
    return out_f32 if out_f32 is not None else D


# The fused SwiGLU forward pays off only when the GEMM's main loop is long enough to hide its epilogue: it is used from a reduction
# length of FUSE_MIN_K on (the teacher's K = 4096); at the student's K = 1024 the element-wise kernel, which uses every warp of the SM,
# is faster (DESIGN.md section 4).
FUSE_MIN_K = 2048


def swiglu_fusable(I, K=None):
    """The fused SwiGLU GEMM tiles the intermediate dimension by 128 (the reference's tiny test shapes with I = 320 take GEMM + silu_mul).
    It is forward-only: a differentiated MLP keeps its pre-activations and runs GEMM + silu_mul."""
    return I % 128 == 0 and (K is None or K >= FUSE_MIN_K)


def gemm_swiglu(x2, w_gu):
    """act[M,I] = SwiGLU(x2 @ w_gu^T) in ONE GEMM (lmod_gemm_swiglu): w_gu is the fused gate|up weight [2I,H] as stored."""
    _need_cuda(x2, w_gu)
    M, H = x2.shape
    I = w_gu.shape[0] // 2
    act = torch.empty(M, I, dtype=x2.dtype, device=x2.device)
    call("lmod_gemm_swiglu", ptr(x2), x2.stride(0), ptr(w_gu), w_gu.stride(0), ptr(act), I, None, 0, M, I, H)
    return act


def grouped_gemm_swiglu(xp, w_gu, offsets, max_rows):
    """Experts' gate|up + SwiGLU on compact expert rows: w_gu [E,2I,H]; returns act [R,I]."""
    E, I2, H = w_gu.shape
    I = I2 // 2
    act = torch.empty(max_rows, I, dtype=xp.dtype, device=xp.device)
    call("lmod_grouped_gemm_swiglu", ptr(xp), xp.stride(0), ptr(w_gu), w_gu.stride(1), ptr(act), I, None, 0, ptr(offsets), E, max_rows, I, H)
    return act


def mlp(x, w_gu, w_dn, g_gu=None, g_dn=None):
    """Dense SwiGLU MLP.  No-grad calls take the fused SwiGLU epilogue where swiglu_fusable allows and keep nothing; differentiated
    calls run GEMM + silu_mul, whose backward needs the pre-activations."""
    I = w_gu.shape[0] // 2
    grad = torch.is_grad_enabled() and (x.requires_grad or g_gu is not None or g_dn is not None)
    if not grad and swiglu_fusable(I, w_gu.shape[1]):
        y = gemm(gemm_swiglu(_rows(x), w_gu), w_dn)
        return y if x.dim() == 2 else y.view(*x.shape[:-1], w_dn.shape[0])
    gu = linear(x, w_gu, None, g_gu, None)
    return linear(silu_mul(gu), w_dn, None, g_dn, None)


def grouped_gemm(a, b, out, offsets, mode, max_rows=None, accumulate=False):
    """lmod_grouped_gemm_bf16 on compact expert rows (offsets [G+1] int32 on device, 128-aligned).
       mode 0: out[R,N] = a[R,K] @ b[G,N,K]^T ; mode 1: out[R,N] = a[R,K] @ b[G,K,N] ; mode 2: out[G,M,N] (+)= a[R,M]^T @ b[R,N] per group."""
    G = offsets.numel() - 1
    R = a.shape[0] if max_rows is None else max_rows
    if mode == 0:
        ldb, ldd, M, N, K, mode, acc = b.stride(1), out.stride(0), 0, b.shape[1], b.shape[2], 0, 0
    elif mode == 1:
        ldb, ldd, M, N, K, mode, acc = b.stride(1), out.stride(0), 0, b.shape[2], b.shape[1], 1, 0
    else:
        ldb, ldd, M, N, K, mode, acc = b.stride(0), out.stride(1), a.shape[1], b.shape[1], 0, 2, 1 if accumulate else 0
    call("lmod_grouped_gemm_bf16", ptr(a), a.stride(0), ptr(b), ldb, ptr(out), ldd, ptr(offsets), G, R, M, N, K, mode, acc)
    return out


class LinearFn(Function):
    """nn.Linear (modeling_qwen2.py:678-680,726,199-200; CLIP / projector linears).  ``wgrad``/``bgrad`` are views
    of the flat gradient buffer (None when the parameter is frozen); wgrad is accumulated in place."""

    @staticmethod
    def forward(ctx, x, w, bias, wgrad, bgrad):
        _need_cuda(x, w)
        ctx.save_for_backward(x, w)
        ctx.wgrad, ctx.bgrad = wgrad, bgrad
        return mm_nt(x, w, bias)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy2 = _c(dy).reshape(-1, dy.shape[-1])
        dx = None
        if ctx.needs_input_grad[0]:
            dx = mm_nn(dy2, w).reshape(x.shape)
        if ctx.wgrad is not None:
            mm_tn_acc(dy2, x.reshape(-1, x.shape[-1]), ctx.wgrad)
        if ctx.bgrad is not None:
            ctx.bgrad.add_(dy2.sum(0).to(ctx.bgrad.dtype))
        return dx, None, None, None, None


def linear(x, w, bias=None, wgrad=None, bgrad=None):
    if torch.is_grad_enabled() and (x.requires_grad or wgrad is not None):
        return LinearFn.apply(x, w, bias, wgrad, bgrad)
    return mm_nt(x, w, bias)


# ---------------------------------------------------------------------------------------------------
# FP8 (e4m3) frozen decoder linears: csrc/quant.cu (row-wise quantisers) + csrc/gemm_fp8.cu (e4m3 wgmma GEMM).  Forward only.
# ---------------------------------------------------------------------------------------------------
class Fp8Rows:
    """Rows quantised to e4m3: ``q`` uint8 [M,K] (the e4m3 bytes), ``scale`` fp32 [M]; row m stands for scale[m] * e4m3(q[m]).  A weight
    [N,K] quantised per output channel, or activations quantised per token."""
    __slots__ = ("q", "scale")

    def __init__(self, q, scale):
        self.q, self.scale = q, scale

    @property
    def shape(self):
        return self.q.shape

    def dequant(self):
        """fp32 [M,K] (exact: an e4m3 value times an fp32 scale is rounded once)."""
        return self.q.view(torch.float8_e4m3fn).float() * self.scale[:, None]


def quant_rows(x):
    """lmod_quant_rows_e4m3 on the rows of a bf16 matrix (row stride free) -> Fp8Rows."""
    _need_cuda(x)
    x2 = x if x.dim() == 2 and x.stride(1) == 1 else _rows(x)
    M, Kd = x2.shape
    out = Fp8Rows(torch.empty(M, Kd, dtype=torch.uint8, device=x.device), torch.empty(M, dtype=torch.float32, device=x.device))
    call("lmod_quant_rows_e4m3", ptr(x2), x2.stride(0), ptr(out.q), ptr(out.scale), M, Kd)
    return out


def rmsnorm_quant(x, w, eps, res=None):
    """K.rmsnorm (no autograd) whose normalised rows come back quantised: -> (Fp8Rows, stream).  lmod_rmsnorm_quant_e4m3."""
    _need_cuda(x, w)
    if torch.is_grad_enabled() and (x.requires_grad or (res is not None and res.requires_grad)):
        raise RuntimeError("an FP8 (e4m3) decoder is forward-only: its input requires grad, run it under torch.no_grad()")
    x = _c(x)
    H = x.shape[-1]
    rows = x.numel() // H
    out = Fp8Rows(torch.empty(rows, H, dtype=torch.uint8, device=x.device), torch.empty(rows, dtype=torch.float32, device=x.device))
    s = torch.empty_like(x) if res is not None else None
    call("lmod_rmsnorm_quant_e4m3", ptr(x), ptr(_c(res)), ptr(w), rows, H, eps, ptr(out.q), ptr(out.scale), ptr(s))
    return out, (s if res is not None else x)


def gemm_fp8(a, w, bias=None):
    """bf16 [M,N] = a (Fp8Rows [M,K]) x w (Fp8Rows [N,K])^T (+bias) on the e4m3 wgmma GEMM (lmod_gemm_e4m3)."""
    M, Kd = a.shape
    out = torch.empty(M, w.shape[0], dtype=BF16, device=a.q.device)
    call("lmod_gemm_e4m3", ptr(a.q), a.q.stride(0), ptr(a.scale), ptr(w.q), w.q.stride(0), ptr(w.scale), ptr(bias),
         ptr(out), out.stride(0), M, w.shape[0], Kd)
    return out


def qkv_rope_fp8(a, w, bias, cos, sin, pos, nh, nkv, hd):
    """K.qkv_rope of a frozen FP8 layer: a = the quantised normalised rows (rmsnorm_quant), w = the quantised fused q|k|v weight."""
    if hd not in ATTN_HEAD_DIMS:
        return rope_(gemm_fp8(a, w, bias), cos, sin, pos, nh, nkv, hd)
    M, Kd = a.shape
    out = torch.empty(M, w.shape[0], dtype=BF16, device=a.q.device)
    call("lmod_gemm_e4m3_qkv_rope", ptr(a.q), a.q.stride(0), ptr(a.scale), ptr(w.q), w.q.stride(0), ptr(w.scale), ptr(bias),
         ptr(out), out.stride(0), M, Kd, nh, nkv, hd, ptr(cos), ptr(sin), ptr(pos))
    return out


def linear_fp8(x, w):
    """K.linear of a frozen FP8 layer for a bf16 input (o_proj on the attention output): quantise the rows, then the e4m3 GEMM."""
    y = gemm_fp8(quant_rows(x), w)
    return y if x.dim() == 2 else y.view(*x.shape[:-1], w.shape[0])


def mlp_fp8(a, w_gu, w_dn):
    """K.mlp of a frozen FP8 layer: a = the quantised normalised rows; gate|up with the SwiGLU epilogue where K.mlp fuses it, the
    activation quantised per token, down_proj."""
    I = w_gu.shape[0] // 2
    if swiglu_fusable(I, w_gu.shape[1]):
        act = torch.empty(a.shape[0], I, dtype=BF16, device=a.q.device)
        call("lmod_gemm_e4m3_swiglu", ptr(a.q), a.q.stride(0), ptr(a.scale), ptr(w_gu.q), w_gu.q.stride(0), ptr(w_gu.scale), ptr(act), I,
             a.shape[0], I, a.shape[1])
    else:
        act = silu_mul(gemm_fp8(a, w_gu))
    return gemm_fp8(quant_rows(act), w_dn)


# ---------------------------------------------------------------------------------------------------
# attention (K7)
# ---------------------------------------------------------------------------------------------------
ATTN_HEAD_DIMS = (64, 128)


def _check_pad(causal, pad):
    """The kernels un-mask the query rows in front of a left-padded sequence (they see no key under the causal mask) and give them
    every key.  Without the causal mask a key-padding mask would restrict those rows to [kv_lo, kv_hi) instead, so padding is only
    accepted together with causal=True (what the decoder passes); CLIP attends without padding."""
    if pad is not None and pad[0] is not None and not causal:
        raise _C.LmodError("attention: key padding (pad / kv_lo, kv_hi) is only supported with causal=True")


def attention_fwd(qkv, B, T, nh, nkv, hd, causal, scale=None, need_lse=False, pad=None):
    """Hand-written wgmma flash-attention forward on the fused QKV buffer [B*T, (nh+2nkv)*hd] -> [B*T, nh*hd] (+ lse [B,nh,T]).
    pad = (kv_lo, kv_hi): int32 [B] device tensors, the real key range of every batch row (padded batches), or None; needs causal."""
    _check_pad(causal, pad)
    _need_cuda(qkv)
    out = torch.empty(B * T, nh * hd, dtype=qkv.dtype, device=qkv.device)
    lse = torch.empty(B, nh, T, dtype=torch.float32, device=qkv.device) if need_lse else None
    lo, hi = pad if pad is not None else (None, None)
    call("lmod_attn_fwd", ptr(qkv), qkv.stride(0), B, T, nh, nkv, hd, 1 if causal else 0, float(scale if scale is not None else hd ** -0.5),
         ptr(out), out.stride(0), ptr(lse), ptr(lo), ptr(hi))
    return out, lse


class AttnFn(Function):
    """Qwen2SdpaAttention core (modeling_qwen2.py:713-721, 4-D mask :1035-1040): our wgmma forward (lmod_attn_fwd) and backward
    (lmod_attn_bwd); dq|dk|dv come back as one fused buffer."""

    @staticmethod
    def forward(ctx, qkv, B, T, nh, nkv, hd, causal, scale, kv_lo, kv_hi):
        scale = float(scale if scale is not None else hd ** -0.5)
        pad = (kv_lo, kv_hi) if kv_lo is not None else None
        out, lse = attention_fwd(qkv, B, T, nh, nkv, hd, causal, scale, need_lse=True, pad=pad)
        ctx.save_for_backward(qkv, out, lse, kv_lo, kv_hi)
        ctx.dims = (B, T, nh, nkv, hd, causal, scale)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, out, lse, kv_lo, kv_hi = ctx.saved_tensors
        B, T, nh, nkv, hd, causal, scale = ctx.dims
        pad = (kv_lo, kv_hi) if kv_lo is not None else None
        return (attention_bwd(qkv, out, _c(dout), lse, B, T, nh, nkv, hd, causal, scale, pad=pad),) + (None,) * 9


def attention_bwd(qkv, out, dout, lse, B, T, nh, nkv, hd, causal, scale, pad=None):
    """Hand-written wgmma flash-attention backward -> fused dqkv (same layout as qkv)."""
    _check_pad(causal, pad)
    dqkv = torch.empty_like(qkv)
    dq32 = torch.empty(B * T, nh * hd, dtype=torch.float32, device=qkv.device)
    dsum = torch.empty(B, nh, T, dtype=torch.float32, device=qkv.device)
    lo, hi = pad if pad is not None else (None, None)
    call("lmod_attn_bwd", ptr(qkv), qkv.stride(0), ptr(out), out.stride(0), ptr(dout), dout.stride(0), ptr(lse), B, T, nh, nkv, hd,
         1 if causal else 0, float(scale), ptr(dqkv), dqkv.stride(0), ptr(dq32), ptr(dsum), ptr(lo), ptr(hi))
    return dqkv


def attention(qkv, B, T, nh, nkv, hd, causal=True, scale=None, pad=None):
    """Self-attention on the fused, RoPE'd QKV buffer [B*T, (nh+2nkv)*hd] -> [B*T, nh*hd], always on the wgmma kernels.
    Head dims other than 64 / 128 (the reference's tiny test shapes) are zero-padded per head to the next built width: the extra
    q/k columns add 0 to every score and the extra v columns produce output columns that are sliced away (softmax scale = hd^-0.5 of
    the TRUE head dim); the pad / slice are plain tensor ops, so autograd carries the gradient back to the unpadded buffer."""
    scale = float(scale if scale is not None else hd ** -0.5)
    _check_pad(causal, pad)
    hp = attn_head_dim(hd)
    if hp != hd:
        o = attention(_pad_heads(qkv, nh + 2 * nkv, hd, hp), B, T, nh, nkv, hp, causal, scale, pad)
        return _unpad_heads(o, nh, hd)
    lo, hi = pad if pad is not None else (None, None)
    if torch.is_grad_enabled() and qkv.requires_grad:
        return AttnFn.apply(qkv, B, T, nh, nkv, hd, causal, scale, lo, hi)
    return attention_fwd(qkv, B, T, nh, nkv, hd, causal, scale, pad=pad)[0]


def attn_head_dim(hd):
    """Head width the attention kernels run for a model head dim: 64 / 128 as they are, smaller ones zero-padded (see attention)."""
    if hd > 128:
        raise _C.LmodError("head_dim %d > 128 is not built" % hd)
    return hd if hd in ATTN_HEAD_DIMS else (64 if hd < 64 else 128)


def _pad_heads(x, heads, hd, hp):
    """[rows, heads*hd] (row stride free) -> contiguous [rows, heads*hp], every head zero-padded to hp columns."""
    return torch.nn.functional.pad(x.view(x.shape[0], heads, hd), (0, hp - hd)).view(x.shape[0], heads * hp)


def _unpad_heads(x, heads, hd):
    """Inverse of _pad_heads: [rows, heads*hp] -> [rows, heads*hd], the first hd columns of every head (x itself when hp == hd)."""
    hp = x.shape[1] // heads
    return x if hp == hd else x.view(x.shape[0], heads, hp)[:, :, :hd].reshape(x.shape[0], heads * hd)


def _check_cache(k_cache, v_cache, B, nkv, hd):
    """The kernels index the cache as dense bf16 [B, nkv, max_len, attn_head_dim(hd)]."""
    want = (B, nkv, k_cache.shape[2] if k_cache.dim() == 4 else -1, attn_head_dim(hd))
    for t in (k_cache, v_cache):
        if t.dtype != BF16 or tuple(t.shape) != want or not t.is_contiguous():
            raise _C.LmodError("KV cache must be contiguous bf16 %s, got %s %s%s" % (want, t.dtype, tuple(t.shape),
                                                                                    "" if t.is_contiguous() else " (strided)"))


def _check_i32(t, B, name):
    if t.dtype != torch.int32 or t.numel() != B or not t.is_contiguous():
        raise _C.LmodError("%s must be a contiguous int32 tensor of %d elements, got %s %s" % (name, B, t.dtype, tuple(t.shape)))


def _cache_qkv(name, qkv, B, n, nh, nkv, hd, k_cache, v_cache, **i32):
    """Checks shared by the cache appends -> the QKV rows [B*n, (nh+2nkv)*hd] with every head padded to the cache's width hp.
    i32: the int32 [B] device arrays of the call, by name."""
    _need_cuda(qkv, k_cache, v_cache, *i32.values())
    _check_cache(k_cache, v_cache, B, nkv, hd)
    for key, t in i32.items():
        _check_i32(t, B, key)
    if qkv.dim() != 2 or qkv.shape[0] != B * n or qkv.shape[1] != (nh + 2 * nkv) * hd or qkv.stride(1) != 1:
        raise _C.LmodError("%s: qkv must be [B*%d, (nh+2nkv)*hd] with unit column stride, got %s" % (name, n, tuple(qkv.shape)))
    hp = k_cache.shape[-1]
    return qkv if hp == hd else _pad_heads(qkv, nh + 2 * nkv, hd, hp)


def kv_append(qkv, B, n_new, nh, nkv, hd, k_cache, v_cache, offsets):
    """DynamicCache.update: the k / v heads of the fused, RoPE'd QKV rows [B*n_new, (nh+2nkv)*hd] -> cache rows offsets[b] + [0, n_new)
    of k_cache / v_cache [B, nkv, max_len, hp] (hp = attn_head_dim(hd); padded heads get zero columns).  offsets: int32 [B] on the device."""
    qkv = _cache_qkv("kv_append", qkv, B, n_new, nh, nkv, hd, k_cache, v_cache, offsets=offsets)
    call("lmod_kv_append", ptr(qkv), qkv.stride(0), B, n_new, nh, nkv, k_cache.shape[3], ptr(offsets), ptr(k_cache), ptr(v_cache),
         k_cache.shape[2])


def kv_append_rows(qkv, B, T, nh, nkv, hd, k_cache, v_cache, src_lo, src_hi, offsets):
    """The prefill of a padded batch into the cache: rows [src_lo[b], src_hi[b]) of sequence b's T rows of the fused, RoPE'd QKV buffer
    [B*T, (nh+2nkv)*hd] -> cache rows offsets[b] + (r - src_lo[b]), so every sequence's real rows are packed from offsets[b].  src_lo /
    src_hi / offsets: int32 [B] on the device (pad_ranges gives the ranges); no other cache row is written."""
    qkv = _cache_qkv("kv_append_rows", qkv, B, T, nh, nkv, hd, k_cache, v_cache, src_lo=src_lo, src_hi=src_hi, offsets=offsets)
    call("lmod_kv_append_rows", ptr(qkv), qkv.stride(0), B, T, nh, nkv, k_cache.shape[3], ptr(src_lo), ptr(src_hi), ptr(offsets),
         ptr(k_cache), ptr(v_cache), k_cache.shape[2])


def attn_decode_ws_elems(B, nh, nkv, hd, max_len):
    return int(_C.lib().lmod_attn_decode_ws_elems(B, nh, nkv, attn_head_dim(hd), max_len))


def _decode_io(name, q, B, T, nh, nkv, hd, k_cache, v_cache, lens, ws, need_lse):
    """Checks shared by the decode-attention forms -> (q with every head padded to the cache's width hp, out [B*T, nh*hp] bf16,
    lse [B*T, nh] fp32 or None)."""
    _need_cuda(q, k_cache, v_cache, lens, ws)
    _check_cache(k_cache, v_cache, B, nkv, hd)
    _check_i32(lens, B, "lens")
    if T < 1 or q.dim() != 2 or q.shape[0] != B * T or q.shape[1] < nh * hd or q.stride(1) != 1 or q.dtype != BF16:
        raise _C.LmodError("%s: q must be bf16 [B*%d, >= nh*hd] with unit column stride, got %s %s" % (name, T, q.dtype, tuple(q.shape)))
    if ws.dtype != torch.float32 or not ws.is_contiguous():
        raise _C.LmodError("%s: ws must be a contiguous fp32 tensor" % name)
    hp = k_cache.shape[3]
    if hp != hd:
        q = _pad_heads(q[:, :nh * hd], nh, hd, hp)
    out = torch.empty(B * T, nh * hp, dtype=q.dtype, device=q.device)
    lse = torch.empty(B * T, nh, dtype=torch.float32, device=q.device) if need_lse else None
    return q, out, lse


def attn_decode(q, nh, nkv, hd, k_cache, v_cache, lens, ws, scale=None, need_lse=False):
    """Single-query attention of every sequence over its cached keys [0, lens[b]) (split-KV, lmod_attn_decode).  q: [B, >= nh*hd] rows
    whose first nh*hd columns are the query heads (the fused QKV rows of a decode step); k_cache / v_cache [B, nkv, max_len, hp];
    lens int32 [B] on the device; ws fp32 of at least attn_decode_ws_elems(...).  -> (out [B, nh*hd] bf16, lse [B, nh] fp32 or None)."""
    B = q.shape[0]
    q, out, lse = _decode_io("attn_decode", q, B, 1, nh, nkv, hd, k_cache, v_cache, lens, ws, need_lse)
    call("lmod_attn_decode", ptr(q), q.stride(0), ptr(k_cache), ptr(v_cache), ptr(lens), B, nh, nkv, k_cache.shape[3], k_cache.shape[2],
         float(scale if scale is not None else hd ** -0.5), ptr(out), out.stride(0), ptr(lse), ptr(ws), ws.numel())
    return _unpad_heads(out, nh, hd), lse


def attn_decode_chunk_ws_elems(B, T, nh, nkv, hd, max_len):
    return int(_C.lib().lmod_attn_decode_chunk_ws_elems(B, T, nh, nkv, attn_head_dim(hd), max_len))


def attn_decode_chunk(q, B, T, nh, nkv, hd, k_cache, v_cache, lens, ws, scale=None, need_lse=False):
    """T new query rows per sequence over the cache (lmod_attn_decode_chunk): row t of sequence b attends to keys
    [0, lens[b] - T + t + 1), where lens is the length after the T rows' k / v were appended.  q: [B*T, >= nh*hd] rows (row b*T + t);
    k_cache / v_cache [B, nkv, max_len, hp]; lens int32 [B] on the device; ws fp32 of at least attn_decode_chunk_ws_elems(...).
    Row t gives the bytes attn_decode gives for that row alone at lens[b] - T + t + 1.  -> (out [B*T, nh*hd] bf16, lse [B*T, nh] or None)."""
    q, out, lse = _decode_io("attn_decode_chunk", q, B, T, nh, nkv, hd, k_cache, v_cache, lens, ws, need_lse)
    call("lmod_attn_decode_chunk", ptr(q), q.stride(0), ptr(k_cache), ptr(v_cache), ptr(lens), B, T, nh, nkv, k_cache.shape[3],
         k_cache.shape[2], float(scale if scale is not None else hd ** -0.5), ptr(out), out.stride(0), ptr(lse), ptr(ws), ws.numel())
    return _unpad_heads(out, nh, hd), lse


def attn_decode_shared_ws_elems(B, n, nh, nkv, hd, max_len):
    return int(_C.lib().lmod_attn_decode_shared_ws_elems(B, n, nh, nkv, attn_head_dim(hd), max_len))


def attn_decode_shared(q, n, nh, nkv, hd, k_prefix, v_prefix, prefix_len, k_suffix, v_suffix, lens, max_len, ws, scale=None,
                       need_lse=False):
    """Single-query attention of n sequences per prompt that share the prompt's cached rows (lmod_attn_decode_shared).  q: [B*n, >= nh*hd]
    rows, row b*n + j copy j of prompt b; k_prefix / v_prefix [B, nkv, P, hp] hold prompt b's keys [0, prefix_len[b]); k_suffix / v_suffix
    [B*n, nkv, S, hp] hold each copy's keys from prefix_len[b] on (key i at row i - prefix_len[b]); lens int32 [B*n] total keys,
    prefix_len int32 [B], both on the device; max_len: the length of the equivalent per-sequence cache, which sets the splits.  Row b*n + j
    gives the bytes attn_decode gives on its materialised cache of max_len rows.  -> (out [B*n, nh*hd] bf16, lse [B*n, nh] or None)."""
    B = k_prefix.shape[0]
    _need_cuda(k_prefix, v_prefix, prefix_len)
    _check_cache(k_prefix, v_prefix, B, nkv, hd)
    _check_i32(prefix_len, B, "prefix_len")
    q, out, lse = _decode_io("attn_decode_shared", q, B * n, 1, nh, nkv, hd, k_suffix, v_suffix, lens, ws, need_lse)
    call("lmod_attn_decode_shared", ptr(q), q.stride(0), ptr(k_prefix), ptr(v_prefix), ptr(prefix_len), k_prefix.shape[2], ptr(k_suffix),
         ptr(v_suffix), k_suffix.shape[2], ptr(lens), B, n, nh, nkv, k_prefix.shape[3], max_len,
         float(scale if scale is not None else hd ** -0.5), ptr(out), out.stride(0), ptr(lse), ptr(ws), ws.numel())
    return _unpad_heads(out, nh, hd), lse


_BEAM_TABLES = collections.OrderedDict()     # buffer pointers -> the device array of them lmod_kv_beam_reorder reads


def kv_beam_reorder(bufs, n, hd, rows, parent):
    """Beam search's cache reorder in place (lmod_kv_beam_reorder), every buffer in one launch: bufs are bf16 [P*n, nkv, cap, hp] (all
    layers' K and V), rows host ints [P] and parent host ints [P*n] in [0, n).  Row r < rows[b] of beam j of prompt b, columns [0, hd), takes
    the bytes of beam parent[b*n + j]'s row r; nothing else is written.  The operands are checked on the host and copied to the device in
    one transfer, so the call reads nothing back."""
    bufs = list(bufs)
    if not bufs:
        raise _C.LmodError("kv_beam_reorder: no buffers")
    _need_cuda(*bufs)
    shape = tuple(bufs[0].shape)
    if len(shape) != 4 or shape[0] % max(1, n) or n < 1:
        raise _C.LmodError("kv_beam_reorder: buffers must be [P*n, nkv, cap, hp] with n = %r, got %s" % (n, shape))
    for t in bufs:
        if t.dtype != BF16 or tuple(t.shape) != shape or not t.is_contiguous() or t.device != bufs[0].device:
            raise _C.LmodError("kv_beam_reorder: every buffer must be contiguous bf16 %s on one device, got %s %s" % (shape, t.dtype,
                                                                                                                     tuple(t.shape)))
    P, cap, hp = shape[0] // n, shape[2], shape[3]
    if not 0 < hd <= hp or hd % 8:
        raise _C.LmodError("kv_beam_reorder: hd %r must be a multiple of 8 in (0, %d]" % (hd, hp))
    rows, parent = [int(r) for r in rows], [int(p) for p in parent]
    if len(rows) != P or len(parent) != P * n:
        raise _C.LmodError("kv_beam_reorder: %d prompts of %d beams need %d rows and %d parents, got %d and %d"
                           % (P, n, P, P * n, len(rows), len(parent)))
    if any(not 0 <= r <= cap for r in rows):
        raise _C.LmodError("kv_beam_reorder: rows %s outside [0, cap = %d]" % (rows, cap))
    if any(not 0 <= p < n for p in parent):
        raise _C.LmodError("kv_beam_reorder: parents %s outside [0, n = %d)" % (parent, n))
    key = tuple(t.data_ptr() for t in bufs)
    table = _BEAM_TABLES.pop(key, None)
    if table is None:
        table = torch.tensor(key, dtype=torch.int64).to(bufs[0].device)
    _BEAM_TABLES[key] = table
    while len(_BEAM_TABLES) > 16:
        _BEAM_TABLES.popitem(last=False)
    ops = torch.tensor(rows + parent, dtype=torch.int32).to(bufs[0].device)
    call("lmod_kv_beam_reorder", ptr(table), len(bufs), P, n, shape[1], cap, hd, hp, ptr(ops), ptr(ops[P:]))


def spec_accept(target_logits, draft_tokens, draft_logits=None, u=None, len_target=None, len_draft=None):
    """Acceptance of one assisted-decoding round (lmod_spec_accept).  target_logits fp32 [B, k+1, V_t]: row j scores draft token j+1 (row k
    the bonus token); draft_tokens int64 [B, k].  Greedy (u None): accept while the draft equals the target's argmax.  Sampling: u fp32
    [B, k+1] uniforms and draft_logits fp32 [B, k, V_d], both after the logits processors (-inf = probability 0).  len_target / len_draft:
    int32 [B] cache lengths, rolled back on the device by k - n_acc.  -> (n_acc int32 [B], next int64 [B]) on the device."""
    if target_logits.dim() != 3 or target_logits.dtype != torch.float32:
        raise _C.LmodError("spec_accept: target_logits must be fp32 [B, k+1, V], got %s %s" % (target_logits.dtype, tuple(target_logits.shape)))
    B, k1, V_t = target_logits.shape
    k = k1 - 1
    if k < 1 or draft_tokens.dtype != torch.int64 or tuple(draft_tokens.shape) != (B, k):
        raise _C.LmodError("spec_accept: draft_tokens must be int64 [B, k] with k >= 1, got %s %s" % (draft_tokens.dtype, tuple(draft_tokens.shape)))
    V_d = 0
    if u is not None:
        if draft_logits is None or draft_logits.dim() != 3 or draft_logits.dtype != torch.float32 or tuple(draft_logits.shape[:2]) != (B, k):
            raise _C.LmodError("spec_accept: sampling needs fp32 draft_logits [B, k, V_d]")
        if u.dtype != torch.float32 or tuple(u.shape) != (B, k + 1):
            raise _C.LmodError("spec_accept: u must be fp32 [B, k+1], got %s %s" % (u.dtype, tuple(u.shape)))
        V_d = draft_logits.shape[2]
        draft_logits, u = draft_logits.contiguous(), u.contiguous()
        _need_cuda(draft_logits, u)
    for t, name in ((len_target, "len_target"), (len_draft, "len_draft")):
        if t is not None:
            _need_cuda(t)
            _check_i32(t, B, name)
    target_logits, draft_tokens = target_logits.contiguous(), draft_tokens.contiguous()
    _need_cuda(target_logits, draft_tokens)
    n_acc = torch.empty(B, dtype=torch.int32, device=target_logits.device)
    nxt = torch.empty(B, dtype=torch.int64, device=target_logits.device)
    call("lmod_spec_accept", ptr(target_logits), V_t, ptr(draft_logits) if u is not None else None, V_d, ptr(draft_tokens), ptr(u), B, k,
         ptr(n_acc), ptr(nxt), ptr(len_target), ptr(len_draft))
    return n_acc, nxt

def pad_ranges(attention_mask):
    """[B,T] bool mask (contiguous real tokens, right or left padded -- what the collators and the multimodal splice produce) ->
    (kv_lo, kv_hi) int32 [B] on the device, no host sync."""
    m = attention_mask.to(torch.int32)
    T = m.shape[1]
    lo = m.argmax(1).to(torch.int32)
    hi = (T - m.flip(1).argmax(1)).to(torch.int32)
    none = m.sum(1) == 0
    return torch.where(none, torch.zeros_like(lo), lo).contiguous(), torch.where(none, torch.zeros_like(hi), hi).contiguous()


# ---------------------------------------------------------------------------------------------------
# norms / rope / activations
# ---------------------------------------------------------------------------------------------------
class RMSNormFn(Function):
    """Qwen2RMSNorm (modeling_qwen2.py:105-110) with the decoder layer's residual add fused in
    (modeling_qwen2.py:796,808 / llava_qwen1_5_moe.py:156,167).  Returns (normed, residual_stream)."""

    @staticmethod
    def forward(ctx, x, res, w, eps, wgrad=None):
        _need_cuda(x, w)
        x = _c(x)
        rstd = torch.empty(x.numel() // x.shape[-1], dtype=torch.float32, device=x.device)
        y, s = _rmsnorm_fwd(x, res, w, eps, rstd)
        ctx.save_for_backward(s, w, rstd)
        ctx.had_res = res is not None
        ctx.wgrad = wgrad                                   # view of the flat gradient buffer when the norm weight trains
        if res is None:
            return y, x.new_empty(0)
        return y, s

    @staticmethod
    def backward(ctx, dy, ds):
        s, w, rstd = ctx.saved_tensors
        H = s.shape[-1]
        rows = s.numel() // H
        dy = _c(dy)
        dsp = None
        if ctx.had_res and ds is not None:
            dsp = ptr(_c(ds))
        dx = torch.empty_like(s)
        call("lmod_rmsnorm_bwd", ptr(dy), ptr(s), ptr(w), ptr(rstd), dsp, rows, H, ptr(dx))
        if ctx.wgrad is not None:
            call("lmod_rmsnorm_wgrad", ptr(dy), ptr(s), ptr(rstd), rows, H, ptr(_zero_ws(s.device, H)), ptr(ctx.wgrad))
        return dx, (dx if ctx.had_res else None), None, None, None


_ZERO_WS = {}


def _zero_ws(device, n):
    """fp32 workspace that kernels receive zeroed and hand back zeroed (lmod_rmsnorm_wgrad)."""
    ws = _ZERO_WS.get(device)
    if ws is None or ws.numel() < n:
        ws = _ZERO_WS[device] = torch.zeros(max(n, 8192), dtype=torch.float32, device=device)
    return ws


def _rmsnorm_fwd(x, res, w, eps, rstd=None):
    """lmod_rmsnorm_fwd -> (y, stream): stream = x + res, or x itself without res.  rstd: fp32 [rows] output, or None."""
    x = _c(x)
    H = x.shape[-1]
    y = torch.empty_like(x)
    s = torch.empty_like(x) if res is not None else None
    call("lmod_rmsnorm_fwd", ptr(x), ptr(_c(res)), ptr(w), x.numel() // H, H, eps, ptr(y), ptr(s), ptr(rstd))
    return y, (s if s is not None else x)


def rmsnorm(x, w, eps, res=None, wgrad=None):
    """-> (y, stream) where stream = x + res (or x).  Without autograd the kernel is called directly."""
    if torch.is_grad_enabled() and (x.requires_grad or (res is not None and res.requires_grad) or wgrad is not None):
        y, s = RMSNormFn.apply(x, res, w, eps, wgrad)
        return y, (s if res is not None else x)
    return _rmsnorm_fwd(x, res, w, eps)


def layernorm(x, w, b, eps):
    """CLIP LayerNorm (transformers CLIPVisionModel via clip_encoder.py:54); frozen tower: forward only."""
    x = _c(x)
    H = x.shape[-1]
    y = torch.empty_like(x)
    call("lmod_layernorm_fwd", ptr(x), ptr(w), ptr(b), x.numel() // H, H, eps, ptr(y))
    return y


def _rope(buf, cos, sin, pos, nh, nkv, hd, inverse):
    """lmod_rope in place on the q and k heads of the fused QKV rows buf [rows, (nh + 2*nkv)*hd]; inverse: the transpose rotation."""
    ld = buf.shape[-1]
    call("lmod_rope", ptr(buf), ld, nh, buf.data_ptr() + nh * hd * 2, ld, nkv, hd, ptr(cos), ptr(sin), ptr(pos), buf.numel() // ld,
         1 if inverse else 0)
    return buf


def _rope_grad(d, cos, sin, pos, nh, nkv, hd):
    # Rotated back in a copy: autograd may hand backward a gradient that is still read elsewhere (the caller's tensor in
    # out.backward(grad), a tensor hook's argument), and rotating it in place would change what those see.
    return _rope(d.clone(memory_format=torch.contiguous_format), cos, sin, pos, nh, nkv, hd, True)


class RopeFn(Function):
    """apply_rotary_pos_emb (modeling_qwen2.py:159-184) in place on the fused QKV projection output
    [rows, (nh + 2*nkv)*hd]: q heads first, then k heads, then v."""

    @staticmethod
    def forward(ctx, qkv, cos, sin, pos, nh, nkv, hd):
        _rope(qkv, cos, sin, pos, nh, nkv, hd, False)
        ctx.mark_dirty(qkv)
        ctx.save_for_backward(cos, sin, pos)
        ctx.dims = (nh, nkv, hd)
        return qkv

    @staticmethod
    def backward(ctx, d):
        cos, sin, pos = ctx.saved_tensors
        return (_rope_grad(d, cos, sin, pos, *ctx.dims),) + (None,) * 6


def _gemm_qkv_rope(x2, w, bias, cos, sin, pos, nh, nkv, hd):
    """lmod_gemm_qkv_rope: [rows, (nh + 2*nkv)*hd] = x2 @ w^T + bias with the q and k heads rotated."""
    out = torch.empty(x2.shape[0], w.shape[0], dtype=x2.dtype, device=x2.device)
    call("lmod_gemm_qkv_rope", ptr(x2), x2.stride(0), ptr(w), w.stride(0), ptr(bias), ptr(out), out.stride(0), x2.shape[0], x2.shape[1],
         nh, nkv, hd, ptr(cos), ptr(sin), ptr(pos))
    return out


class QKVRopeFn(Function):
    """q|k|v projection + rotary embedding (modeling_qwen2.py:678-691): ONE GEMM whose epilogue adds the bias and rotates the q / k heads
    (lmod_gemm_qkv_rope).  Backward: the transpose rotation on a copy of the incoming dqkv, then dgrad / wgrad / bias gradient as LinearFn."""

    @staticmethod
    def forward(ctx, x, w, bias, cos, sin, pos, nh, nkv, hd, wgrad, bgrad):
        x2 = _rows(x)
        out = _gemm_qkv_rope(x2, w, bias, cos, sin, pos, nh, nkv, hd)
        ctx.save_for_backward(x2, w, cos, sin, pos)
        ctx.dims = (nh, nkv, hd)
        ctx.g = (wgrad, bgrad)
        ctx.xshape = x.shape
        return out

    @staticmethod
    def backward(ctx, d):
        x2, w, cos, sin, pos = ctx.saved_tensors
        wgrad, bgrad = ctx.g
        d = _rope_grad(d, cos, sin, pos, *ctx.dims)
        dx = mm_nn(d, w).reshape(ctx.xshape) if ctx.needs_input_grad[0] else None
        if wgrad is not None:
            mm_tn_acc(d, x2, wgrad)
        if bgrad is not None:
            bgrad.add_(d.sum(0).to(bgrad.dtype))
        return (dx,) + (None,) * 10


def qkv_rope(x, w, bias, cos, sin, pos, nh, nkv, hd, wgrad=None, bgrad=None):
    """Fused q|k|v projection + RoPE for the head dims the epilogue is built for; other head dims (tiny test shapes) take GEMM + lmod_rope.
    Both return [rows, (nh + 2 nkv) hd]: the unfused path rotates the GEMM output in place, so it must not be a view LinearFn made."""
    if hd not in ATTN_HEAD_DIMS:
        return rope_(linear(_rows(x), w, bias, wgrad, bgrad), cos, sin, pos, nh, nkv, hd)
    if torch.is_grad_enabled() and (x.requires_grad or wgrad is not None):
        return QKVRopeFn.apply(x, w, bias, cos, sin, pos, nh, nkv, hd, wgrad, bgrad)
    return _gemm_qkv_rope(_rows(x), w, bias, cos, sin, pos, nh, nkv, hd)


def rope_(qkv, cos, sin, pos, nh, nkv, hd):
    if torch.is_grad_enabled() and qkv.requires_grad:
        return RopeFn.apply(qkv, cos, sin, pos, nh, nkv, hd)
    return _rope(qkv, cos, sin, pos, nh, nkv, hd, False)


def _silu_mul(gu):
    """lmod_silu_mul_fwd on the contiguous fused gate|up rows gu [..., 2I] -> [..., I]."""
    I = gu.shape[-1] // 2
    out = torch.empty(gu.shape[:-1] + (I,), dtype=gu.dtype, device=gu.device)
    call("lmod_silu_mul_fwd", ptr(gu), 2 * I, gu.numel() // gu.shape[-1], I, ptr(out))
    return out


class SiluMulFn(Function):
    """act_fn(gate_proj(x)) * up_proj(x) (modeling_qwen2.py:199-200) on the fused [rows, 2I] gate|up GEMM output."""

    @staticmethod
    def forward(ctx, gu):
        gu = _c(gu)
        ctx.save_for_backward(gu)
        return _silu_mul(gu)

    @staticmethod
    def backward(ctx, d):
        (gu,) = ctx.saved_tensors
        return silu_mul_bwd(d, gu)


def silu_mul(gu):
    if torch.is_grad_enabled() and gu.requires_grad:
        return SiluMulFn.apply(gu)
    return _silu_mul(_c(gu))


def silu_mul_bwd(d, gu):
    I = gu.shape[-1] // 2
    dgu = torch.empty_like(gu)
    call("lmod_silu_mul_bwd", ptr(_c(d)), ptr(gu), 2 * I, gu.numel() // gu.shape[-1], I, ptr(dgu))
    return dgu


ACT_GELU, ACT_QUICK_GELU, ACT_NONE = 0, 1, 2


def bias_act(x, bias, act):
    x = _c(x)
    n = x.shape[-1]
    y = torch.empty_like(x)
    call("lmod_bias_act_fwd", ptr(x), ptr(bias), x.numel() // n, n, act, ptr(y))
    return y


def add_(a, b):
    """a += b in place, element by element in bf16 (lmod_add); a and b contiguous with the same number of elements."""
    call("lmod_add", ptr(a), ptr(b), a.numel(), ptr(a))
    return a


class GeluFn(Function):
    """nn.GELU() of the mlp2x_gelu projector (multimodal_projector/builder.py:57-61)."""

    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        ctx.save_for_backward(x)
        return bias_act(x, None, ACT_GELU)

    @staticmethod
    def backward(ctx, d):
        (x,) = ctx.saved_tensors
        dx = torch.empty_like(x)
        call("lmod_gelu_bwd", ptr(_c(d)), ptr(x), x.numel(), ptr(dx))
        return dx


def gelu(x):
    if torch.is_grad_enabled() and x.requires_grad:
        return GeluFn.apply(x)
    return bias_act(x, None, ACT_GELU)


# ---------------------------------------------------------------------------------------------------
# multimodal splice (llava_arch.py:228-320): the integer plan is built on the host (see llava_arch.py in this
# package); the device part is one gather kernel and, backwards, one scatter into the projector output grads.
# ---------------------------------------------------------------------------------------------------
def _splice_embed(feats, embed_w, src, img_index, n_patches):
    """lmod_splice_embed -> [B, T, H]: embedding rows of the tokens of src [B, T], image feature rows where it points at them."""
    B, T = src.shape
    H = embed_w.shape[1]
    out = torch.empty(B, T, H, dtype=embed_w.dtype, device=embed_w.device)
    call("lmod_splice_embed", ptr(embed_w), ptr(feats), ptr(src), ptr(img_index), B * T, H, n_patches, ptr(out))
    return out


class SpliceFn(Function):
    @staticmethod
    def forward(ctx, feats, embed_w, src, img_index, n_patches, embed_grad=None, order=None):
        out = _splice_embed(feats, embed_w, src, img_index, n_patches)
        ctx.save_for_backward(src, img_index, order)
        ctx.fshape = feats.shape
        ctx.n_patches = n_patches
        ctx.embed_grad = embed_grad                         # view of the flat gradient buffer when embed_tokens trains
        return out

    @staticmethod
    def backward(ctx, d):
        src, img_index, order = ctx.saved_tensors
        dfeats = torch.zeros(ctx.fshape, dtype=d.dtype, device=d.device)
        B, T = src.shape
        d = _c(d)
        call("lmod_splice_embed_bwd", ptr(d), ptr(src), ptr(img_index), B * T, d.shape[-1], ctx.n_patches, ptr(dfeats))
        if ctx.embed_grad is not None:
            embed_grad_(d, src, order, ctx.embed_grad)
        return dfeats, None, None, None, None, None, None


def embed_grad_(dout, src, order, grad):
    """grad[t] = bf16(grad[t] + bf16(sum of the rows of dout whose src is t)) (lmod_embed_grad); order from llava_arch.embed_grad_order."""
    H = grad.shape[-1]
    call("lmod_embed_grad", ptr(_c(dout)), ptr(_c(src)), ptr(_c(order)), src.numel(), H, ptr(grad))
    return grad


def splice_embed(feats, embed_w, src, img_index, n_patches, embed_grad=None, order=None):
    """order (the rows grouped by token, llava_arch.embed_grad_order) is required with embed_grad."""
    feats = _c(feats)
    if embed_grad is not None and order is None:
        raise ValueError("splice_embed: the embedding gradient needs the plan's row order (llava_arch.embed_grad_order)")
    if torch.is_grad_enabled() and (feats.requires_grad or embed_grad is not None):
        return SpliceFn.apply(feats, embed_w, src, img_index, n_patches, embed_grad, order)
    return _splice_embed(feats, embed_w, src, img_index, n_patches)


# ---------------------------------------------------------------------------------------------------
# MoE layer (DeepSpeed 0.9.5 MoE; call site llava_qwen1_5_moe.py:536-546, SURVEY.md Appendix A)
# ---------------------------------------------------------------------------------------------------
def moe_capacity(S, E, capacity_factor, min_capacity, k=2):
    """DeepSpeed's _capacity, ceil(S/E * cf * 2) for top-2 and ceil(S/E * cf) for top-1, raised to min_capacity, with cf as the Python
    double the user set."""
    fn = _C.lib().lmod_moe_capacity if k == 2 else _C.lib().lmod_moe_capacity_top1
    return int(fn(S, E, float(capacity_factor), int(min_capacity)))


def _check_k(k):
    if k not in (1, 2):
        raise ValueError("Only top-1 and top-2 gatings are supported (k = %r)" % (k,))


LAYOUT_COMPACT, LAYOUT_SLABS, LAYOUT_ALIGNED = 0, 1, 2


def moe_route_scatter(x, wg, noise, capacity_factor, min_capacity, layout=LAYOUT_ALIGNED, padded=None, k=2):
    """Two ordinary launches (gate, seat+scatter): fp32 gate GEMV, softmax, top-1 / Gumbel top-2, stable capacity positions,
    renormalised weights, l_aux, expert offsets and the token scatter.  Returns a dict of device tensors.
    layout: 0 compact rows, 1 capacity-padded [E,C] slabs, 2 compact with 128-row aligned groups (grouped GEMM input).
    k = 1: top1gating with random token selection, noise being the uniform [S,E] in [0, 1); a selection launch runs between the two
    (the C routed tokens with the largest uniform keep their seat), w[:,0] is the raw gate and the second choice is empty (-1 / 0)."""
    _need_cuda(x, wg, noise)
    _check_k(k)
    if padded is not None:
        layout = LAYOUT_SLABS if padded else LAYOUT_COMPACT
    S, H = x.shape
    E = wg.shape[0]
    if k == 1 and S < min_capacity:
        raise ValueError("top-1 routing of %d tokens with min_capacity %d: top1gating requires at least min_capacity tokens" % (S, min_capacity))
    C = moe_capacity(S, E, capacity_factor, min_capacity, k)
    if k == 1 and C > S:
        raise ValueError("top-1 routing of %d tokens: capacity %d exceeds the token count (top1gating's topk over the tokens needs C <= S)"
                         % (S, C))
    dev = x.device
    r = dict(
        logits=torch.empty(S, E, dtype=torch.float32, device=dev), gates=torch.empty(S, E, dtype=torch.float32, device=dev),
        idx=torch.empty(S, 2, dtype=torch.int32, device=dev), row=torch.empty(S, 2, dtype=torch.int32, device=dev),
        w=torch.empty(S, 2, dtype=torch.float32, device=dev), offsets=torch.empty(E + 1, dtype=torch.int32, device=dev),
        meta=torch.empty(4 + E, dtype=torch.float32, device=dev), capacity=C)
    rows = E * C if layout == LAYOUT_SLABS else (min(k * S, E * C) + (128 * E if layout == LAYOUT_ALIGNED else 0))
    r["max_rows"] = rows
    r["k"] = k
    r["xp"] = torch.empty(rows, H, dtype=x.dtype, device=dev)      # the op zeroes the padding rows itself (inert for the wgrad reduction)
    top1 = "_top1" if k == 1 else ""
    ws = torch.empty(int(getattr(_C.lib(), "lmod_moe_route%s_ws_elems" % top1)(S, E)), dtype=torch.int32, device=dev)   # per call
    call("lmod_moe_route_scatter" + top1, ptr(x), ptr(wg), ptr(noise), S, H, E, float(capacity_factor), int(min_capacity), int(layout),
         ptr(r["logits"]), ptr(r["gates"]), ptr(r["idx"]), ptr(r["row"]), ptr(r["w"]), ptr(r["offsets"]), ptr(r["meta"]), ptr(r["xp"]),
         ptr(ws))
    return r


def moe_gather_combine(y, row, w, residual=None):
    S = row.shape[0]
    H = y.shape[-1]
    out = torch.empty(S, H, dtype=y.dtype, device=y.device)
    call("lmod_moe_gather_combine", ptr(y), ptr(row), ptr(w), ptr(residual), S, H, ptr(out))
    return out


def moe_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, min_cap, k=2):
    """The MoE forward as MoEFn runs it, returning every intermediate (the router's record, xp, h1, act, y, out).  k: routing width (1: noise
    is the uniform of top-1's selection)."""
    E, I2, H = w_gu.shape
    r = moe_route_scatter(x, wg, noise, cf, min_cap, LAYOUT_ALIGNED, k=k)
    R = r["max_rows"]
    xp, offs = r["xp"], r["offsets"]
    # only xp (and dy in the backward) are zero-filled: in the 128-aligned layout the grouped GEMM writes EVERY row below offsets[E],
    # so the padding rows of h1 / act / y come out as exact zeros (0 @ W); rows past offsets[E] are never read by a GEMM
    h1 = torch.empty(R, I2, dtype=x.dtype, device=x.device)
    grouped_gemm(xp, w_gu, h1, offs, 0)                                # [R,2I] = xp @ w_gu[e]^T
    act = silu_mul(h1)                                                 # [R,I]
    y = torch.empty(R, H, dtype=x.dtype, device=x.device)
    grouped_gemm(act, w_dn, y, offs, 0)                                # [R,H] = act @ w_dn[e]^T
    r.update(h1=h1, act=act, y=y, out=moe_gather_combine(y, r["row"], r["w"], res))
    return r


def moe_backward_stages(st, x, wg, w_gu, w_dn, dout, dlaux, grads, dres=None):
    """The MoE backward as MoEFn runs it, from moe_forward_stages' record; returns every intermediate (dy, dw, dact, dh1, dxp, dlogits,
    dx).  Weight gradients accumulate in place into grads['wg'|'w_gu'|'w_dn'] (None or a missing key = frozen).
    dres: another addend of dx [S,H], summed in the scatter-backward kernel."""
    E, I2, H = w_gu.shape
    xp, h1, act, y, row, w, gates, idx, meta, offs = (st[k] for k in ("xp", "h1", "act", "y", "row", "w", "gates", "idx", "meta", "offsets"))
    R = xp.shape[0]
    S = x.shape[0]
    dy = torch.zeros(R, H, dtype=dout.dtype, device=dout.device)
    dw = torch.empty(S, 2, dtype=torch.float32, device=dout.device)
    call("lmod_moe_combine_bwd", ptr(dout), ptr(y), ptr(row), ptr(w), S, H, ptr(dy), ptr(dw))
    g = grads
    dact = torch.empty(R, I2 // 2, dtype=dout.dtype, device=dout.device)
    grouped_gemm(dy, w_dn, dact, offs, 1)                              # dact = dy @ w_dn[e]
    dh1 = silu_mul_bwd(dact, h1)
    out = dict(dy=dy, dw=dw, dact=dact)
    if g is not None and g.get("w_dn") is not None:
        grouped_gemm(dy, act, g["w_dn"], offs, 2, accumulate=True)      # dW_dn[e] += dy_e^T @ act_e
    dxp = torch.empty(R, H, dtype=dout.dtype, device=dout.device)
    grouped_gemm(dh1, w_gu, dxp, offs, 1)                              # dxp = dh1 @ w_gu[e]
    if g is not None and g.get("w_gu") is not None:
        grouped_gemm(dh1, xp, g["w_gu"], offs, 2, accumulate=True)      # dW_gu[e] += dh1_e^T @ xp_e
    dlogits = torch.empty(S, E, dtype=torch.float32, device=dout.device)
    gl = None
    if dlaux is not None:
        gl = dlaux.to(torch.float32).reshape(1).contiguous()
    call("lmod_moe_gate_bwd_top1" if st.get("k", 2) == 1 else "lmod_moe_gate_bwd", ptr(gates), ptr(idx), ptr(row), ptr(dw), ptr(meta),
         ptr(gl), S, E, ptr(dlogits))
    dx = torch.empty_like(x)
    call("lmod_moe_scatter_bwd", ptr(dxp), ptr(row), ptr(dlogits), ptr(wg), ptr(dres), S, H, E, ptr(dx))
    if g is not None and g.get("wg") is not None:
        ws = torch.empty(32, E, H, dtype=torch.float32, device=dout.device)
        call("lmod_moe_wg_grad", ptr(x), ptr(dlogits), S, H, E, ptr(ws), ptr(g["wg"]))
    out.update(dh1=dh1, dxp=dxp, dlogits=dlogits, dx=dx)
    return out


class MoEFn(Function):
    """x: post-attention-layernorm hidden [S,H]; res: residual stream [S,H].  Experts are SwiGLU MLPs with fused gate|up weights
    w_gu [E,2I,H] and w_dn [E,H,I].  Expert GEMMs run as ONE grouped wgmma GEMM each over COMPACT expert rows (no capacity
    padding; the reference computes E*C = 1.5x the routed rows).  Returns (res + moe_out, l_aux)."""

    @staticmethod
    def forward(ctx, x, res, wg, w_gu, w_dn, noise, cf, min_cap, grads, k=2):
        x = _c(x)
        res = _c(res)
        st = moe_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, min_cap, k)
        ctx.save_for_backward(x, wg, w_gu, w_dn, *(st[n] for n in _MOE_SAVED))
        ctx.k = k
        ctx.grads = grads
        return st["out"], st["meta"][0].clone()

    @staticmethod
    def backward(ctx, dout, dlaux):
        x, wg, w_gu, w_dn, *saved = ctx.saved_tensors
        st = dict(zip(_MOE_SAVED, saved), k=ctx.k)
        dx = moe_backward_stages(st, x, wg, w_gu, w_dn, _c(dout), dlaux, ctx.grads)["dx"]
        return dx, dout, None, None, None, None, None, None, None, None


_MOE_SAVED = ("xp", "h1", "act", "y", "row", "w", "gates", "idx", "meta", "offsets")


def moe_forward_nograd(x, res, wg, w_gu, w_dn, noise, cf, min_cap, k=2):
    E, I2, H = w_gu.shape
    r = moe_route_scatter(_c(x), wg, noise, cf, min_cap, LAYOUT_ALIGNED, k=k)
    R = r["max_rows"]
    if swiglu_fusable(I2 // 2, H):
        act = grouped_gemm_swiglu(r["xp"], w_gu, r["offsets"], R)
    else:
        h1 = torch.empty(R, I2, dtype=x.dtype, device=x.device)
        grouped_gemm(r["xp"], w_gu, h1, r["offsets"], 0)
        act = silu_mul(h1)
    y = torch.empty(R, H, dtype=x.dtype, device=x.device)
    grouped_gemm(act, w_dn, y, r["offsets"], 0)
    return moe_gather_combine(y, r["row"], r["w"], _c(res)), r["meta"][0].clone(), r


# ---- Residual-MoE (DeepSpeed MoE(use_residual=True), SURVEY.md Appendix A "Residual"): the routed output and the dense MLP on every token,
# mixed per token by softmax(coefficient(x)) [S,2] (csrc/moe.cu lmod_moe_residual_mix / _bwd); the routed part runs with no residual.
def moe_residual_mix(x, moe, mlp_out, res, wc, bc):
    """-> (bf16(res + bf16(bf16(moe*c0) + bf16(mlp*c1))) [S,H], coef [S,2] bf16), c = bf16(softmax(bf16(x Wc^T + bc)))."""
    _need_cuda(x, moe, mlp_out, res, wc)
    S, H = x.shape
    out = torch.empty(S, H, dtype=x.dtype, device=x.device)
    coef = torch.empty(S, 2, dtype=x.dtype, device=x.device)
    call("lmod_moe_residual_mix", ptr(x), ptr(moe), ptr(mlp_out), ptr(_c(res)), ptr(wc), ptr(bc), S, H, ptr(out), ptr(coef))
    return out, coef


def moe_residual_mix_bwd(g, x, moe, mlp_out, coef, wc, dwc=None, dbc=None):
    """Backward of moe_residual_mix for upstream g: returns dict(d_moe, d_mlp [S,H] bf16, dz [S,2] fp32, dx [S,H] bf16 = the
    coefficient's term of dx, which callers accumulate the other addends onto).  dwc / dbc: gradient views accumulated in place
    (deterministic two-stage reduction); None = frozen."""
    S, H = g.shape
    dev = g.device
    d = dict(d_moe=torch.empty(S, H, dtype=g.dtype, device=dev), d_mlp=torch.empty(S, H, dtype=g.dtype, device=dev),
             dz=torch.empty(S, 2, dtype=torch.float32, device=dev), dx=torch.empty(S, H, dtype=g.dtype, device=dev))
    ws = None
    if dwc is not None or dbc is not None:
        ws = torch.empty(int(_C.lib().lmod_moe_residual_ws_elems(H)), dtype=torch.float32, device=dev)
    call("lmod_moe_residual_mix_bwd", ptr(g), ptr(x), ptr(moe), ptr(mlp_out), ptr(coef), ptr(wc), S, H, ptr(d["d_moe"]), ptr(d["d_mlp"]),
         ptr(d["dz"]), ptr(d["dx"]), ptr(ws), ptr(dwc), ptr(dbc))
    return d


def moe_residual_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, min_cap, r_gu, r_dn, wc, bc, k=2):
    """The Residual-MoE forward as ResidualMoEFn runs it: moe_forward_stages with no residual (its 'out' is kept as 'moe'), the dense
    SwiGLU MLP (r_gu [2I,H], r_dn [H,I]; pre-activations kept) and the mix.  Returns every intermediate; 'out' is the new stream."""
    st = moe_forward_stages(x, None, wg, w_gu, w_dn, noise, cf, min_cap, k)
    m_h1 = gemm(x, r_gu)
    m_act = silu_mul(m_h1)
    m_y = gemm(m_act, r_dn)
    out, coef = moe_residual_mix(x, st["out"], m_y, res, wc, bc)
    st.update(moe=st["out"], mlp_h1=m_h1, mlp_act=m_act, mlp=m_y, coef=coef, out=out)
    return st


def moe_residual_backward_stages(st, x, wg, w_gu, w_dn, r_gu, r_dn, wc, dout, dlaux, grads):
    """Backward of moe_residual_forward_stages.  The mix backward splits dout into the routed and dense branches and writes the
    coefficient's dx term; the dense dgrad GEMM accumulates onto that term, and the routed scatter-backward adds the sum (its dres), so dx
    takes no extra pass.  grads: the keys of moe_backward_stages plus 'r_gu', 'r_dn', 'wc', 'bc' (None or missing = frozen)."""
    g = grads or {}
    mix = moe_residual_mix_bwd(dout, x, st["moe"], st["mlp"], st["coef"], wc, g.get("wc"), g.get("bc"))
    d_mlp = mix["d_mlp"]
    m_dh1 = silu_mul_bwd(mm_nn(d_mlp, r_dn), st["mlp_h1"])
    if g.get("r_dn") is not None:
        mm_tn_acc(d_mlp, st["mlp_act"], g["r_dn"])
    dres = mix["dx"]
    gemm(m_dh1, r_gu, b_mn=True, out=dres, accumulate=True)            # dx_coef + dh1 @ W_gu
    if g.get("r_gu") is not None:
        mm_tn_acc(m_dh1, x, g["r_gu"])
    out = moe_backward_stages(st, x, wg, w_gu, w_dn, mix["d_moe"], dlaux, g, dres=dres)
    out.update(mix=mix, mlp_dh1=m_dh1, dres=dres)
    return out


class ResidualMoEFn(Function):
    """MoEFn with DeepSpeed's use_residual=True: (res + bf16(moe*c0) + bf16(mlp*c1), l_aux), the dense MLP r_gu / r_dn (the module the
    experts were up-cycled from) run on every token, c = softmax(coefficient(x)).  grads: MoEFn's keys plus 'r_gu', 'r_dn', 'wc', 'bc'."""

    @staticmethod
    def forward(ctx, x, res, wg, w_gu, w_dn, noise, cf, min_cap, r_gu, r_dn, wc, bc, grads, k=2):
        x = _c(x)
        res = _c(res)
        st = moe_residual_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, min_cap, r_gu, r_dn, wc, bc, k)
        ctx.save_for_backward(x, wg, w_gu, w_dn, r_gu, r_dn, wc, *(st[n] for n in _MOE_SAVED + _RES_SAVED))
        ctx.k = k
        ctx.grads = grads
        return st["out"], st["meta"][0].clone()

    @staticmethod
    def backward(ctx, dout, dlaux):
        x, wg, w_gu, w_dn, r_gu, r_dn, wc, *saved = ctx.saved_tensors
        st = dict(zip(_MOE_SAVED + _RES_SAVED, saved), k=ctx.k)
        dx = moe_residual_backward_stages(st, x, wg, w_gu, w_dn, r_gu, r_dn, wc, _c(dout), dlaux, ctx.grads)["dx"]
        return (dx, dout) + (None,) * 12


_RES_SAVED = ("moe", "mlp_h1", "mlp_act", "mlp", "coef")


def moe_residual_forward_nograd(x, res, wg, w_gu, w_dn, noise, cf, min_cap, r_gu, r_dn, wc, bc, k=2):
    """moe_forward_nograd with use_residual=True -> (new stream, l_aux, routing record with 'coef')."""
    x = _c(x)
    moe, l_aux, r = moe_forward_nograd(x, None, wg, w_gu, w_dn, noise, cf, min_cap, k)
    out, coef = moe_residual_mix(x, moe, mlp(x, r_gu, r_dn), res, wc, bc)
    r["coef"] = coef
    return out, l_aux, r


# ---------------------------------------------------------------------------------------------------
# activation checkpointing of one decoder layer (HF gradient checkpointing, modeling_qwen2.py:1062-1072)
# ---------------------------------------------------------------------------------------------------
_ANCHOR = torch.empty(0, requires_grad=True)


class CheckpointFn(Function):
    """One decoder layer as a checkpointed segment.  run(*inputs) -> tuple of output tensors runs the layer on the Functions above; it
    must draw no random numbers (the caller draws the router noise before the segment and binds it into run).
    Forward: run under autograd on detached copies of the inputs, so the very kernels of the un-checkpointed layer run (grad forms
    included), then drop that graph: only the inputs are kept.  Backward: run again -- the same kernels on the same bytes give the same
    bytes -- and back-propagate the incoming gradients through it; parameter gradients accumulate into their arena views as in the plain
    layer.  anchor: a tensor that requires grad, so the segment of a trainable layer whose inputs do not require grad still gets a
    backward (what enable_input_require_grads works around in the reference)."""

    @staticmethod
    def forward(ctx, run, anchor, *inputs):
        ctx.run = run
        ctx.save_for_backward(*inputs)
        with torch.enable_grad():
            outs = run(*_ckpt_inputs(inputs, ctx.needs_input_grad[2:]))
        return tuple(o.detach() for o in outs)

    @staticmethod
    def backward(ctx, *grads):
        xs = _ckpt_inputs(ctx.saved_tensors, ctx.needs_input_grad[2:])
        with torch.enable_grad():
            outs = ctx.run(*xs)
        pairs = [(o, g) for o, g in zip(outs, grads) if o.requires_grad and g is not None]
        if pairs:
            torch.autograd.backward([o for o, _ in pairs], [g for _, g in pairs])
        return (None, None) + tuple(x.grad if x.requires_grad else None for x in xs)


def _ckpt_inputs(inputs, needs):
    return [t.detach().requires_grad_(n) for t, n in zip(inputs, needs)]


def checkpoint(run, *inputs):
    """CheckpointFn on the segment inputs -> run's outputs, none of run's intermediates kept."""
    return CheckpointFn.apply(run, _ANCHOR, *inputs)


# ---------------------------------------------------------------------------------------------------
# fused lm_head + mimic-KL (+ shifted CE) loss head
# ---------------------------------------------------------------------------------------------------
# optional per-kernel device timing (bench.py roofline): name -> list of (start_event, end_event) on the launching stream
TIMERS = None


class _Timed:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if TIMERS is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.a.record()

    def __exit__(self, *exc):
        if TIMERS is not None:
            self.b.record()
            TIMERS.setdefault(self.name, []).append((self.a, self.b))


def kl_fused(s_logits, t_logits, labels, seq_len, vocab, w_kd, w_ce, distill_all=False, dlogits=None, rows=None):
    """Raw kernel call.  s_logits/t_logits [N,ld] bf16, labels [N] int64.  Returns (out4, row_out).
    out4 = {align_loss, ce_loss, n_kd, n_ce}.  dlogits (may alias s_logits) receives the gradient.
    rows = (perm, count) from active_rows(): the logits buffers hold only the active rows, compacted."""
    _need_cuda(s_logits, t_logits, labels)
    N = labels.numel()
    dev = s_logits.device
    counts = torch.empty(2, dtype=torch.float32, device=dev)
    row_out = torch.empty(N, 4, dtype=torch.float32, device=dev)
    out4 = torch.empty(4, dtype=torch.float32, device=dev)
    da = 1 if distill_all else 0
    perm, count = rows if rows is not None else (None, None)
    call("lmod_kl_counts", ptr(labels), N, seq_len, da, ptr(counts))
    with _Timed("kl_fwd_bwd"):
        call("lmod_kl_fwd_bwd_rows", ptr(s_logits), s_logits.stride(0), ptr(t_logits), t_logits.stride(0), ptr(labels), N, seq_len, vocab, da,
             float(w_kd), float(w_ce), ptr(counts), ptr(row_out), ptr(dlogits), dlogits.stride(0) if dlogits is not None else 0,
             ptr(perm), ptr(count))
    call("lmod_kl_finalize", ptr(row_out), ptr(labels), N, seq_len, da, ptr(out4))
    return out4, row_out


class DistillHeadFn(Function):
    """lm_head GEMM (llava_qwen1_5_moe.py:407-408) + get_logp / compute_align_loss against the teacher's logits
    (align_trainer.py:497-528) + the model's shifted CE (llava_qwen1_5_moe.py:413-421), forward and backward in one
    sweep over the vocabulary.  Returns (w_kd*align + w_ce*ce, align, ce); only the first is differentiable."""

    @staticmethod
    def forward(ctx, hidden, w_head, t_logits, labels, seq_len, vocab, w_kd, w_ce, distill_all, head_grad, perm, count):
        h2 = _c(hidden).reshape(-1, hidden.shape[-1])
        rows = (perm, count) if perm is not None else None
        if rows is not None:
            h2 = gather_rows(h2, perm, count)                             # active rows only; t_logits is compact the same way
        logits = gemm(h2, w_head, m_dev=count)                            # [N(+pad), Vs] bf16
        if logits.shape[1] != vocab and w_ce != 0.0:
            raise _C.LmodError("fused CE needs student vocab == kd vocab slice")
        out4, _ = kl_fused(logits, t_logits, labels.reshape(-1), seq_len, vocab, w_kd, w_ce, distill_all, dlogits=logits, rows=rows)
        if logits.shape[1] > vocab:
            logits[:, vocab:].zero_()
        ctx.save_for_backward(logits, w_head, h2, perm, count)
        ctx.hshape = hidden.shape
        ctx.head_grad = head_grad
        align, ce = out4[0], out4[1]
        total = w_kd * align + (w_ce * ce if w_ce != 0.0 else 0.0)
        ctx.mark_non_differentiable(align, ce)
        return total, align, ce

    @staticmethod
    def backward(ctx, g, _a, _c2):
        dlogits, w_head, h2, perm, count = ctx.saved_tensors
        # the kernel produced d(total)/d(logits); the upstream scalar g multiplies the two SMALL operands instead of the [N,V] / [V,H] results:
        # dH = g * (dlogits @ W),  dW += dlogits^T @ (g * h).  g is applied in fp32 and each product rounded to bf16 once: a g rounded to bf16
        # first would scale both gradients by bf16(g) / g (up to 2^-9 off 1, the same sign on every element).  At g = 1 both are exact.
        g = g.float()
        dh = (mm_nn(dlogits, w_head, m_dev=count).float() * g).to(h2.dtype)
        if perm is not None:
            n = 1
            for d in ctx.hshape[:-1]:
                n *= d
            dh = scatter_rows(dh, perm, count, n)
        dh = dh.reshape(ctx.hshape)
        if ctx.head_grad is not None:
            mm_tn_acc(dlogits, (h2.float() * g).to(h2.dtype), ctx.head_grad, k_dev=count)
        return dh, None, None, None, None, None, None, None, None, None, None, None


def distill_head(hidden, w_head, t_logits, labels, vocab, w_kd, w_ce, distill_all=False, head_grad=None, rows=None):
    """rows = (perm, count) from active_rows(labels): t_logits then holds the teacher logits of the active rows only (compact)."""
    perm, count = rows if rows is not None else (None, None)
    return DistillHeadFn.apply(hidden, w_head, t_logits, labels, labels.shape[-1], vocab, float(w_kd), float(w_ce), bool(distill_all), head_grad,
                               perm, count)


# ---------------------------------------------------------------------------------------------------
# DPO log-prob head (dpo_trainer.py:483-495)
# ---------------------------------------------------------------------------------------------------
def logp_gather(logits, labels, average=False):
    """logits [B,T,V] bf16 (contiguous), labels [B,T] int64 -> (seq_logp [B], tok_logp [B*T], lse [B*T])."""
    B, T, V = logits.shape
    dev = logits.device
    tok = torch.empty(B * T, dtype=torch.float32, device=dev)
    lse = torch.empty(B * T, dtype=torch.float32, device=dev)
    seq = torch.empty(B, dtype=torch.float32, device=dev)
    with _Timed("logp_fwd"):
        call("lmod_logp_gather_fwd", ptr(logits), logits.stride(1), ptr(labels), B, T, V, ptr(tok), ptr(lse), ptr(seq), 1 if average else 0)
    return seq, tok, lse


def logp_gather_bwd(logits, labels, lse, g_seq, out):
    """d seq_logp / d logits of logp_gather for the upstream gradient g_seq [B] fp32, written to out [B,T,V] (out may be logits)."""
    B, T, V = logits.shape
    call("lmod_logp_gather_bwd", ptr(logits), logits.stride(1), ptr(labels), B, T, V, ptr(lse), ptr(g_seq), 0, ptr(out), out.stride(1))
    return out


class LogpHeadFn(Function):
    """lm_head GEMM + DPOTrainer.get_logp; backward writes d logits in place and returns d hidden."""

    @staticmethod
    def forward(ctx, hidden, w_head, labels, head_grad):
        B, T, H = hidden.shape
        logits = mm_nt(_c(hidden).reshape(-1, H), w_head).view(B, T, -1)
        labels = _c(labels)
        seq, tok, lse = logp_gather(logits, labels)
        ctx.save_for_backward(logits, w_head, labels, lse, hidden)
        ctx.head_grad = head_grad
        return seq

    @staticmethod
    def backward(ctx, g):
        logits, w_head, labels, lse, hidden = ctx.saved_tensors
        B, T, V = logits.shape
        g = _c(g.to(torch.float32))
        with _Timed("logp_bwd"):
            logp_gather_bwd(logits, labels, lse, g, logits)
        d2 = logits.view(B * T, V)
        dh = mm_nn(d2, w_head).view(hidden.shape)
        if ctx.head_grad is not None:
            mm_tn_acc(d2, hidden.reshape(B * T, -1), ctx.head_grad)
        return dh, None, None, None


def logp_head(hidden, w_head, labels, head_grad=None):
    return LogpHeadFn.apply(hidden, w_head, labels, head_grad)


# ---------------------------------------------------------------------------------------------------
# API-compat materialising forms (AlignTrainer.get_p / get_logp / compute_align_loss signatures)
# ---------------------------------------------------------------------------------------------------
def softmax_rows(logits_bf16, vocab, log_mode):
    x = _c(logits_bf16)
    V = x.shape[-1]
    n = x.numel() // V
    out = torch.empty(x.shape[:-1] + (vocab,), dtype=torch.float32, device=x.device)
    call("lmod_softmax_rows", ptr(x), V, n, vocab, 1 if log_mode else 0, ptr(out), vocab)
    return out


def align_loss_dense(logp, probs, labels, distill_all=False):
    V = logp.shape[-1]
    n = logp.numel() // V
    row_x = torch.empty(n, dtype=torch.float32, device=logp.device)
    out = torch.empty(1, dtype=torch.float32, device=logp.device)
    call("lmod_align_loss_dense", ptr(_c(logp)), ptr(_c(probs)), V, ptr(_c(labels)), n, V, 1 if distill_all else 0, ptr(row_x), ptr(out))
    return out[0]


# ---------------------------------------------------------------------------------------------------
# optimizer
# ---------------------------------------------------------------------------------------------------
ADAMW8_BLOCK = 2048          # elements per absmax of the 8-bit state (A8_BLOCK in csrc/optim.cu)


def sumsq_(buf, out):
    call("lmod_sumsq", ptr(buf), 1 if buf.dtype == torch.float32 else 0, buf.numel(), ptr(out))


def adamw_(master, m, v, grad, model, lr, beta1, beta2, eps, wd, step, gnorm_sq=None, max_norm=0.0, grad_scale=1.0):
    call("lmod_adamw", ptr(master), ptr(m), ptr(v), ptr(grad), 1 if grad.dtype == torch.float32 else 0,
         ptr(model), master.numel(), float(lr), float(beta1), float(beta2), float(eps), float(wd),
         int(step), ptr(gnorm_sq), float(max_norm), float(grad_scale))


def adamw_8bit_(master, m8, v8, absmax_m, absmax_v, grad, model, lr, beta1, beta2, eps, wd, step, gnorm_sq=None, max_norm=0.0,
                grad_scale=1.0):
    """adamw_ with 8-bit block-wise moments (``--optim adamw_bnb_8bit``): codes ``m8`` / ``v8`` [n] uint8, scales ``absmax_m`` /
    ``absmax_v`` [ceil(n / 2048)] fp32, ``grad`` bf16."""
    _need_cuda(master, m8, v8, absmax_m, absmax_v, grad, model)
    if grad.dtype != BF16 or m8.dtype != torch.uint8 or v8.dtype != torch.uint8 or absmax_m.dtype != torch.float32 \
            or absmax_v.dtype != torch.float32:
        raise _C.LmodError("adamw_8bit_: bf16 gradient, uint8 codes and fp32 scales expected")
    n = master.numel()
    nb = (n + ADAMW8_BLOCK - 1) // ADAMW8_BLOCK
    if not (m8.numel() == v8.numel() == grad.numel() == n and absmax_m.numel() == absmax_v.numel() == nb
            and (model is None or model.numel() == n)):
        raise _C.LmodError("adamw_8bit_: %d elements need %d codes per moment and %d scales per moment" % (n, n, nb))
    call("lmod_adamw_8bit", ptr(master), ptr(m8), ptr(v8), ptr(absmax_m), ptr(absmax_v), ptr(grad), ptr(model),
         n, float(lr), float(beta1), float(beta2), float(eps), float(wd), int(step), ptr(gnorm_sq),
         float(max_norm), float(grad_scale))
