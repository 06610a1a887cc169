"""Torch-facing wrappers (``torch.autograd.Function``) around the C ABI of liblmod_b200.so.

Each wrapper cites the reference call site it stands in for.  Tensors are bf16 CUDA, contiguous; fp32 only
where the reference keeps fp32 (router gate, loss scalars, optimizer state).  No CPU fallback.
"""
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
    return t if t.is_contiguous() else t.contiguous()


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
        out = torch.zeros(M, Kout, dtype=dy.dtype, device=dy.device)         # rows past the dynamic extent stay zero
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
    call("lmod_gather_rows", ptr(x2), x2.stride(0), ptr(perm) if perm is not None else None, ptr(count), out.shape[0], h, ROW_PAD,
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
    dyn = (ptr(m_dev) if m_dev is not None else None, ptr(k_dev) if k_dev is not None else None)
    if out_f32 is not None:
        call("lmod_gemm_bf16_dyn", ptr(a), a.stride(0), int(a_mn), ptr(b), b.stride(0), int(b_mn), None, out_f32.stride(0), M, N, K, None,
             (int(split_k) << 8) if split_k > 1 else 0, ptr(out_f32), *dyn)
        return out_f32
    if out is None:
        out = torch.empty(M, N, dtype=a.dtype, device=a.device)
    call("lmod_gemm_bf16_dyn", ptr(a), a.stride(0), int(a_mn), ptr(b), b.stride(0), int(b_mn), ptr(out), out.stride(0), M, N, K,
         ptr(bias) if bias is not None else None, 1 if accumulate else 0, None, *dyn)
    return out


# Epilogue fusions pay off only when the GEMM's main loop is long enough to hide them: the fused SwiGLU forward is used from a reduction
# length of FUSE_MIN_K on (the teacher's K = 4096); at the student's K = 1024 the element-wise kernels, which use every warp of the SM,
# are preferred.  The (lighter) RoPE epilogue of the q|k|v projection is always fused.  LLAVAMOD_FUSE_SWIGLU: "auto" (by
# reduction length), "1" always, "0" never; LLAVAMOD_FUSE_ROPE: "0" = GEMM + lmod_rope.  Measured again with asynchronous MMAs
# (DESIGN.md section 4): "1" is within the step's run-to-run spread of "auto".
FUSE_SWIGLU = _os.environ.get("LLAVAMOD_FUSE_SWIGLU", "auto")
FUSE_ROPE = _os.environ.get("LLAVAMOD_FUSE_ROPE", "auto")
# residual add in the o_proj / down_proj (CLIP: out_proj / fc2) epilogue of no-grad forwards.  Bit-identical to the add inside the next norm's
# kernel; opt-in: the add is cheap inside the norm kernel, and the fused form measures within the step's spread (DESIGN.md section 4)
FUSE_RESIDUAL = _os.environ.get("LLAVAMOD_FUSE_RESIDUAL", "0")
FUSE_MIN_K = 2048


def _fuse(mode, K):
    return mode == "1" or (mode == "auto" and K >= FUSE_MIN_K)


def swiglu_fusable(I, K=None, training=False):
    """The fused SwiGLU GEMM tiles the intermediate dimension by 128 (the reference's tiny test shapes with I = 320 take GEMM + silu_mul);
    training keeps the pre-activations, which makes the epilogue heavier still: fused only on request."""
    if I % 128 != 0:
        return False
    if K is None:
        return True
    if training:
        return FUSE_SWIGLU == "1"
    return _fuse(FUSE_SWIGLU, K)


def gemm_swiglu(x2, w_gu, save_h1):
    """act[M,I] (, h1[M,2I]) = SwiGLU(x2 @ w_gu^T) in ONE GEMM (lmod_gemm_swiglu): w_gu is the fused gate|up weight [2I,H] as stored."""
    _need_cuda(x2, w_gu)
    M, H = x2.shape
    I = w_gu.shape[0] // 2
    act = torch.empty(M, I, dtype=x2.dtype, device=x2.device)
    h1 = torch.empty(M, 2 * I, dtype=x2.dtype, device=x2.device) if save_h1 else None
    call("lmod_gemm_swiglu", ptr(x2), x2.stride(0), ptr(w_gu), w_gu.stride(0), ptr(act), I, ptr(h1), 2 * I, M, I, H)
    return act, h1


def gemm_silu_bwd(dy2, w_dn, h1):
    """dh1[M,2I] = silu_mul_bwd(dy2 @ w_dn, h1) in the epilogue of the down_proj dgrad (lmod_gemm_silu_bwd); w_dn [H,I] as stored."""
    M, H = dy2.shape
    I = w_dn.shape[1]
    dh1 = torch.empty(M, 2 * I, dtype=dy2.dtype, device=dy2.device)
    call("lmod_gemm_silu_bwd", ptr(dy2), dy2.stride(0), ptr(w_dn), w_dn.stride(0), ptr(h1), h1.stride(0), ptr(dh1), 2 * I, M, I, H)
    return dh1


def grouped_gemm_swiglu(xp, w_gu, offsets, max_rows, save_h1):
    """Experts' gate|up + SwiGLU on compact expert rows: w_gu [E,2I,H]; returns (act [R,I], h1 [R,2I] or None)."""
    E, I2, H = w_gu.shape
    I = I2 // 2
    act = torch.empty(max_rows, I, dtype=xp.dtype, device=xp.device)
    h1 = torch.empty(max_rows, I2, dtype=xp.dtype, device=xp.device) if save_h1 else None
    call("lmod_grouped_gemm_swiglu", ptr(xp), xp.stride(0), ptr(w_gu), w_gu.stride(1), ptr(act), I, ptr(h1), I2, ptr(offsets), E, max_rows, I, H)
    return act, h1


def grouped_gemm_silu_bwd(dy, w_dn, h1, offsets, max_rows):
    """dh1 [R,2I] = silu_mul_bwd(dy @ w_dn[e], h1) per expert group; w_dn [E,H,I]."""
    E, H, I = w_dn.shape
    dh1 = torch.empty(max_rows, 2 * I, dtype=dy.dtype, device=dy.device)
    call("lmod_grouped_gemm_silu_bwd", ptr(dy), dy.stride(0), ptr(w_dn), w_dn.stride(1), ptr(h1), h1.stride(0), ptr(dh1), 2 * I, ptr(offsets), E,
         max_rows, I, H)
    return dh1


class MLPFn(Function):
    """Qwen2MLP (modeling_qwen2.py:188-200) as two GEMMs: gate|up with the SwiGLU epilogue (pre-activations kept for the backward), then
    down_proj.  Backward: the down_proj dgrad GEMM turns dY straight into d(gate)|d(up) in its epilogue; wgrads accumulate in place into
    the flat gradient buffer views ``g_gu`` / ``g_dn`` (None = frozen)."""

    @staticmethod
    def forward(ctx, x, w_gu, w_dn, g_gu, g_dn):
        x2 = _rows(x)
        act, h1 = gemm_swiglu(x2, w_gu, True)
        y = gemm(act, w_dn)
        ctx.save_for_backward(x2, w_gu, w_dn, h1, act)
        ctx.g = (g_gu, g_dn)
        ctx.xshape = x.shape
        return y.view(*x.shape[:-1], w_dn.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w_gu, w_dn, h1, act = ctx.saved_tensors
        g_gu, g_dn = ctx.g
        dy2 = _c(dy).reshape(-1, dy.shape[-1])
        dh1 = gemm_silu_bwd(dy2, w_dn, h1)
        if g_dn is not None:
            mm_tn_acc(dy2, act, g_dn)
        dx = mm_nn(dh1, w_gu).reshape(ctx.xshape) if ctx.needs_input_grad[0] else None
        if g_gu is not None:
            mm_tn_acc(dh1, x2, g_gu)
        return dx, None, None, None, None


def mlp(x, w_gu, w_dn, g_gu=None, g_dn=None, res=None):
    """Dense SwiGLU MLP.  Fused SwiGLU epilogues whenever the intermediate size allows; frozen / no-grad calls keep nothing.
    res (no-grad calls only, see residual_fusable): the residual stream, added in the down_proj epilogue -- the return value is the new stream."""
    I = w_gu.shape[0] // 2
    grad = torch.is_grad_enabled() and (x.requires_grad or g_gu is not None or g_dn is not None)
    assert res is None or not grad
    if swiglu_fusable(I, w_gu.shape[1], training=grad):
        if grad:
            return MLPFn.apply(x, w_gu, w_dn, g_gu, g_dn)
        act, _ = gemm_swiglu(_rows(x), w_gu, False)
        if res is not None:
            return gemm_residual(act, w_dn, None, res)
        y = gemm(act, w_dn)
        return y if x.dim() == 2 else y.view(*x.shape[:-1], w_dn.shape[0])
    gu = linear(x, w_gu, None, g_gu, None)
    if res is not None:
        return gemm_residual(silu_mul(gu), w_dn, None, res)
    return linear(silu_mul(gu), w_dn, None, g_dn, None)


def grouped_gemm(a, b, out, offsets, mode, max_rows=None, accumulate=False):
    """lmod_grouped_gemm_bf16 on compact expert rows (offsets [G+1] int32 on device, 128-aligned).
       mode 0: out[R,N] = a[R,K] @ b[G,N,K]^T ; mode 1: out[R,N] = a[R,K] @ b[G,K,N] ; mode 2: out[G,M,N] (+)= a[R,M]^T @ b[R,N] per group."""
    G = offsets.numel() - 1
    R = a.shape[0] if max_rows is None else max_rows
    if mode == 0:
        N, K = b.shape[1], b.shape[2]
        call("lmod_grouped_gemm_bf16", ptr(a), a.stride(0), ptr(b), b.stride(1), ptr(out), out.stride(0), ptr(offsets), G, R, 0, N, K, 0, 0)
    elif mode == 1:
        K, N = b.shape[1], b.shape[2]
        call("lmod_grouped_gemm_bf16", ptr(a), a.stride(0), ptr(b), b.stride(1), ptr(out), out.stride(0), ptr(offsets), G, R, 0, N, K, 1, 0)
    else:
        M, N = a.shape[1], b.shape[1]
        call("lmod_grouped_gemm_bf16", ptr(a), a.stride(0), ptr(b), b.stride(0), ptr(out), out.stride(1), ptr(offsets), G, R, M, N, 0, 2,
             1 if accumulate else 0)
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


def residual_fusable(x, res, *grads):
    """The projection's epilogue may add the residual stream itself when nothing of the call is differentiated (frozen teacher, CLIP tower,
    eval): the trainable students keep the add inside the next norm's kernel, whose backward needs the un-added branch anyway."""
    if FUSE_RESIDUAL != "1" or res is None:
        return False
    if not torch.is_grad_enabled():
        return True
    return not (x.requires_grad or res.requires_grad or any(g is not None for g in grads))


def gemm_residual(x, w, bias, res, inplace=False):
    """bf16( bf16(x @ w^T + bias) + res ) in one GEMM (lmod_gemm_residual): the output IS the new residual stream (inplace: written over res)."""
    _need_cuda(x, w, res)
    x2, r2 = _rows(x), _rows(res)
    M, Kd = x2.shape
    N = w.shape[0]
    out = r2 if inplace else torch.empty(M, N, dtype=x2.dtype, device=x2.device)
    call("lmod_gemm_residual", ptr(x2), x2.stride(0), ptr(w), w.stride(0), ptr(bias) if bias is not None else None, ptr(r2), r2.stride(0),
         ptr(out), out.stride(0), M, N, Kd)
    return out if res.dim() == 2 else out.view(res.shape)


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
         ptr(out), out.stride(0), ptr(lse) if lse is not None else None, ptr(lo), ptr(hi))
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
    if hd not in ATTN_HEAD_DIMS:
        hp = 64 if hd < 64 else 128
        if hd > 128:
            raise _C.LmodError("head_dim %d > 128 is not built" % hd)
        q3 = torch.nn.functional.pad(qkv.view(B * T, nh + 2 * nkv, hd), (0, hp - hd)).view(B * T, (nh + 2 * nkv) * hp)
        o = attention(q3, B, T, nh, nkv, hp, causal, scale, pad)
        return o.view(B * T, nh, hp)[:, :, :hd].reshape(B * T, nh * hd)
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


def kv_append(qkv, B, n_new, nh, nkv, hd, k_cache, v_cache, offsets):
    """DynamicCache.update: the k / v heads of the fused, RoPE'd QKV rows [B*n_new, (nh+2nkv)*hd] -> cache rows offsets[b] + [0, n_new)
    of k_cache / v_cache [B, nkv, max_len, hp] (hp = attn_head_dim(hd); padded heads get zero columns).  offsets: int32 [B] on the device."""
    _need_cuda(qkv, k_cache, v_cache, offsets)
    _check_cache(k_cache, v_cache, B, nkv, hd)
    _check_i32(offsets, B, "offsets")
    if qkv.dim() != 2 or qkv.shape[0] != B * n_new or qkv.shape[1] != (nh + 2 * nkv) * hd or qkv.stride(1) != 1:
        raise _C.LmodError("kv_append: qkv must be [B*n_new, (nh+2nkv)*hd] with unit column stride, got %s" % (tuple(qkv.shape),))
    hp = k_cache.shape[-1]
    if hp != hd:
        qkv = _pad_heads(qkv, nh + 2 * nkv, hd, hp)
    call("lmod_kv_append", ptr(qkv), qkv.stride(0), B, n_new, nh, nkv, hp, ptr(offsets), ptr(k_cache), ptr(v_cache), k_cache.shape[2])


def attn_decode_ws_elems(B, nh, nkv, hd, max_len):
    return int(_C.lib().lmod_attn_decode_ws_elems(B, nh, nkv, attn_head_dim(hd), max_len))


def attn_decode(q, nh, nkv, hd, k_cache, v_cache, lens, ws, scale=None, need_lse=False):
    """Single-query attention of every sequence over its cached keys [0, lens[b]) (split-KV, lmod_attn_decode).  q: [B, >= nh*hd] rows
    whose first nh*hd columns are the query heads (the fused QKV rows of a decode step); k_cache / v_cache [B, nkv, max_len, hp];
    lens int32 [B] on the device; ws fp32 of at least attn_decode_ws_elems(...).  -> (out [B, nh*hd] bf16, lse [B, nh] fp32 or None)."""
    _need_cuda(q, k_cache, v_cache, lens, ws)
    B = q.shape[0]
    _check_cache(k_cache, v_cache, B, nkv, hd)
    _check_i32(lens, B, "lens")
    if q.dim() != 2 or q.shape[1] < nh * hd or q.stride(1) != 1 or q.dtype != BF16:
        raise _C.LmodError("attn_decode: q must be bf16 [B, >= nh*hd] with unit column stride, got %s %s" % (q.dtype, tuple(q.shape)))
    if ws.dtype != torch.float32 or not ws.is_contiguous():
        raise _C.LmodError("attn_decode: ws must be a contiguous fp32 tensor")
    hp, max_len = k_cache.shape[-1], k_cache.shape[2]
    scale = float(scale if scale is not None else hd ** -0.5)
    if hp != hd:
        q = _pad_heads(q[:, :nh * hd], nh, hd, hp)
    out = torch.empty(B, nh * hp, dtype=q.dtype, device=q.device)
    lse = torch.empty(B, nh, dtype=torch.float32, device=q.device) if need_lse else None
    call("lmod_attn_decode", ptr(q), q.stride(0), ptr(k_cache), ptr(v_cache), ptr(lens), B, nh, nkv, hp, max_len, scale, ptr(out), out.stride(0),
         ptr(lse), ptr(ws), ws.numel())
    if hp != hd:
        out = out.view(B, nh, hp)[:, :, :hd].reshape(B, nh * hd)
    return out, lse


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
        H = x.shape[-1]
        rows = x.numel() // H
        y = torch.empty_like(x)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        if res is not None:
            res = _c(res)
            s = torch.empty_like(x)
            call("lmod_rmsnorm_fwd", ptr(x), ptr(res), ptr(w), rows, H, eps, ptr(y), ptr(s), ptr(rstd))
        else:
            s = x
            call("lmod_rmsnorm_fwd", ptr(x), None, ptr(w), rows, H, eps, ptr(y), None, ptr(rstd))
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


def rmsnorm(x, w, eps, res=None, wgrad=None):
    """-> (y, stream) where stream = x + res (or x).  Without autograd the kernel is called directly."""
    if torch.is_grad_enabled() and (x.requires_grad or (res is not None and res.requires_grad) or wgrad is not None):
        y, s = RMSNormFn.apply(x, res, w, eps, wgrad)
        return y, (s if res is not None else x)
    x = _c(x)
    H = x.shape[-1]
    rows = x.numel() // H
    y = torch.empty_like(x)
    if res is not None:
        s = torch.empty_like(x)
        call("lmod_rmsnorm_fwd", ptr(x), ptr(_c(res)), ptr(w), rows, H, eps, ptr(y), ptr(s), None)
        return y, s
    call("lmod_rmsnorm_fwd", ptr(x), None, ptr(w), rows, H, eps, ptr(y), None, None)
    return y, x


def layernorm(x, w, b, eps):
    """CLIP LayerNorm (transformers CLIPVisionModel via clip_encoder.py:54); frozen tower: forward only."""
    x = _c(x)
    H = x.shape[-1]
    y = torch.empty_like(x)
    call("lmod_layernorm_fwd", ptr(x), ptr(w), ptr(b), x.numel() // H, H, eps, ptr(y))
    return y


class RopeFn(Function):
    """apply_rotary_pos_emb (modeling_qwen2.py:159-184) in place on the fused QKV projection output
    [rows, (nh + 2*nkv)*hd]: q heads first, then k heads, then v."""

    @staticmethod
    def forward(ctx, qkv, cos, sin, pos, nh, nkv, hd):
        rows = qkv.numel() // qkv.shape[-1]
        ld = qkv.shape[-1]
        call("lmod_rope", ptr(qkv), ld, nh, qkv.data_ptr() + nh * hd * 2, ld, nkv, hd, ptr(cos), ptr(sin), ptr(pos), rows, 0)
        ctx.mark_dirty(qkv)
        ctx.save_for_backward(cos, sin, pos)
        ctx.dims = (nh, nkv, hd)
        return qkv

    @staticmethod
    def backward(ctx, d):
        cos, sin, pos = ctx.saved_tensors
        nh, nkv, hd = ctx.dims
        d = d.contiguous().clone()
        rows = d.numel() // d.shape[-1]
        ld = d.shape[-1]
        call("lmod_rope", ptr(d), ld, nh, d.data_ptr() + nh * hd * 2, ld, nkv, hd, ptr(cos), ptr(sin), ptr(pos), rows, 1)
        return d, None, None, None, None, None, None


class QKVRopeFn(Function):
    """q|k|v projection + rotary embedding (modeling_qwen2.py:678-691): ONE GEMM whose epilogue adds the bias and rotates the q / k heads
    (lmod_gemm_qkv_rope).  Backward: the transpose rotation in place on the incoming dqkv, then dgrad / wgrad / bias gradient as LinearFn."""

    @staticmethod
    def forward(ctx, x, w, bias, cos, sin, pos, nh, nkv, hd, wgrad, bgrad):
        x2 = _rows(x)
        M, Kd = x2.shape
        out = torch.empty(M, w.shape[0], dtype=x.dtype, device=x.device)
        call("lmod_gemm_qkv_rope", ptr(x2), x2.stride(0), ptr(w), w.stride(0), ptr(bias) if bias is not None else None, ptr(out), out.stride(0), M, Kd,
             nh, nkv, hd, ptr(cos), ptr(sin), ptr(pos))
        ctx.save_for_backward(x2, w, cos, sin, pos)
        ctx.dims = (nh, nkv, hd)
        ctx.g = (wgrad, bgrad)
        ctx.xshape = x.shape
        return out

    @staticmethod
    def backward(ctx, d):
        x2, w, cos, sin, pos = ctx.saved_tensors
        nh, nkv, hd = ctx.dims
        wgrad, bgrad = ctx.g
        d = _c(d)                                         # the fused dq|dk|dv buffer of the attention backward: rotated back in place
        ld = d.shape[-1]
        call("lmod_rope", ptr(d), ld, nh, d.data_ptr() + nh * hd * 2, ld, nkv, hd, ptr(cos), ptr(sin), ptr(pos), d.numel() // ld, 1)
        dx = mm_nn(d, w).reshape(ctx.xshape) if ctx.needs_input_grad[0] else None
        if wgrad is not None:
            mm_tn_acc(d, x2, wgrad)
        if bgrad is not None:
            bgrad.add_(d.sum(0).to(bgrad.dtype))
        return (dx,) + (None,) * 10


def qkv_rope(x, w, bias, cos, sin, pos, nh, nkv, hd, wgrad=None, bgrad=None):
    """Fused q|k|v projection + RoPE for the head dims the epilogue is built for; other head dims (tiny test shapes) take GEMM + lmod_rope."""
    if hd not in ATTN_HEAD_DIMS or FUSE_ROPE == "0":
        return rope_(linear(x, w, bias, wgrad, bgrad), cos, sin, pos, nh, nkv, hd)
    if torch.is_grad_enabled() and (x.requires_grad or wgrad is not None):
        return QKVRopeFn.apply(x, w, bias, cos, sin, pos, nh, nkv, hd, wgrad, bgrad)
    x2 = _rows(x)
    out = torch.empty(x2.shape[0], w.shape[0], dtype=x.dtype, device=x.device)
    call("lmod_gemm_qkv_rope", ptr(x2), x2.stride(0), ptr(w), w.stride(0), ptr(bias) if bias is not None else None, ptr(out), out.stride(0), x2.shape[0],
         x2.shape[1], nh, nkv, hd, ptr(cos), ptr(sin), ptr(pos))
    return out


def rope_(qkv, cos, sin, pos, nh, nkv, hd):
    if torch.is_grad_enabled() and qkv.requires_grad:
        return RopeFn.apply(qkv, cos, sin, pos, nh, nkv, hd)
    rows = qkv.numel() // qkv.shape[-1]
    ld = qkv.shape[-1]
    call("lmod_rope", ptr(qkv), ld, nh, qkv.data_ptr() + nh * hd * 2, ld, nkv, hd, ptr(cos), ptr(sin), ptr(pos), rows, 0)
    return qkv


class SiluMulFn(Function):
    """act_fn(gate_proj(x)) * up_proj(x) (modeling_qwen2.py:199-200) on the fused [rows, 2I] gate|up GEMM output."""

    @staticmethod
    def forward(ctx, gu):
        gu = _c(gu)
        I = gu.shape[-1] // 2
        rows = gu.numel() // gu.shape[-1]
        out = torch.empty(gu.shape[:-1] + (I,), dtype=gu.dtype, device=gu.device)
        call("lmod_silu_mul_fwd", ptr(gu), 2 * I, rows, I, ptr(out))
        ctx.save_for_backward(gu)
        return out

    @staticmethod
    def backward(ctx, d):
        (gu,) = ctx.saved_tensors
        I = gu.shape[-1] // 2
        rows = gu.numel() // gu.shape[-1]
        dgu = torch.empty_like(gu)
        call("lmod_silu_mul_bwd", ptr(_c(d)), ptr(gu), 2 * I, rows, I, ptr(dgu))
        return dgu


def silu_mul(gu):
    if torch.is_grad_enabled() and gu.requires_grad:
        return SiluMulFn.apply(gu)
    gu = _c(gu)
    I = gu.shape[-1] // 2
    out = torch.empty(gu.shape[:-1] + (I,), dtype=gu.dtype, device=gu.device)
    call("lmod_silu_mul_fwd", ptr(gu), 2 * I, gu.numel() // gu.shape[-1], I, ptr(out))
    return out


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
class SpliceFn(Function):
    @staticmethod
    def forward(ctx, feats, embed_w, src, img_index, n_patches, embed_grad=None):
        B, T = src.shape
        H = embed_w.shape[1]
        out = torch.empty(B, T, H, dtype=embed_w.dtype, device=embed_w.device)
        call("lmod_splice_embed", ptr(embed_w), ptr(feats) if feats is not None else None, ptr(src), ptr(img_index),
             B * T, H, n_patches, ptr(out))
        ctx.save_for_backward(src, img_index)
        ctx.fshape = feats.shape
        ctx.n_patches = n_patches
        ctx.embed_grad = embed_grad                         # view of the flat gradient buffer when embed_tokens trains
        return out

    @staticmethod
    def backward(ctx, d):
        src, img_index = ctx.saved_tensors
        dfeats = torch.zeros(ctx.fshape, dtype=d.dtype, device=d.device)
        B, T = src.shape
        d = _c(d)
        call("lmod_splice_embed_bwd", ptr(d), ptr(src), ptr(img_index), B * T, d.shape[-1], ctx.n_patches, ptr(dfeats))
        if ctx.embed_grad is not None:
            call("lmod_embed_grad", ptr(d), ptr(src), B * T, d.shape[-1], ptr(ctx.embed_grad))
        return dfeats, None, None, None, None, None


def splice_embed(feats, embed_w, src, img_index, n_patches, embed_grad=None):
    feats = _c(feats)
    if torch.is_grad_enabled() and (feats.requires_grad or embed_grad is not None):
        return SpliceFn.apply(feats, embed_w, src, img_index, n_patches, embed_grad)
    B, T = src.shape
    H = embed_w.shape[1]
    out = torch.empty(B, T, H, dtype=embed_w.dtype, device=embed_w.device)
    call("lmod_splice_embed", ptr(embed_w), ptr(feats), ptr(src), ptr(img_index), B * T, H, n_patches, ptr(out))
    return out


# ---------------------------------------------------------------------------------------------------
# MoE layer (DeepSpeed 0.9.5 MoE; call site llava_qwen1_5_moe.py:536-546, SURVEY.md Appendix A)
# ---------------------------------------------------------------------------------------------------
def moe_capacity(S, E, capacity_factor, min_capacity):
    """DeepSpeed's _capacity, ceil(S/E * cf * 2) raised to min_capacity, with cf as the Python double the user set."""
    return int(_C.lib().lmod_moe_capacity(S, E, float(capacity_factor), int(min_capacity)))


LAYOUT_COMPACT, LAYOUT_SLABS, LAYOUT_ALIGNED = 0, 1, 2


def moe_route_scatter(x, wg, noise, capacity_factor, min_capacity, layout=LAYOUT_ALIGNED, padded=None):
    """Two ordinary launches (gate, seat+scatter): fp32 gate GEMV, softmax, top-1 / Gumbel top-2, stable capacity positions,
    renormalised weights, l_aux, expert offsets and the token scatter.  Returns a dict of device tensors.
    layout: 0 compact rows, 1 capacity-padded [E,C] slabs, 2 compact with 128-row aligned groups (grouped GEMM input)."""
    _need_cuda(x, wg, noise)
    if padded is not None:
        layout = LAYOUT_SLABS if padded else LAYOUT_COMPACT
    S, H = x.shape
    E = wg.shape[0]
    C = moe_capacity(S, E, capacity_factor, min_capacity)
    dev = x.device
    r = dict(
        logits=torch.empty(S, E, dtype=torch.float32, device=dev), gates=torch.empty(S, E, dtype=torch.float32, device=dev),
        idx=torch.empty(S, 2, dtype=torch.int32, device=dev), row=torch.empty(S, 2, dtype=torch.int32, device=dev),
        w=torch.empty(S, 2, dtype=torch.float32, device=dev), offsets=torch.empty(E + 1, dtype=torch.int32, device=dev),
        meta=torch.empty(4 + E, dtype=torch.float32, device=dev), capacity=C)
    rows = E * C if layout == LAYOUT_SLABS else (min(2 * S, E * C) + (128 * E if layout == LAYOUT_ALIGNED else 0))
    r["max_rows"] = rows
    r["xp"] = torch.empty(rows, H, dtype=x.dtype, device=dev)      # the op zeroes the padding rows itself (inert for the wgrad reduction)
    ws = torch.empty(int(_C.lib().lmod_moe_route_ws_elems(S, E)), dtype=torch.int32, device=dev)       # per call: safe across streams
    call("lmod_moe_route_scatter", ptr(x), ptr(wg), ptr(noise), S, H, E, float(capacity_factor), int(min_capacity), int(layout),
         ptr(r["logits"]), ptr(r["gates"]), ptr(r["idx"]), ptr(r["row"]), ptr(r["w"]), ptr(r["offsets"]), ptr(r["meta"]), ptr(r["xp"]),
         ptr(ws))
    return r


def moe_gather_combine(y, row, w, residual=None):
    S = row.shape[0]
    H = y.shape[-1]
    out = torch.empty(S, H, dtype=y.dtype, device=y.device)
    call("lmod_moe_gather_combine", ptr(y), ptr(row), ptr(w), ptr(residual) if residual is not None else None, S, H, ptr(out))
    return out


def moe_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, min_cap, fused):
    """The MoE forward as MoEFn runs it, returning every intermediate (the router's record, xp, h1, act, y, out).  fused: SwiGLU in the
    grouped GEMM's epilogue instead of GEMM + silu_mul (bit-identical)."""
    E, I2, H = w_gu.shape
    r = moe_route_scatter(x, wg, noise, cf, min_cap, LAYOUT_ALIGNED)
    R = r["max_rows"]
    xp, offs = r["xp"], r["offsets"]
    # only xp (and dy in the backward) are zero-filled: in the 128-aligned layout the grouped GEMM writes EVERY row below offsets[E],
    # so the padding rows of h1 / act / y come out as exact zeros (0 @ W); rows past offsets[E] are never read by a GEMM
    if fused:
        act, h1 = grouped_gemm_swiglu(xp, w_gu, offs, R, True)         # act [R,I], pre-activations [R,2I]: SwiGLU in the GEMM epilogue
    else:
        h1 = torch.empty(R, I2, dtype=x.dtype, device=x.device)
        grouped_gemm(xp, w_gu, h1, offs, 0)                            # [R,2I] = xp @ w_gu[e]^T
        act = silu_mul(h1)                                             # [R,I]
    y = torch.empty(R, H, dtype=x.dtype, device=x.device)
    grouped_gemm(act, w_dn, y, offs, 0)                                # [R,H] = act @ w_dn[e]^T
    r.update(h1=h1, act=act, y=y, out=moe_gather_combine(y, r["row"], r["w"], res), fused=fused)
    return r


def moe_backward_stages(st, x, wg, w_gu, w_dn, dout, dlaux, grads):
    """The MoE backward as MoEFn runs it, from moe_forward_stages' record; returns every intermediate (dy, dw, dact on the unfused
    path, dh1, dxp, dlogits, dx).  Weight gradients accumulate in place into grads['wg'|'w_gu'|'w_dn'] (None or a missing key = frozen)."""
    E, I2, H = w_gu.shape
    xp, h1, act, y, row, w, gates, idx, meta, offs = (st[k] for k in ("xp", "h1", "act", "y", "row", "w", "gates", "idx", "meta", "offsets"))
    R = xp.shape[0]
    S = x.shape[0]
    dy = torch.zeros(R, H, dtype=dout.dtype, device=dout.device)
    dw = torch.empty(S, 2, dtype=torch.float32, device=dout.device)
    call("lmod_moe_combine_bwd", ptr(dout), ptr(y), ptr(row), ptr(w), S, H, ptr(dy), ptr(dw))
    g = grads
    out = dict(dy=dy, dw=dw, dact=None)
    if st["fused"]:
        dh1 = grouped_gemm_silu_bwd(dy, w_dn, h1, offs, R)             # d(gate)|d(up) straight from the dgrad GEMM's epilogue
    else:
        dact = torch.empty(R, I2 // 2, dtype=dout.dtype, device=dout.device)
        grouped_gemm(dy, w_dn, dact, offs, 1)                          # dact = dy @ w_dn[e]
        dh1 = silu_mul_bwd(dact, h1)
        out["dact"] = dact
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
    call("lmod_moe_gate_bwd", ptr(gates), ptr(idx), ptr(row), ptr(dw), ptr(meta), ptr(gl) if gl is not None else None, S, E, ptr(dlogits))
    dx = torch.empty_like(x)
    call("lmod_moe_scatter_bwd", ptr(dxp), ptr(row), ptr(dlogits), ptr(wg), None, S, H, E, ptr(dx))
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
    def forward(ctx, x, res, wg, w_gu, w_dn, noise, cf, min_cap, grads):
        x = _c(x)
        res = _c(res)
        E, I2, H = w_gu.shape
        st = moe_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, min_cap, swiglu_fusable(I2 // 2, H, training=True))
        ctx.save_for_backward(x, wg, w_gu, w_dn, *(st[k] for k in _MOE_SAVED))
        ctx.fused = st["fused"]
        ctx.grads = grads
        return st["out"], st["meta"][0].clone()

    @staticmethod
    def backward(ctx, dout, dlaux):
        x, wg, w_gu, w_dn, *saved = ctx.saved_tensors
        st = dict(zip(_MOE_SAVED, saved), fused=ctx.fused)
        dx = moe_backward_stages(st, x, wg, w_gu, w_dn, _c(dout), dlaux, ctx.grads)["dx"]
        return dx, dout, None, None, None, None, None, None, None


_MOE_SAVED = ("xp", "h1", "act", "y", "row", "w", "gates", "idx", "meta", "offsets")


def moe_forward_nograd(x, res, wg, w_gu, w_dn, noise, cf, min_cap):
    E, I2, H = w_gu.shape
    r = moe_route_scatter(_c(x), wg, noise, cf, min_cap, LAYOUT_ALIGNED)
    R = r["max_rows"]
    if swiglu_fusable(I2 // 2, H):
        act, _ = grouped_gemm_swiglu(r["xp"], w_gu, r["offsets"], R, False)
    else:
        h1 = torch.empty(R, I2, dtype=x.dtype, device=x.device)
        grouped_gemm(r["xp"], w_gu, h1, r["offsets"], 0)
        act = silu_mul(h1)
    y = torch.empty(R, H, dtype=x.dtype, device=x.device)
    grouped_gemm(act, w_dn, y, r["offsets"], 0)
    return moe_gather_combine(y, r["row"], r["w"], _c(res)), r["meta"][0].clone(), r


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
    call("lmod_kl_counts", ptr(labels), N, seq_len, da, ptr(counts))
    with _Timed("kl_fwd_bwd"):
        call("lmod_kl_fwd_bwd_rows", ptr(s_logits), s_logits.stride(0), ptr(t_logits), t_logits.stride(0), ptr(labels), N, seq_len, vocab, da,
             float(w_kd), float(w_ce), ptr(counts), ptr(row_out), ptr(dlogits) if dlogits is not None else None,
             dlogits.stride(0) if dlogits is not None else 0, ptr(rows[0]) if rows is not None else None,
             ptr(rows[1]) if rows is not None else None)
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
        # dH = g * (dlogits @ W),  dW += dlogits^T @ (g * h)
        gs = g.to(h2.dtype)
        dh = mm_nn(dlogits, w_head, m_dev=count) * gs
        if perm is not None:
            n = 1
            for d in ctx.hshape[:-1]:
                n *= d
            dh = scatter_rows(dh, perm, count, n)
        dh = dh.reshape(ctx.hshape)
        if ctx.head_grad is not None:
            mm_tn_acc(dlogits, h2 * gs, ctx.head_grad, k_dev=count)
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
            call("lmod_logp_gather_bwd", ptr(logits), logits.stride(1), ptr(labels), B, T, V, ptr(lse), ptr(g), 0, ptr(logits), logits.stride(1))
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
def sumsq_(buf, out):
    call("lmod_sumsq", ptr(buf), 1 if buf.dtype == torch.float32 else 0, buf.numel(), ptr(out))


def adamw_(master, m, v, grad, model, lr, beta1, beta2, eps, wd, step, gnorm_sq=None, max_norm=0.0, grad_scale=1.0):
    call("lmod_adamw", ptr(master), ptr(m), ptr(v), ptr(grad), 1 if grad.dtype == torch.float32 else 0,
         ptr(model) if model is not None else None, master.numel(), float(lr), float(beta1), float(beta2), float(eps), float(wd),
         int(step), ptr(gnorm_sq) if gnorm_sq is not None else None, float(max_norm), float(grad_scale))
