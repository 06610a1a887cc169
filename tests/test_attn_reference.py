"""CPU pins of the float64 attention reference in tests/helpers.py (the yardstick of the element-wise attention tests), of K.pad_ranges, and
of the refusal of key padding without the causal mask."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import restated as R
from tests.helpers import attn_reference_fp64, attn_visible


def _keep(B, T, lens, side):
    keep = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lens):
        if n:
            if side == "right":
                keep[b, :n] = True
            else:
                keep[b, T - n:] = True
    return keep


def _sdpa(qkv, B, T, nh, nkv, hd, causal, scale, keep):
    """F.scaled_dot_product_attention in float64 under R.sdpa_mask (the reference model's 4-D mask), GQA by repeat_interleave."""
    x = qkv.view(B, T, nh + 2 * nkv, hd)
    q = x[:, :, :nh].transpose(1, 2)
    k = x[:, :, nh:nh + nkv].transpose(1, 2).repeat_interleave(nh // nkv, 1)
    v = x[:, :, nh + nkv:].transpose(1, 2).repeat_interleave(nh // nkv, 1)
    mask = R.sdpa_mask(keep, B, T, torch.float64) if keep is not None else None
    if mask is None:
        o = F.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=scale)
        s = (q @ k.transpose(-1, -2)) * scale
        if causal:
            s = s.masked_fill(torch.ones(T, T, dtype=torch.bool).triu(1), float("-inf"))
    else:
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=scale)
        s = (q @ k.transpose(-1, -2)) * scale + mask
    return o.transpose(1, 2).reshape(B * T, nh * hd), torch.logsumexp(s, -1)


CASES = [  # B, T, nh, nkv, hd, causal, side, lens
    (2, 9, 2, 2, 8, True, None, None),
    (2, 9, 2, 2, 8, False, None, None),
    (1, 1, 4, 2, 8, True, None, None),
    (1, 1, 2, 1, 16, False, None, None),
    (3, 12, 6, 2, 8, True, "right", [12, 5, 0]),
    (3, 12, 6, 2, 8, True, "left", [12, 5, 0]),
    (4, 7, 4, 1, 16, True, "left", [1, 7, 3, 6]),
    (2, 10, 3, 3, 8, True, "right", [1, 4]),
    (2, 5, 2, 1, 8, False, None, None),
]


@pytest.mark.parametrize("B,T,nh,nkv,hd,causal,side,lens", CASES)
def test_attn_reference_matches_sdpa_and_autograd(B, T, nh, nkv, hd, causal, side, lens):
    g = torch.Generator().manual_seed(B * 100 + T * 10 + nh + hd)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, generator=g, dtype=torch.float64).to(torch.bfloat16)
    dout = torch.randn(B * T, nh * hd, generator=g, dtype=torch.float64).to(torch.bfloat16)
    keep = _keep(B, T, lens, side) if side else None
    scale = hd ** -0.5
    ref = attn_reference_fp64(qkv, B, T, nh, nkv, hd, causal, scale, keep=keep, dout=dout)
    x = qkv.double().requires_grad_(True)
    o, lse = _sdpa(x, B, T, nh, nkv, hd, causal, scale, keep)
    torch.testing.assert_close(ref["o"], o.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["lse"], lse.detach(), rtol=1e-12, atol=1e-12)
    o.backward(dout.double())
    torch.testing.assert_close(ref["dqkv"], x.grad, rtol=1e-10, atol=1e-12)
    for key in ("o_tol", "lse_tol", "dqkv_tol"):
        t = ref[key]
        assert torch.isfinite(t).all() and (t > 0).all(), key
    # the bounds are majorants of the terms they name: never below the bf16 store of the value itself
    assert (ref["o_tol"] >= 2.0 ** -8 * ref["o"].abs()).all()
    assert (ref["dqkv_tol"] >= 2.0 ** -8 * ref["dqkv"].abs()).all()


def test_attn_reference_masks():
    """attn_visible against R.sdpa_mask: a key is visible exactly where the additive mask is 0, incl. the un-masked rows in front of a
    left-padded sequence and in an all-padding sample."""
    B, T = 4, 9
    for side in ("right", "left"):
        keep = _keep(B, T, [9, 4, 1, 0], side)
        m = R.sdpa_mask(keep, B, T, torch.float64)[:, 0]
        assert torch.equal(attn_visible(B, T, True, keep), m == 0)
    vis = attn_visible(B, T, True, _keep(B, T, [9, 4, 1, 0], "left"))
    assert vis[3].all()                                   # all padding: every row sees every key
    assert vis[1, :5].all() and not vis[1, 5, :5].any()   # rows before kv_lo = 5 see everything, row 5 only key 5
    assert torch.equal(attn_visible(2, T, False), torch.ones(2, T, T, dtype=torch.bool))
    with pytest.raises(AssertionError):
        attn_visible(B, T, False, keep)


def test_pad_ranges_on_cpu_masks():
    from llavamod import kernels as K
    T = 10
    keep = torch.zeros(7, T, dtype=torch.bool)
    keep[0] = True                     # no padding
    # keep[1]: all padding
    keep[2, 4] = True                  # one token inside
    keep[3, 0] = True                  # one token at the start
    keep[4, T - 1] = True              # one token at the end
    keep[5, :6] = True                 # right padding
    keep[6, 3:] = True                 # left padding
    lo, hi = K.pad_ranges(keep)
    assert lo.dtype == torch.int32 and hi.dtype == torch.int32 and lo.is_contiguous() and hi.is_contiguous()
    assert lo.tolist() == [0, 0, 4, 0, T - 1, 0, 3]
    assert hi.tolist() == [T, 0, 5, 1, T, 6, T]


def test_key_padding_without_causal_mask_is_rejected():
    """Non-causal attention with a key range would un-mask the rows in front of kv_lo instead of limiting them to [kv_lo, kv_hi): every
    entry point refuses it.  The Python checks run before any device work; the C entry points check their arguments before they read a
    pointer, so this runs without a GPU."""
    from llavamod import _C, kernels as K
    B, T, nh, hd = 2, 8, 2, 64
    qkv = torch.zeros(B * T, 3 * nh * hd, dtype=torch.bfloat16)
    pad = (torch.zeros(B, dtype=torch.int32), torch.full((B,), T, dtype=torch.int32))
    with pytest.raises(_C.LmodError, match="causal"):
        K.attention(qkv, B, T, nh, nh, hd, causal=False, pad=pad)
    with pytest.raises(_C.LmodError, match="causal"):
        K.attention_fwd(qkv, B, T, nh, nh, hd, False, pad=pad)
    with pytest.raises(_C.LmodError, match="causal"):
        K.attention_bwd(qkv, qkv[:, :nh * hd], qkv[:, :nh * hd], None, B, T, nh, nh, hd, False, hd ** -0.5, pad=pad)
    L = _C.lib()
    fake = ctypes.c_void_p(1 << 20)     # never dereferenced: the argument checks return first
    rc = L.lmod_attn_fwd(fake, 3 * nh * hd, B, T, nh, nh, hd, 0, 0.125, fake, nh * hd, None, fake, fake, None)
    assert rc != 0 and b"causal" in L.lmod_last_error()
    rc = L.lmod_attn_bwd(fake, 3 * nh * hd, fake, nh * hd, fake, nh * hd, fake, B, T, nh, nh, hd, 0, 0.125, fake, 3 * nh * hd, fake, fake,
                         fake, fake, None)
    assert rc != 0 and b"causal" in L.lmod_last_error()
