"""lmod_attn_decode_chunk (T new query rows per sequence over the KV cache, the verify step of assisted decoding) against float64 attention,
and row by row byte for byte against lmod_attn_decode on that row alone at len - T + t + 1.

As in test_attn_decode_gpu.py, cache rows at or past len[b] are NaN and needle keys sit at the first, last and split-edge positions; the
lengths put the rows' limits on both sides of the 64-key block, ring and split edges."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from llavamod import kernels as K  # noqa: E402
from tests.test_attn_decode_gpu import BK, NST, decode_reference_fp64, make_cache, run_decode, split_keys  # noqa: E402


def run_chunk(q, k, v, lens, B, T, nh, nkv, hd):
    max_len = k.shape[2]
    ws = torch.empty(K.attn_decode_chunk_ws_elems(B, T, nh, nkv, hd, max_len), dtype=torch.float32, device="cuda")
    lt = torch.tensor(lens, dtype=torch.int32, device="cuda")
    return K.attn_decode_chunk(q, B, T, nh, nkv, hd, k, v, lt, ws, need_lse=True)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("G,nkv", [(1, 2), (2, 2), (7, 1), (8, 2)])
def test_chunk_rows_equal_single_query_and_match_fp64(hd, G, nkv):
    nh = G * nkv
    max_len = 1024
    sk = split_keys(max_len, nkv)
    ring = NST[hd] * BK
    for T in range(1, 9):
        edges = sorted({BK, ring, sk, 2 * sk, max_len})
        lens = sorted({T, T + 1} | {min(max_len, max(T, e + T // 2)) for e in edges} | {min(max_len, e + T - 1) for e in edges})
        B = len(lens)
        needles = []
        for b, n in enumerate(lens):
            needles.append((b, n - 1, 24.0))
            if n - T > 1:
                needles.append((b, n - T - 1, 20.0))             # the last key every row sees
            if n > 2:
                needles.append((b, 0, 16.0))
            if n > sk + 1:
                needles.append((b, sk - 1, 20.0))
        q1, k, v = make_cache(B, nh, nkv, hd, lens, max_len, seed=1000 * hd + 10 * G + T, needles=needles)
        g = torch.Generator(device="cuda").manual_seed(T)
        q = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
        q.view(B, T, -1)[:, T - 1] = q1                            # the last row carries the needle-aligned query
        out, lse = run_chunk(q, k, v, lens, B, T, nh, nkv, hd)
        o3, l3 = out.view(B, T, nh * hd), lse.view(B, T, nh)
        for t in range(T):
            lens_t = [n - T + t + 1 for n in lens]
            qt = q.view(B, T, -1)[:, t].contiguous()
            o1, l1 = run_decode(qt, k, v, lens_t, nh, nkv, hd)
            assert torch.equal(o3[:, t], o1) and torch.equal(l3[:, t], l1), (hd, G, T, t)
            if T in (1, 4, 8):
                ref, ref_lse, tol, tol_lse = decode_reference_fp64(qt, k, v, lens_t, nh, nkv, hd, hd ** -0.5)
                o = o3[:, t].double().view(B, nh, hd)
                assert torch.isfinite(o).all()
                assert ((o - ref).abs() <= tol).all(), (hd, G, T, t)
                assert ((l3[:, t].double() - ref_lse).abs() <= tol_lse).all(), (hd, G, T, t)


def test_chunk_head_dim_below_64_and_bad_arguments():
    """hd 32 runs in the zero-padded cache layout; a workspace too small or a q of the wrong row count is refused."""
    nh, nkv, hd, T = 4, 2, 32, 3
    lens = [5, 70]
    q1, k, v = make_cache(2, nh, nkv, hd, lens, 256, seed=3)
    q = torch.randn(2 * T, nh * hd, device="cuda").to(torch.bfloat16)
    out, lse = run_chunk(q, k, v, lens, 2, T, nh, nkv, hd)
    for t in range(T):
        o1, l1 = run_decode(q.view(2, T, -1)[:, t].contiguous(), k, v, [n - T + t + 1 for n in lens], nh, nkv, hd)
        assert torch.equal(out.view(2, T, -1)[:, t], o1) and torch.equal(lse.view(2, T, -1)[:, t], l1)
    lt = torch.tensor(lens, dtype=torch.int32, device="cuda")
    small = torch.empty(K.attn_decode_ws_elems(2, nh, nkv, hd, 256), dtype=torch.float32, device="cuda")
    with pytest.raises(Exception):
        K.attn_decode_chunk(q, 2, T, nh, nkv, hd, k, v, lt, small)
    ws = torch.empty(K.attn_decode_chunk_ws_elems(2, T, nh, nkv, hd, 256), dtype=torch.float32, device="cuda")
    with pytest.raises(Exception):
        K.attn_decode_chunk(q[:-1], 2, T, nh, nkv, hd, k, v, lt, ws)
