"""lmod_attn_decode and lmod_attn_decode_chunk (csrc/decode.cu) bit for bit on operands that make them exact (tests/decode_exact.py), at
every template instantiation, ring regime and block / ring / split edge; lmod_kv_append and lmod_kv_append_rows at the cache's ends.

The float64 bound of test_attn_decode_gpu.py has to cover a worst-case fp32 sum over thousands of keys, so one lost, doubled or shifted
key stays inside it.  Here every probability is 0 or 1 (tier 1) or a small power of two (tier 2) and every value a small integer, so the
kernel's sums are exact whatever their order and the output must equal bf16(fp32(sum w v) / fp32(sum w)) in every bit.  The cases run
with uninitialised memory poisoned (out, lse and the workspace start as NaN), cache rows from len on are NaN, and q is a row of a wider
fused buffer whose columns past nh * hd are NaN.

The splits depend on the SM count; the case list is built from the device's, and the module asserts that it launches every instantiation
(HD 64 / 128 x G 1..8 for the single-query kernel, x VG 1..8 for the chunk kernel) and every ring regime on the device at hand."""
import json
import zlib
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from llavamod import kernels as K  # noqa: E402
from tests import decode_exact as D  # noqa: E402
from tests.helpers import poisoned_uninitialised_memory  # noqa: E402

SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
REGIMES = ["one split", "split = NST blocks", "split = NST + 1 blocks", "split >= 2 NST + 1 blocks", "short last split"]
PROJECT = [(64, 16, 16), (128, 16, 16), (128, 32, 32), (64, 14, 2), (128, 28, 4)]     # hd, nh, nkv of the models' attention
REPORT = {}


def split_keys(max_len, nkv):
    return D.decode_splits(max_len, nkv, SMS)[1] * D.BK


def _regime_shape(hd, regime):
    """The cheapest (nkv, max_len) whose full-length launch runs `regime` on this device."""
    best = None
    for nkv in (1, 2, 4, 8, 16, 32):
        for blocks in range(1, 257):
            if (hd, regime) in D.ring_regimes(hd, blocks * D.BK, nkv, SMS):
                if best is None or nkv * blocks < best[0] * best[1] // D.BK:
                    best = (nkv, blocks * D.BK)
                break
    assert best is not None, (hd, regime, SMS)
    return best


def _single_cases():
    """(name, hd, nh, nkv, max_len, tier, mult)"""
    cases = [("inst_hd%d_g%d" % (hd, G), hd, 2 * G, 2, 1024, 1, 1) for hd in (64, 128) for G in range(1, 9)]
    cases += [("pad_hd32_g2", 32, 4, 2, 512, 1, 1), ("pad_hd80_g7", 80, 7, 1, 512, 1, 1)]
    for hd in (64, 128):
        for reg in REGIMES:
            nkv, max_len = _regime_shape(hd, reg)
            cases.append(("regime_hd%d_%s" % (hd, reg.replace(" ", "_")), hd, 2 * nkv, nkv, max_len, 1, 1))
    for hd, nh, nkv in PROJECT:
        for max_len in (4096, 8192):
            cases.append(("model_hd%d_%d_%d_len%d" % (hd, nh, nkv, max_len), hd, nh, nkv, max_len, 1, 1))
    cases.append(("long_hd128_28_4_len32768", 128, 28, 4, 32768, 1, 1))
    cases.append(("scale2_hd64_g4", 64, 8, 2, 2048, 1, 2))
    return cases


def _chunk_cases():
    """(name, hd, nh, nkv, max_len, T): G 1 with T 1..9, 12, 17 (T > 8 gives a second, partial row group), G 3 (two rows per group), G 8."""
    ts = list(range(1, 10)) + [12, 17]
    cases = [("chunk_hd%d_g1_T%d" % (hd, T), hd, 2, 2, 1024, T) for hd in (64, 128) for T in ts]
    cases += [("chunk_hd%d_g3_T%d" % (hd, T), hd, 6, 2, 1024, T) for hd in (64, 128) for T in ts]
    cases += [("chunk_hd%d_g8_T%d" % (hd, T), hd, 8, 1, 1024, T) for hd in (64, 128) for T in (1, 3, 9)]
    cases += [("chunk_hd128_32_32_len4096_T5", 128, 32, 32, 4096, 5), ("chunk_hd64_16_16_len8192_T4", 64, 16, 16, 8192, 4)]
    return cases


SINGLE = _single_cases()
CHUNK = _chunk_cases()
TIER2 = [("tier2_hd64_g2", 64, 4, 2, 4096, 2, 1), ("tier2_hd128_g4", 128, 8, 2, 4096, 2, 1), ("tier2_hd128_32_32", 128, 32, 32, 8192, 2, 1),
         ("tier2_scale2_hd64_g8", 64, 16, 2, 2048, 2, 2)]

INSTANTIATIONS = sorted({(D.head_dim_padded(c[1]), c[2] // c[3]) for c in SINGLE})
CHUNK_INSTANTIATIONS = sorted({(D.head_dim_padded(c[1]), min(c[5], D.MAX_G // (c[2] // c[3])) * (c[2] // c[3])) for c in CHUNK})
RING_REGIMES = sorted(set().union(*(D.ring_regimes(c[1], c[4], c[3], SMS) for c in SINGLE)))
_ALL = [(hp, g) for hp in (64, 128) for g in range(1, D.MAX_G + 1)]
assert INSTANTIATIONS == _ALL, INSTANTIATIONS
assert CHUNK_INSTANTIATIONS == _ALL, CHUNK_INSTANTIATIONS
assert set(RING_REGIMES) >= {(hp, r) for hp in (64, 128) for r in REGIMES}, (SMS, RING_REGIMES)


def _lens(max_len, nkv, hd, T=1):
    ring = D.NST[D.head_dim_padded(hd)] * D.BK
    return [n for n in D.edge_lengths(max_len, split_keys(max_len, nkv), ring) if n >= T]


def _run_single(q, d, lens):
    B = q.shape[0]
    ws = torch.empty(K.attn_decode_ws_elems(B, d.nh, d.nkv, d.hd, d.max_len), dtype=torch.float32, device="cuda")
    lt = torch.tensor(lens, dtype=torch.int32, device="cuda")
    return K.attn_decode(q, d.nh, d.nkv, d.hd, d.k, d.v, lt, ws, scale=d.scale, need_lse=True)


def _run_chunk(d):
    ws = torch.empty(K.attn_decode_chunk_ws_elems(d.B, d.T, d.nh, d.nkv, d.hd, d.max_len), dtype=torch.float32, device="cuda")
    lt = torch.tensor(d.lens, dtype=torch.int32, device="cuda")
    return K.attn_decode_chunk(d.q, d.B, d.T, d.nh, d.nkv, d.hd, d.k, d.v, lt, ws, scale=d.scale, need_lse=True)


def _check(name, d, out, lse):
    want, want_lse, lse_tol = d.expected()
    diff = out.view(torch.int16) != want.view(torch.int16)
    if bool(diff.any()):
        r, c = (int(i) for i in torch.nonzero(diff)[0])
        raise AssertionError("%s: %d / %d outputs differ in bits; first row %d (len %d) head %d column %d: got %r want %r"
                             % (name, int(diff.sum()), diff.numel(), r, d.lims[r], c // d.hd, c % d.hd, float(out[r, c]), float(want[r, c])))
    err = (lse.double() - want_lse).abs()
    ratio = float((err / lse_tol).max())
    REPORT[name] = round(ratio, 4)
    assert bool(torch.isfinite(lse).all()) and ratio <= 1.0, (name, ratio)


def _single(case):
    name, hd, nh, nkv, max_len, tier, mult = case
    lens = _lens(max_len, nkv, hd)
    with poisoned_uninitialised_memory():
        d = D.Design(len(lens), 1, nh, nkv, hd, lens, max_len, split_keys(max_len, nkv), seed=zlib.crc32(name.encode()), tier=tier, mult=mult,
                     device="cuda")
        out, lse = _run_single(d.q, d, lens)
        _check(name, d, out, lse)
        out2, lse2 = _run_single(d.q, d, lens)
    assert torch.equal(out.view(torch.int16), out2.view(torch.int16)) and torch.equal(lse, lse2), name


@pytest.mark.parametrize("case", SINGLE, ids=[c[0] for c in SINGLE])
def test_decode_exact(case):
    _single(case)


@pytest.mark.parametrize("case", TIER2, ids=[c[0] for c in TIER2])
def test_decode_exact_tier2(case):
    """Scores 0, -1, -2, -3: ex2.approx.ftz must be exact at small negative integers."""
    _single(case)


@pytest.mark.parametrize("case", CHUNK, ids=[c[0] for c in CHUNK])
def test_decode_chunk_exact(case):
    """Every row t of the chunk matches the exact expectation at its own limit len - T + t + 1 and the bytes lmod_attn_decode gives for that
    row alone."""
    name, hd, nh, nkv, max_len, T = case
    lens = _lens(max_len, nkv, hd, T)
    with poisoned_uninitialised_memory():
        d = D.Design(len(lens), T, nh, nkv, hd, lens, max_len, split_keys(max_len, nkv), seed=zlib.crc32(name.encode()), device="cuda")
        out, lse = _run_chunk(d)
        _check(name, d, out, lse)
        o3, l3 = out.view(d.B, T, -1), lse.view(d.B, T, -1)
        for t in range(T):
            o1, l1 = _run_single(d.q.view(d.B, T, -1)[:, t], d, [n - T + t + 1 for n in lens])
            assert torch.equal(o3[:, t].view(torch.int16), o1.view(torch.int16)) and torch.equal(l3[:, t], l1), (name, t)
        out2, lse2 = _run_chunk(d)
    assert torch.equal(out.view(torch.int16), out2.view(torch.int16)) and torch.equal(lse, lse2), name


# ---- lmod_kv_append / lmod_kv_append_rows: the cache is a view inside a larger buffer with sentinels on both sides ----
def _cache_in_buffer(B, nkv, max_len, hp, fill):
    n, pre, post = B * nkv * max_len * hp, 16 * hp, max_len * hp
    buf = torch.full((pre + n + post,), -777.0, dtype=torch.bfloat16, device="cuda")
    buf[pre:pre + n] = fill
    return buf, buf[pre:pre + n].view(B, nkv, max_len, hp)


def _assert_same(name, got, want):
    diff = got.view(torch.int16) != want.view(torch.int16)
    assert not bool(diff.any()), "%s: %d elements differ, first at %d" % (name, int(diff.sum()), int(torch.nonzero(diff)[0]))


@pytest.mark.parametrize("hd", [64, 128, 80])
def test_kv_append_at_the_cache_ends(hd):
    """Appends that end at row max_len - 1, and offsets whose rows run past max_len (or start below 0): the kernel writes the rows inside
    the cache and drops the rest; nothing else changes, the sentinels around the cache included."""
    B, nh, nkv, max_len = 3, 4, 2, 200
    hp = D.head_dim_padded(hd)
    g = torch.Generator(device="cuda").manual_seed(hd)
    kb, kc = _cache_in_buffer(B, nkv, max_len, hp, -555.0)
    vb, vc = _cache_in_buffer(B, nkv, max_len, hp, -333.0)
    wk, wv = kb.clone(), vb.clone()
    wkc, wvc = wk[16 * hp:16 * hp + kc.numel()].view_as(kc), wv[16 * hp:16 * hp + vc.numel()].view_as(vc)
    for n_new, offs in [(5, [max_len - 5, 0, 100]), (7, [max_len - 3, max_len, 150]), (1, [max_len - 1, max_len + 5, 0]),
                        (4, [-2, 10, max_len - 1])]:
        qkv = torch.randn(B * n_new, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
        with poisoned_uninitialised_memory():
            K.kv_append(qkv, B, n_new, nh, nkv, hd, kc, vc, torch.tensor(offs, dtype=torch.int32, device="cuda"))
        x = qkv.view(B, n_new, nh + 2 * nkv, hd)
        for b in range(B):
            for r in range(n_new):
                pos = offs[b] + r
                if 0 <= pos < max_len:
                    wkc[b, :, pos] = 0
                    wvc[b, :, pos] = 0
                    wkc[b, :, pos, :hd] = x[b, r, nh:nh + nkv]
                    wvc[b, :, pos, :hd] = x[b, r, nh + nkv:]
        _assert_same("k %s %s" % (n_new, offs), kb, wk)
        _assert_same("v %s %s" % (n_new, offs), vb, wv)


@pytest.mark.parametrize("hd", [64, 128])
def test_kv_append_rows_empty_and_full_ranges(hd):
    """kv_append_rows with empty ranges (lo = hi), ranges that end at T, and a packed range that ends at row max_len - 1."""
    B, T, nh, nkv, max_len = 4, 9, 4, 2, 64
    hp = D.head_dim_padded(hd)
    g = torch.Generator(device="cuda").manual_seed(hd + 1)
    kb, kc = _cache_in_buffer(B, nkv, max_len, hp, -555.0)
    vb, vc = _cache_in_buffer(B, nkv, max_len, hp, -333.0)
    wk, wv = kb.clone(), vb.clone()
    wkc, wvc = wk[16 * hp:16 * hp + kc.numel()].view_as(kc), wv[16 * hp:16 * hp + vc.numel()].view_as(vc)
    for lo, hi, offs in [([0, 3, 9, 5], [9, 3, 9, 9], [0, 7, 0, max_len - 4]), ([2, 0, 0, 8], [9, 0, 1, 9], [max_len - 7, 0, max_len - 1, 3])]:
        qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
        i32 = lambda a: torch.tensor(a, dtype=torch.int32, device="cuda")  # noqa: E731
        with poisoned_uninitialised_memory():
            K.kv_append_rows(qkv, B, T, nh, nkv, hd, kc, vc, i32(lo), i32(hi), i32(offs))
        x = qkv.view(B, T, nh + 2 * nkv, hd)
        for b in range(B):
            for r in range(lo[b], hi[b]):
                pos = offs[b] + r - lo[b]
                wkc[b, :, pos, :hd] = x[b, r, nh:nh + nkv]
                wvc[b, :, pos, :hd] = x[b, r, nh + nkv:]
        _assert_same("k rows %s %s" % (lo, hi), kb, wk)
        _assert_same("v rows %s %s" % (lo, hi), vb, wv)


def test_coverage_on_this_device():
    print("SMs %d; single-query instantiations %s; chunk instantiations %s; ring regimes %s"
          % (SMS, INSTANTIATIONS, CHUNK_INSTANTIATIONS, RING_REGIMES))
    assert INSTANTIATIONS == _ALL and CHUNK_INSTANTIATIONS == _ALL


def teardown_module(module):
    out = os.environ.get("LLAVAMOD_TEST_REPORT")
    if out and REPORT:
        with open(out, "a") as f:
            f.write(json.dumps({"decode_exact_lse_err_over_bound": REPORT}) + "\n")
    print("decode exact lse err/bound:", json.dumps(REPORT))
