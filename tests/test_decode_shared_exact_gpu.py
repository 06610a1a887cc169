"""lmod_attn_decode_shared (csrc/decode.cu) against lmod_attn_decode on the materialised per-sequence cache, bit for bit in out and lse.

Sequence b*n + j's materialised cache is prompt b's prefix rows [0, prefix_len[b]) followed by copy j's suffix rows, in a plain
[B*n, nkv, max_len, hp] cache; lmod_attn_decode runs on it at the same max_len.  Every row past a length is NaN in all three buffers
(prefix past prefix_len, suffix past len - prefix_len, materialised past len), out, lse and the workspace start as NaN, and q is a row of
a wider fused buffer whose columns past nh * hd are NaN, so a row that is read when it should not be shows up as a NaN.  Both results are
also held to the float64 reference's bound (tests/decode_exact.py).

The cases cover head widths 64 and 128, every virtual-head instantiation (copies per CTA * query heads per KV head, 1..8), G in {1, 2, 7,
8} with n in {1, 2, 3, 8} (n * G > 8 spreads a KV head's copies over several CTAs), prefix lengths on both sides of 64-key block, ring
and split edges, suffix lengths 0, 1, across a block edge and at S_max, a different prefix length per prompt, and every split regime of
this device's SM count."""
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu

from llavamod import kernels as K  # noqa: E402
from tests import decode_exact as D  # noqa: E402
from tests.helpers import poisoned_uninitialised_memory  # noqa: E402

SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
REGIMES = ["one split", "split = NST blocks", "split = NST + 1 blocks", "split >= 2 NST + 1 blocks", "short last split"]
S_MAX = 100


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


def _cases():
    """(name, hd, G, nkv, n, max_len)"""
    cases = [("g%d_n%d_hd%d" % (G, n, hd), hd, G, 2, n, 1024) for hd in (64, 128) for G in (1, 2, 7, 8) for n in (1, 2, 3, 8)]
    cases += [("vg%d_hd%d" % (n, hd), hd, 1, 1, n, 1024) for hd in (64, 128) for n in (4, 5, 6, 7)]     # every virtual-head count
    for hd in (64, 128):
        for reg in REGIMES:
            nkv, max_len = _regime_shape(hd, reg)
            cases.append(("regime_hd%d_%s" % (hd, reg.replace(" ", "_")), hd, 2, nkv, 5, max_len))
    cases += [("teacher_hd128_32_32_n4_len1024", 128, 1, 32, 4, 1024), ("student_hd64_16_16_n8_len1024", 64, 1, 16, 8, 1024),
              ("gqa_hd128_28_4_n4_len8704", 128, 7, 4, 4, 8704), ("gqa_hd64_14_2_n8_len8704", 64, 7, 2, 8, 8704)]
    return cases


CASES = _cases()
INSTANTIATIONS = {(D.head_dim_padded(c[1]), min(c[4], D.MAX_G // c[2]) * c[2]) for c in CASES}     # (hp, virtual heads per CTA)
RING_REGIMES = set().union(*(D.ring_regimes(c[1], c[5], c[3], SMS) for c in CASES))


def _s_max(max_len):
    return min(S_MAX, max_len // 2)


def _prefix_lengths(max_len, nkv, hd):
    """Prefix lengths on both sides of the block, ring-pass and split edges, leaving S_max rows for the suffix."""
    ring = D.NST[D.head_dim_padded(hd)] * D.BK
    sk = D.decode_splits(max_len, nkv, SMS)[1] * D.BK
    top = max_len - _s_max(max_len)
    return sorted({n for n in D.edge_lengths(max_len, sk, ring) + [top, 37] if 1 <= n <= top})


def _suffix_lengths(plen, n, b, s_max):
    """Suffix lengths of prompt b's n copies: 0, 1, across the next 64-key block edge and S_max, a different mix per prompt."""
    opts = [0, 1, min(s_max, D.BK - plen % D.BK + 1), s_max]
    return [opts[(b + j) % 4] for j in range(n)]


def _operands(name, hd, G, nkv, n, max_len):
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(name.encode()))
    hp = D.head_dim_padded(hd)
    nh = G * nkv
    plens = _prefix_lengths(max_len, nkv, hd)
    B = len(plens)
    sm = _s_max(max_len)
    slens = [s for b, p in enumerate(plens) for s in _suffix_lengths(p, n, b, sm)]
    lens = [plens[r // n] + slens[r] for r in range(B * n)]
    nan = float("nan")

    def rnd(*shape):
        return torch.randn(*shape, device="cuda", generator=g).to(torch.bfloat16)

    kp, vp = rnd(B, nkv, max_len, hp), rnd(B, nkv, max_len, hp)
    ks, vs = rnd(B * n, nkv, sm, hp), rnd(B * n, nkv, sm, hp)
    km = torch.full((B * n, nkv, max_len, hp), nan, dtype=torch.bfloat16, device="cuda")
    vm = torch.full_like(km, nan)
    for b, p in enumerate(plens):
        kp[b, :, p:], vp[b, :, p:] = nan, nan
        for j in range(n):
            r, s = b * n + j, slens[b * n + j]
            ks[r, :, s:], vs[r, :, s:] = nan, nan
            km[r, :, :p], vm[r, :, :p] = kp[b, :, :p], vp[b, :, :p]
            km[r, :, p:p + s], vm[r, :, p:p + s] = ks[r, :, :s], vs[r, :, :s]
    ld = (nh + 2 * nkv) * hd
    q = torch.full((B * n, ld), nan, dtype=torch.bfloat16, device="cuda")
    q[:, :nh * hd] = rnd(B * n, nh * hd)
    i32 = lambda a: torch.tensor(a, dtype=torch.int32, device="cuda")  # noqa: E731
    return dict(B=B, nh=nh, q=q, kp=kp, vp=vp, ks=ks, vs=vs, km=km, vm=vm, plen=i32(plens), lens=i32(lens), lens_host=lens)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_decode_shared_equals_decode_on_the_materialised_cache(case):
    name, hd, G, nkv, n, max_len = case
    o = _operands(*case)
    B, nh = o["B"], o["nh"]
    with poisoned_uninitialised_memory():
        ws1 = torch.empty(K.attn_decode_ws_elems(B * n, nh, nkv, hd, max_len), dtype=torch.float32, device="cuda")
        want, want_lse = K.attn_decode(o["q"], nh, nkv, hd, o["km"], o["vm"], o["lens"], ws1, need_lse=True)
        ws2 = torch.empty(K.attn_decode_shared_ws_elems(B, n, nh, nkv, hd, max_len), dtype=torch.float32, device="cuda")
        got, lse = K.attn_decode_shared(o["q"], n, nh, nkv, hd, o["kp"], o["vp"], o["plen"], o["ks"], o["vs"], o["lens"], max_len, ws2,
                                        need_lse=True)
    diff = got.view(torch.int16) != want.view(torch.int16)
    if bool(diff.any()):
        r, c = (int(i) for i in torch.nonzero(diff)[0])
        raise AssertionError("%s: %d / %d outputs differ in bits; first row %d (len %d) head %d: got %r want %r"
                             % (name, int(diff.sum()), diff.numel(), r, o["lens_host"][r], c // hd, float(got[r, c]), float(want[r, c])))
    assert torch.equal(lse, want_lse), name
    assert bool(torch.isfinite(got.float()).all()) and bool(torch.isfinite(lse).all()), name
    ref, ref_lse, tol, tol_lse = D.decode_reference_fp64(o["q"], o["km"], o["vm"], o["lens_host"], nh, nkv, hd, hd ** -0.5)
    assert bool(((got.double().view(B * n, nh, hd) - ref).abs() <= tol).all()), name
    assert bool(((lse.double() - ref_lse).abs() <= tol_lse).all()), name


def test_decode_shared_cases_cover_every_instantiation_and_regime():
    """The cases launch every (head width, virtual heads per CTA) instantiation and every split regime of this device."""
    want = {(hp, vg) for hp in (64, 128) for vg in range(1, D.MAX_G + 1)}
    assert INSTANTIATIONS >= want, sorted(want - INSTANTIATIONS)
    assert RING_REGIMES >= {(hp, r) for hp in (64, 128) for r in REGIMES}, (SMS, sorted(RING_REGIMES))


def test_decode_shared_rejects_bad_operands():
    o = _operands("bad", 64, 2, 2, 3, 512)
    B, nh = o["B"], o["nh"]
    ws = torch.empty(K.attn_decode_shared_ws_elems(B, 3, nh, 2, 64, 512), dtype=torch.float32, device="cuda")
    with pytest.raises(Exception, match="workspace"):
        K.attn_decode_shared(o["q"], 3, nh, 2, 64, o["kp"], o["vp"], o["plen"], o["ks"], o["vs"], o["lens"], 512, ws[:10])
    with pytest.raises(Exception, match="KV cache"):
        K.attn_decode_shared(o["q"], 2, nh, 2, 64, o["kp"], o["vp"], o["plen"], o["ks"], o["vs"], o["lens"], 512, ws)
