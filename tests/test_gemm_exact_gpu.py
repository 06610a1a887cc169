"""The bf16 wgmma GEMM family (csrc/gemm.cu: lmod_gemm_bf16(_dyn), lmod_grouped_gemm_bf16 and the fused-epilogue forms) element by
element against float64, at the tile, layout, ring and extent edges where a kernel goes wrong.

Operand kinds (every value exact in bf16):
  exact      integers in [-4, 4] (bias, D_old: small integers): every partial sum is exact in fp32, so the fp32 output equals float64 and
             the bf16 output equals ref.to(bf16) with zero tolerance (+0 and -0 alike) -- a dropped, doubled or misplaced k-block, a
             swizzle error or a stale ring stage fails
  one-hot    A[m, k] = 1 iff k == (7m + 3) % K, B integer codes in [-125, 125]: D[m, n] = B[n, f(m)] exactly, a failure names the index
  random, cancelling (alternating signs, magnitudes 16..32), huge_tiny (one 2^7-scale product among 2^-6-scale ones): within
             helpers._gemm_tol(ref, maj, K) = 2^-8 |ref| + (1 + 2^-8)(ceil(K/16) + 1) 2^-23 maj, maj = |A||B|^T (+ |bias| + |D_old|): the
             bf16 store and the wgmma accumulator, which truncates at each k = 16 step.  The fp32 output adds one alignment step and one
             fp32 add per split (splits 2^-23 maj), and the add of D_old 2^-23 |ref|.
Every stored operand has NaN in the gap columns of its row stride, every output a sentinel in its gap columns and in rows past M; no NaN
may reach a valid element and no sentinel may change.  Each case prints its worst err / bound."""
import pytest
import torch

from tests.helpers import _gemm_tol, poisoned_uninitialised_memory

pytestmark = pytest.mark.gpu

F64, BF16 = torch.float64, torch.bfloat16
NAN = float("nan")
SENT = 12345.0                                     # bf16 12352; fp32 exact
LAYOUTS = [(False, False), (False, True), (True, True), (True, False)]
KINDS = ["exact", "onehot", "random", "cancelling", "huge_tiny"]
EXACT_KINDS = ("exact", "onehot")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_bn(m_tiles, N):
    """The tile width gemm.cu's pick_bn chooses: 256 unless a 256-wide tiling leaves the SMs under 1.5 waves (and N > 128)."""
    return 256 if (m_tiles * ((N + 255) // 256) >= _sms() * 3 // 2 or N <= 128) else 128


def _pad8(n):
    return (n + 7) // 8 * 8


def _bf(x):
    return x.to(BF16).to(F64)


def operands(kind, M, N, K, gen):
    """Logical A [M, K], B [N, K], bias [N], D_old [M, N] (float64 on the GPU, exact in bf16)."""
    dev = "cuda"
    ri = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, device=dev, generator=gen).to(F64)   # noqa: E731
    if kind == "exact":
        A, B, bias, old = ri(-4, 4, M, K), ri(-4, 4, N, K), ri(-16, 16, N), ri(-64, 64, M, N)
    elif kind == "onehot":
        A = torch.zeros(M, K, dtype=F64, device=dev)
        A[torch.arange(M, device=dev), (7 * torch.arange(M, device=dev) + 3) % K] = 1.0
        B, bias, old = ri(-125, 125, N, K), ri(-16, 16, N), ri(-64, 64, M, N)
    else:
        rn = lambda *s: torch.randn(s, device=dev, generator=gen, dtype=F64)                  # noqa: E731
        ru = lambda *s: torch.rand(s, device=dev, generator=gen, dtype=F64)                   # noqa: E731
        bias, old = _bf(rn(N)), _bf(rn(M, N))
        if kind == "random":
            A, B = _bf(rn(M, K)), _bf(rn(N, K))
        elif kind == "cancelling":
            sign = 1.0 - 2.0 * (torch.arange(K, device=dev) % 2).to(F64)
            A, B = _bf(16 * (1 + ru(M, K)) * sign), _bf(16 * (1 + ru(N, K)))
        else:
            A = rn(M, K).sign() * 2.0 ** -6
            A[:, K // 3] = 2.0 ** 7 * rn(M).sign()
            B = _bf(rn(N, K).sign() * (1 + ru(N, K)))
    return A, B, bias, old


def lay(X, mn, strided):
    """Store the logical [rows, K] operand K-major ([rows, ld]) or MN-major ([K, ld]) in bf16 with NaN in the gap columns; returns the view."""
    X = X.t() if mn else X
    R, C = X.shape
    buf = torch.full((R, _pad8(C) + (8 if strided else 0)), NAN, dtype=F64, device="cuda")
    buf[:, :C] = X
    return buf.to(BF16)[:, :C]


def compare(name, got, ref, tol, report):
    """got: kernel output (bf16 or fp32), ref / tol float64.  tol None: exact (value equality, ±0 alike).  Returns the worst err / bound."""
    g = got.to(F64)
    if tol is None:
        if got.dtype == BF16:
            ref = _bf(ref)
        bad = ~(g == ref)
        worst = 0.0
    else:
        err = (g - ref).abs()
        bad = ~(err <= tol)
        ratio = torch.where(err == 0, torch.zeros_like(err), err / tol).nan_to_num(float("inf"), float("inf"), 0.0)
        worst = float(ratio.max()) if ratio.numel() else 0.0
    report[name] = max(worst, report.get(name, 0.0))
    nbad = int(bad.sum())
    if nbad:
        i = tuple(int(t) for t in torch.nonzero(bad)[0])
        raise AssertionError(f"{name}: {nbad} / {bad.numel()} elements wrong; first at {i}: got {g[i].item()!r} want {ref[i].item()!r}"
                             + ("" if tol is None else f" bound {tol[i].item():.3g}, max err/bound {worst:.3g}"))
    return worst


def untouched(name, before, after, keep):
    """Bits of `after` equal `before` wherever keep is False (the gap columns and the rows the kernel must not store)."""
    iv = torch.int16 if before.dtype == BF16 else torch.int32
    diff = (before.view(iv) != after.view(iv)) & ~keep
    n = int(diff.sum())
    assert n == 0, f"{name}: {n} elements outside the output changed; first at {tuple(int(t) for t in torch.nonzero(diff)[0])}"


def run_dense(M, N, K, a_mn, b_mn, kind, epi="plain", bias=False, strided=True, splits=1, m_dev=None, k_dev=None, seed=0):
    """One lmod_gemm_bf16(_dyn) call against float64.  epi: "plain" (bf16 D), "accumulate" (D = bf16(D_old + acc)), "f32" (D32 += acc,
    split-K with splits > 1).  m_dev / k_dev: device extents; A rows at or past m_dev are NaN; for k_dev, A is zero on
    [k_dev, round_up(k_dev, 64)) and both operands NaN from there on.  Returns (worst err / bound, tile width)."""
    from llavamod import kernels as Kk
    gen = torch.Generator(device="cuda").manual_seed(seed * 7919 + M * 31 + N * 7 + K)
    A, B, bvec, old = operands(kind, M, N, K, gen)
    m_eff = M if m_dev is None else max(0, min(M, m_dev))
    k_eff = K if k_dev is None else max(0, min(K, k_dev))
    if k_dev is not None:
        k_read = min(K, (k_eff + 63) // 64 * 64)
        A[:, k_eff:k_read] = 0.0
        A[:, k_read:] = NAN
        B[:, k_read:] = NAN
    if m_dev is not None:
        A[m_eff:] = NAN
    m_store = M if m_dev is None else min(M, (m_eff + 127) // 128 * 128)
    ref = A[:m_eff, :k_eff] @ B[:, :k_eff].t()
    maj = A[:m_eff, :k_eff].abs() @ B[:, :k_eff].abs().t()
    extra = torch.zeros_like(ref)
    if bias:
        ref, maj = ref + bvec, maj + bvec.abs()
    if epi in ("accumulate", "f32"):
        ref, maj = ref + old[:m_eff], maj + old[:m_eff].abs()
        extra = 2.0 ** -23 * ref.abs()
    if epi == "f32":
        extra = extra + splits * 2.0 ** -23 * maj
    a, b = lay(A, a_mn, strided), lay(B, b_mn, strided)
    ldd = N + (8 if strided else 0)
    dyn = dict(m_dev=None if m_dev is None else torch.tensor([m_dev], dtype=torch.int32, device="cuda"),
               k_dev=None if k_dev is None else torch.tensor([k_dev], dtype=torch.int32, device="cuda"))
    if epi == "f32":
        buf = torch.full((M + 3, ldd), SENT, dtype=torch.float32, device="cuda")
        buf[:M, :N] = old.float()
        before = buf.clone()
        Kk.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=buf[:M, :N], split_k=splits, **dyn)
    else:
        buf = torch.full((M + 3, ldd), SENT, dtype=BF16, device="cuda")
        if epi == "accumulate":
            buf[:M, :N] = old.to(BF16)
        before = buf.clone()
        Kk.gemm(a, b, a_mn=a_mn, b_mn=b_mn, bias=bvec.to(BF16) if bias else None, out=buf[:M, :N], accumulate=epi == "accumulate", **dyn)
    torch.cuda.synchronize()
    keep = torch.zeros_like(buf, dtype=torch.bool)
    keep[:m_store, :N] = True
    untouched("D", before, buf, keep)
    tol = None if kind in EXACT_KINDS else _gemm_tol(ref, maj, k_eff) + extra
    report = {}
    worst = compare("D", buf[:m_eff, :N], ref, tol, report)
    bn = pick_bn(-(-M // 128) * splits, N)
    return worst, bn


def _print(tag, worst, bn):
    print(f"\nGEMMEXACT {tag}: BN={bn} worst err/bound {worst:.3g}")


# ---- layouts x tile widths: all five kinds, strided operands and outputs, bias ------------------------------------------------------
# (M, N, K): N <= 128 takes 256-wide tiles; a small 520-wide problem 128-wide ones; (1700, 3600) fills 1.5 waves of 132 SMs with
# 256-wide tiles (test_layout_grid_covers_both_tile_widths asserts the mix on the device the suite runs on)
GRID = [(129, 120, 200), (300, 520, 200), (1700, 3600, 136)]


def test_layout_grid_covers_both_tile_widths():
    widths = {pick_bn(-(-M // 128), N) for (M, N, K) in GRID}
    assert widths == {128, 256}, widths


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("M,N,K", GRID)
def test_layouts_and_tile_widths(M, N, K, a_mn, b_mn, kind):
    worst, bn = run_dense(M, N, K, a_mn, b_mn, kind, bias=not a_mn)
    _print(f"grid {M}x{N}x{K} a_mn={a_mn} b_mn={b_mn} {kind}", worst, bn)


# ---- M / N / K tails -----------------------------------------------------------------------------------------------------------------
TAILS = ([(m, 264, 200) for m in (1, 127, 129, 3 * 128 + 1, 2 * 128 + 64, 2 * 128 + 127)]
         + [(200, n, 136) for n in (8, 136, 256 + 8, 512 + 128, 256 + 248)]
         + [(200, 264, k) for k in (8, 16, 48)])


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("M,N,K", TAILS)
def test_tails(M, N, K, a_mn, b_mn, kind):
    worst, bn = run_dense(M, N, K, a_mn, b_mn, kind)
    _print(f"tail {M}x{N}x{K} a_mn={a_mn} b_mn={b_mn} {kind}", worst, bn)


# ---- k-block counts with >= 3 tiles per CTA: the 4- and 6-stage rings wrap inside a tile and the phase carries across tiles ---------
def ring_shape(bn, nk):
    """A problem of about three tiles per CTA at the given width on this device: BN = 256 takes 3 M tiles x SMs N tiles; BN = 128 one M
    tile x (2j + 1) N tiles with j + 1 256-wide tiles just under 1.5 waves."""
    sms = _sms()
    if bn == 256:
        return 3 * 128 - 5, 256 * sms - 8, 64 * nk
    j = (3 * sms) // 2 - 2
    return 100, 128 * (2 * j + 1), 64 * nk


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("nk", [1, 2, 3, 5, 7, 13])
@pytest.mark.parametrize("bn", [128, 256])
def test_ring_wraps_inside_and_across_tiles(bn, nk, kind):
    M, N, K = ring_shape(bn, nk)
    tiles = -(-M // 128) * -(-N // bn)
    assert pick_bn(-(-M // 128), N) == bn
    assert tiles >= 2 * _sms() + _sms() * 9 // 10, (tiles, _sms())      # at least 90 % of the CTAs run three tiles
    worst, got_bn = run_dense(M, N, K, False, nk % 2 == 0, kind, strided=nk in (3, 7))
    _print(f"ring BN={bn} nk={nk} {M}x{N}x{K} tiles={tiles} {kind}", worst, got_bn)


# ---- epilogues: bias, D = bf16(D_old + acc), fp32 D32 += acc, split-K -----------------------------------------------------------------
@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True), (False, True)])
@pytest.mark.parametrize("epi,bias,splits", [("plain", True, 1), ("accumulate", False, 1), ("accumulate", True, 1), ("f32", False, 1),
                                             ("f32", False, 3), ("f32", False, 16)])
def test_epilogues(epi, bias, splits, a_mn, b_mn, kind):
    # K = 7 k-blocks (3 splits do not divide them) or 5 (16 splits: 11 empty ones add nothing)
    M, N, K = 300, 520, 64 * (5 if splits == 16 else 7) - 24
    worst, bn = run_dense(M, N, K, a_mn, b_mn, kind, epi=epi, bias=bias, splits=splits)
    _print(f"epilogue {epi} bias={bias} splits={splits} a_mn={a_mn} b_mn={b_mn} {kind}", worst, bn)


# ---- dynamic extents (lmod_gemm_bf16_dyn): m_dev (forward / dgrad), k_dev (wgrad), NaN past each extent ------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("epi", ["plain", "f32"])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("m_dev", [0, 1, 127, 128, 129, 300, 1000])
def test_dynamic_m(m_dev, b_mn, epi, kind):
    worst, bn = run_dense(300, 264, 200, False, b_mn, kind, epi=epi, splits=3 if epi == "f32" else 1, m_dev=m_dev)
    _print(f"m_dev={m_dev} b_mn={b_mn} {epi} {kind}", worst, bn)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("epi", ["accumulate", "f32"])
@pytest.mark.parametrize("a_mn,b_mn", [(True, True), (False, False)])
@pytest.mark.parametrize("k_dev", [0, 1, 63, 64, 65, 320, 1000])
def test_dynamic_k(k_dev, a_mn, b_mn, epi, kind):
    worst, bn = run_dense(264, 136, 320, a_mn, b_mn, kind, epi=epi, k_dev=k_dev)
    _print(f"k_dev={k_dev} a_mn={a_mn} b_mn={b_mn} {epi} {kind}", worst, bn)


# ---- grouped GEMM (experts): modes 0 (forward), 1 (dgrad), 2 (wgrad) ---------------------------------------------------------------
GROUPS = {
    "one": [256],
    "two_first_empty": [0, 384],
    "two_last_empty": [128, 0],
    "eight_mixed": [128, 0, 256, 128, 0, 0, 384, 128],
    "eight_all_empty": [0] * 8,
}


def _offsets(sizes):
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    return offs


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("groups", list(GROUPS))
@pytest.mark.parametrize("mode", [0, 1])
def test_grouped_row_modes(mode, groups, kind):
    """D[rows_g] = A[rows_g] B[g]^T (mode 0) or A[rows_g] B[g] (mode 1); A rows past offsets[G] are NaN, D rows there a sentinel."""
    from llavamod import kernels as Kk
    sizes = GROUPS[groups]
    G, N, K = len(sizes), 264, 200
    offs = _offsets(sizes)
    R = offs[-1] + 128
    gen = torch.Generator(device="cuda").manual_seed(mode * 100 + G + R)
    A, Bl, _, _ = operands(kind, R, G * N, K, gen)
    A[offs[-1]:] = NAN
    Bg = Bl.view(G, N, K)
    a = lay(A, False, True)
    if mode == 0:
        bbuf = torch.full((G, N, K + 8), NAN, dtype=F64, device="cuda")
        bbuf[:, :, :K] = Bg
        b = bbuf.to(BF16)[:, :, :K]
    else:
        bbuf = torch.full((G, K, N + 8), NAN, dtype=F64, device="cuda")
        bbuf[:, :, :N] = Bg.transpose(1, 2)
        b = bbuf.to(BF16)[:, :, :N]
    buf = torch.full((R, N + 8), SENT, dtype=BF16, device="cuda")
    before = buf.clone()
    offsets = torch.tensor(offs, dtype=torch.int32, device="cuda")
    Kk.grouped_gemm(a, b, buf[:, :N], offsets, mode)
    torch.cuda.synchronize()
    keep = torch.zeros_like(buf, dtype=torch.bool)
    keep[:offs[-1], :N] = True
    untouched("D", before, buf, keep)
    report = {}
    for g in range(G):
        r0, r1 = offs[g], offs[g + 1]
        if r1 == r0:
            continue
        Ag = A[r0:r1]
        ref, maj = Ag @ Bg[g].t(), Ag.abs() @ Bg[g].abs().t()
        compare(f"D group {g}", buf[r0:r1, :N], ref, None if kind in EXACT_KINDS else _gemm_tol(ref, maj, K), report)
    print(f"\nGEMMEXACT grouped mode {mode} {groups} {kind}: worst err/bound {max(report.values(), default=0.0):.3g}")


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("groups", ["one_64", "two_first_empty", "three_middle_empty_64", "eight_last_empty_64", "eight_all_empty"])
def test_grouped_wgrad(groups, accumulate, kind):
    """Mode 2: D[g] (+)= A[rows_g]^T B[rows_g] with 64-aligned group boundaries, as its header allows; rows past offsets[G] are NaN.  A group
    without rows writes zeros (or leaves D_old bit for bit with accumulate)."""
    from llavamod import kernels as Kk
    sizes = {"one_64": [192], "two_first_empty": [0, 256], "three_middle_empty_64": [64, 0, 320],
             "eight_last_empty_64": [64, 128, 192, 64, 0, 128, 64, 0], "eight_all_empty": [0] * 8}[groups]
    G, M, N = len(sizes), 200, 136
    offs = _offsets(sizes)
    R = offs[-1] + 64
    gen = torch.Generator(device="cuda").manual_seed(G * 10 + R + accumulate)
    At, Bt, _, old = operands(kind, M, N, R, gen)                     # A^T [M, R], B^T [N, R]: the reduction runs over the rows
    At[:, offs[-1]:] = NAN
    Bt[:, offs[-1]:] = NAN
    a, b = lay(At, True, True), lay(Bt, True, True)                    # stored [R, M] and [R, N]
    olds = torch.stack([old * (g + 1) % 61 for g in range(G)]) if kind in EXACT_KINDS else _bf(torch.stack([old] * G))
    buf = torch.full((G, M, N + 8), SENT, dtype=BF16, device="cuda")
    if accumulate:
        buf[:, :, :N] = olds.to(BF16)
    before = buf.clone()
    offsets = torch.tensor(offs, dtype=torch.int32, device="cuda")
    Kk.grouped_gemm(a, b, buf[:, :, :N], offsets, 2, accumulate=accumulate)
    torch.cuda.synchronize()
    keep = torch.zeros_like(buf, dtype=torch.bool)
    keep[:, :, :N] = True
    untouched("D", before, buf, keep)
    report = {}
    for g in range(G):
        r0, r1 = offs[g], offs[g + 1]
        ref, maj = At[:, r0:r1] @ Bt[:, r0:r1].t(), At[:, r0:r1].abs() @ Bt[:, r0:r1].abs().t()
        if accumulate:
            ref, maj = ref + olds[g], maj + olds[g].abs()
        exact = kind in EXACT_KINDS or r1 == r0
        tol = None if exact else _gemm_tol(ref, maj, r1 - r0) + 2.0 ** -23 * ref.abs()
        compare(f"D group {g}", buf[g, :, :N], ref, tol, report)
    print(f"\nGEMMEXACT grouped mode 2 {groups} accumulate={accumulate} {kind}: worst err/bound {max(report.values(), default=0.0):.3g}")


# ---- fused forms at the tails, bit for bit against the unfused chain, with every output NaN-prefilled ---------------------------------
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rnd(gen, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=gen) * scale).to(BF16)


def _bits_equal(name, got, want):
    assert got.shape == want.shape, (name, got.shape, want.shape)
    diff = got.view(torch.int16) != want.view(torch.int16)
    n = int(diff.sum())
    assert n == 0, f"{name}: {n} / {got.numel()} elements differ in bits; first at {tuple(int(t) for t in torch.nonzero(diff)[0])}"


@pytest.mark.parametrize("M", [1, 127, 128, 129, 255, 256, 257, 300])
def test_fused_swiglu_tails(M):
    from llavamod import kernels as Kk
    H, I = 200, 128
    g = _gen(M)
    x, w = _rnd(g, M, H), _rnd(g, 2 * I, H, scale=0.1)
    with poisoned_uninitialised_memory():
        act = Kk.gemm_swiglu(x, w)
        act_ref = Kk.silu_mul(Kk.gemm(x, w))
    _bits_equal("act", act, act_ref)
    assert bool(torch.isfinite(act).all())


QKV = [(300, 200, 4, 2, 64), (300, 200, 2, 1, 128), (2560, 136, 16, 16, 64), (2560, 136, 8, 8, 128), (129, 64, 3, 1, 64)]


def test_qkv_rope_cases_cover_both_widths():
    for hd in (64, 128):
        assert {pick_bn(-(-M // 128), (nh + 2 * nkv) * d) for M, _, nh, nkv, d in QKV if d == hd} == {128, 256}, hd


@pytest.mark.parametrize("M,H,nh,nkv,hd", QKV)
def test_fused_qkv_rope_tails(M, H, nh, nkv, hd):
    from llavamod import kernels as Kk
    from llavamod.model.language_model.qwen2_core import rope_tables
    N, max_pos = (nh + 2 * nkv) * hd, 4096
    g = _gen(M + hd + nh)
    x, w, b = _rnd(g, M, H), _rnd(g, N, H, scale=0.1), _rnd(g, N)
    pos = torch.randint(0, max_pos, (M,), device="cuda", generator=g)
    pos[::3] = 0
    pos[1::3] = max_pos - 1
    cos, sin = rope_tables(hd, max_pos, 1e6, BF16, "cuda")
    with torch.no_grad(), poisoned_uninitialised_memory():
        fused = Kk.qkv_rope(x, w, b, cos, sin, pos, nh, nkv, hd)
        two = Kk.rope_(Kk.gemm(x, w, bias=b), cos, sin, pos, nh, nkv, hd)
    _bits_equal("qkv", fused, two)
    assert bool(torch.isfinite(fused).all())
    print(f"\nGEMMEXACT qkv_rope M={M} N={N} hd={hd}: BN={pick_bn(-(-M // 128), N)}")


@pytest.mark.parametrize("sizes,I", [([128, 0, 256], 128), ([0, 384], 256), ([128, 0, 128, 0, 0, 256, 128, 0], 128)])
def test_fused_grouped_swiglu_forms(sizes, I):
    """Grouped SwiGLU forward on expert groups (empty first, middle, last): bit for bit against the grouped GEMM + silu_mul on the rows
    below offsets[G].  The slab has rows past offsets[G] (NaN in A, not read)."""
    from llavamod import kernels as Kk
    G, H = len(sizes), 200
    offs = _offsets(sizes)
    R = offs[-1] + 128
    g = _gen(G + I + R)
    xp, w_gu = _rnd(g, R, H), _rnd(g, G, 2 * I, H, scale=0.1)
    xp[offs[-1]:] = NAN
    offsets = torch.tensor(offs, dtype=torch.int32, device="cuda")
    n = offs[-1]
    with poisoned_uninitialised_memory():
        act = Kk.grouped_gemm_swiglu(xp, w_gu, offsets, R)
        h1_ref = torch.zeros(R, 2 * I, dtype=BF16, device="cuda")
        Kk.grouped_gemm(xp, w_gu, h1_ref, offsets, 0)
    _bits_equal("act", act[:n], Kk.silu_mul(h1_ref)[:n])
    assert bool(torch.isfinite(act[:n]).all())

