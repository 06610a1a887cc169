"""The e4m3 GEMM (csrc/gemm_fp8.cu: lmod_gemm_e4m3 and its fused q|k|v+RoPE and SwiGLU forms) element by element against float64, at
the tile, ring, promotion and extent edges where a kernel goes wrong, and the quantisers' non-finite rows through it end to end.

Everything is built from e4m3 bytes and fp32 scales; the reference is the float64 product of the dequantised operands, so quantisation
error stays out.  Operand kinds:
  exact      integer codes in [-2, 2], scales s_a = 2^-3 and s_w = 2^-5, small-integer bias: every partial sum of a 512-element promotion
             group is an integer of magnitude at most 2^11, the fp32 promotion adds are exact and so is the epilogue, so the output equals
             ref.to(bf16) with zero tolerance (this leans on the tensor core keeping about 13 fractional bits of its largest addend, DESIGN
             section 4) -- a dropped, doubled or misplaced k-block, a swizzle error, a stale ring stage or an accumulator not reset fails
  onehot     A[m, k] = 1 iff k == (7m + 3) % K, W all 254 finite e4m3 codes, power-of-two scales: D[m, n] is one code times the scales
  codes      A[i, k0] = byte i, W[j, k0] = byte j for all 256 bytes, zeros elsewhere: D[i, j] = a_i w_j exactly in bf16 (two 4-bit
             significands), every code including +-0, the subnormals, +-448 and the NaN bytes (whose rows and columns must be NaN)
  random, maxmag, huge_tiny  as in test_gemm_fp8_gpu.py, within its bound 2^-8 |ref| + ACC_EPS sum|a||w|
Every operand lives in a wider buffer: e4m3 rows of stride K + 16 with NaN bytes (0x7F) in the gap and NaN rows past the last one, the
scales and the bias views of NaN-filled buffers; every output has ldd = N + 8 and three extra rows, all a sentinel that must not change.
Each case prints its worst err / bound; the file prints its wall time."""
import time

import pytest
import torch

from tests.test_gemm_exact_gpu import SENT, compare, ring_shape, untouched
from tests.test_gemm_fp8_gpu import ACC_EPS, _e4m3_operand

pytestmark = pytest.mark.gpu

F64, BF16 = torch.float64, torch.bfloat16
NAN = float("nan")
NAN_BYTE = 0x7F
EXACT_KINDS = ("exact", "onehot")
FINITE_CODES = torch.tensor([c for c in range(256) if c & 0x7F != 0x7F], dtype=torch.uint8)     # 254 codes


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.perf_counter()
    yield
    print(f"\nGEMMFP8EXACT wall time {time.perf_counter() - t0:.1f} s")


def _f64(q):
    return q.view(torch.float8_e4m3fn).to(F64)


def _e4m3(v):
    return v.to(torch.float8_e4m3fn).view(torch.uint8)


# ---- poisoned storage -----------------------------------------------------------------------------------------------------------------
def lay8(q, extra_rows=5):
    """e4m3 bytes [R, K] in a buffer of row stride K + 16 with NaN bytes in the gap and `extra_rows` NaN rows after R; returns the view."""
    R, K = q.shape
    buf = torch.full((R + extra_rows, K + 16), NAN_BYTE, dtype=torch.uint8, device="cuda")
    buf[:R, :K] = q
    return buf[:R, :K]


def in_nan(v, dtype=torch.float32):
    """v as a view 16 bytes into a NaN-filled buffer with NaN after it too (16-byte aligned, as the kernels require of s_w)."""
    off = 16 // torch.empty((), dtype=dtype).element_size()
    buf = torch.full((v.numel() + 2 * off,), NAN, dtype=dtype, device="cuda")
    buf[off:off + v.numel()] = v.to(dtype)
    return buf[off:off + v.numel()]


def out_buf(M, N):
    buf = torch.full((M + 3, N + 8), SENT, dtype=BF16, device="cuda")
    return buf, buf.clone()


def keep_mask(buf, M, N):
    keep = torch.zeros_like(buf, dtype=torch.bool)
    keep[:M, :N] = True
    return keep


def gemm8(aq, sa, wq, sw, bias, D):
    """lmod_gemm_e4m3 on views (row strides passed as they are) into the view D."""
    from llavamod import kernels as Kk
    M, K = aq.shape
    N = wq.shape[0]
    Kk.call("lmod_gemm_e4m3", Kk.ptr(aq), aq.stride(0), Kk.ptr(sa), Kk.ptr(wq), wq.stride(0), Kk.ptr(sw),
            Kk.ptr(bias) if bias is not None else None, Kk.ptr(D), D.stride(0), M, N, K)


# ---- operands ---------------------------------------------------------------------------------------------------------------------------
def operands(kind, M, N, K, gen):
    """(A bytes [M, K], s_a [M], W bytes [N, K], s_w [N], bias [N] bf16) on the GPU."""
    dev = "cuda"
    ri = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, device=dev, generator=gen).float()     # noqa: E731
    bias = ri(-16, 16, N).to(BF16)
    if kind == "exact":
        return (_e4m3(ri(-2, 2, M, K)), torch.full((M,), 2.0 ** -3, device=dev), _e4m3(ri(-2, 2, N, K)),
                torch.full((N,), 2.0 ** -5, device=dev), bias)
    if kind == "onehot":
        a = torch.zeros(M, K, dtype=torch.uint8, device=dev)
        a[torch.arange(M, device=dev), (7 * torch.arange(M, device=dev) + 3) % K] = 0x38            # 1.0
        codes = FINITE_CODES.to(dev)
        w = codes[(torch.arange(N * K, device=dev) * 7 + 11) % codes.numel()].view(N, K)
        sa = torch.exp2(-ri(0, 4, M))
        sw = torch.exp2(-ri(0, 6, N))
        return a, sa, w, sw, bias
    sa = torch.rand(M, device=dev, generator=gen) * 0.02 + 1e-3
    sw = torch.rand(N, device=dev, generator=gen) * 0.01 + 1e-4
    a = _e4m3_operand(M, K, kind, gen)
    w = _e4m3_operand(N, K, "random" if kind == "huge_tiny" else kind, gen)
    return a, sa, w, sw, torch.randn(N, device=dev, generator=gen).to(BF16)


def reference(a, sa, w, sw, bias):
    A, W = _f64(a), _f64(w)
    sc = sa.double()[:, None] * sw.double()[None, :]
    ref, maj = (A @ W.t()) * sc, (A.abs() @ W.abs().t()) * sc
    if bias is not None:
        ref, maj = ref + bias.double(), maj + bias.double().abs()
    return ref, maj


def run(M, N, K, kind, bias=True, seed=0):
    """One poisoned lmod_gemm_e4m3 call against float64; returns the worst err / bound."""
    gen = torch.Generator(device="cuda").manual_seed(seed * 7919 + M * 31 + N * 7 + K)
    a, sa, w, sw, b = operands(kind, M, N, K, gen)
    assert not (bias and kind == "onehot")
    buf, before = out_buf(M, N)
    gemm8(lay8(a), in_nan(sa), lay8(w), in_nan(sw), in_nan(b, BF16) if bias else None, buf[:M, :N])
    torch.cuda.synchronize()
    untouched("D", before, buf, keep_mask(buf, M, N))
    ref, maj = reference(a, sa, w, sw, b if bias else None)
    tol = None if kind in EXACT_KINDS else 2.0 ** -8 * ref.abs() + ACC_EPS * maj + 2.0 ** -126
    name = "D" if kind != "onehot" else f"D (onehot: row m reads W[n, (7m + 3) % {K}])"
    return compare(name, buf[:M, :N], ref, tol, {})


def _print(tag, worst):
    print(f"\nGEMMFP8EXACT {tag}: worst err/bound {worst:.3g}")


# ---- kinds at a few shapes, bias absent and present -----------------------------------------------------------------------------------
# one-hot runs without bias: a code times the scales plus an integer may need more than fp32's 24 bits, and would not be exact
KIND_BIAS = [(k, b) for k in ("exact", "random", "maxmag", "huge_tiny") for b in (False, True)] + [("onehot", False)]


@pytest.mark.parametrize("kind,bias", KIND_BIAS)
@pytest.mark.parametrize("M,N,K", [(129, 264, 208), (300, 520, 1040), (2 * 128 + 127, 1000, 4112)])
def test_kinds(M, N, K, kind, bias):
    _print(f"kinds {M}x{N}x{K} {kind} bias={bias}", run(M, N, K, kind, bias=bias))


# ---- M / N / K tails --------------------------------------------------------------------------------------------------------------------
TAILS = ([(m, 264, 208) for m in (1, 127, 129, 3 * 128 + 1, 2 * 128 + 127)]
         + [(200, n, 208) for n in (8, 136, 264, 520, 1000)]
         + [(200, 264, k) for k in (16, 48, 112, 128, 144, 4112)])


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("M,N,K", TAILS)
def test_tails(M, N, K, kind):
    _print(f"tail {M}x{N}x{K} {kind}", run(M, N, K, kind))


# ---- k-block counts with >= 3 tiles per CTA: promotion groups of 4 k-blocks against a 6-stage ring --------------------------------------
@pytest.mark.parametrize("kind", ["exact", "random", "maxmag"])
@pytest.mark.parametrize("nk", [1, 3, 4, 5, 6, 7, 8, 9, 11, 12, 13, 25])
def test_promotion_and_ring_edges(nk, kind):
    M, N, _ = ring_shape(128, nk)
    K = 128 * nk
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-M // 128) * -(-N // 128)
    assert tiles >= 2 * sms + sms * 9 // 10, (tiles, sms)               # at least 90 % of the CTAs run three tiles
    _print(f"ring nk={nk} {M}x{N}x{K} tiles={tiles} {kind}", run(M, N, K, kind, bias=nk % 2 == 1))


# ---- every code pair ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k0", [0, 127, 128, 511, 512, 1039])
def test_every_code_pair(k0):
    """D[i, j] = e4m3(i) * e4m3(j): every byte against every byte at one k, the rest zero.  Exact in bf16, NaN where either byte is NaN."""
    K = 1040                                                            # 9 k-blocks, the last one 16 wide: k0 = K - 1 sits in the tail
    codes = torch.arange(256, device="cuda").to(torch.uint8)
    a = torch.zeros(256, K, dtype=torch.uint8, device="cuda")
    a[:, k0] = codes
    w = a.clone()
    ones = torch.ones(256, device="cuda")
    buf, before = out_buf(256, 256)
    gemm8(lay8(a), in_nan(ones), lay8(w), in_nan(ones), None, buf[:256, :256])
    torch.cuda.synchronize()
    untouched("D", before, buf, keep_mask(buf, 256, 256))
    v = _f64(codes)
    ref = v[:, None] * v[None, :]
    got = buf[:256, :256]
    nan_ref, nan_got = ref.isnan(), got.isnan()
    wrong_nan = nan_ref != nan_got
    assert not wrong_nan.any(), "NaN in %d places it should not be or missing; first at codes %s" % (
        int(wrong_nan.sum()), [hex(int(t)) for t in torch.nonzero(wrong_nan)[0]])
    compare("D (index = the two codes)", torch.where(nan_got, 0.0, got.double()).to(BF16), torch.where(nan_ref, 0.0, ref), None, {})
    _print(f"codes k0={k0}", 0.0)


# ---- fused forms bit for bit against the unfused chain, at the tails, under the same poisoning ---------------------------------------
QKV_HEADS = [(3, 1, 64), (5, 1, 64), (7, 1, 64), (14, 2, 64), (1, 1, 128), (2, 1, 128), (28, 4, 128)]


def _bits_equal(name, got, want):
    assert got.shape == want.shape, (name, got.shape, want.shape)
    diff = got.view(torch.int16) != want.view(torch.int16)
    n = int(diff.sum())
    assert n == 0, f"{name}: {n} / {got.numel()} elements differ in bits; first at {tuple(int(t) for t in torch.nonzero(diff)[0])}"


def rope_tables_poisoned(hd, max_pos):
    """cos / sin [max_pos, hd] of rope_tables with NaN in every row but 0 and max_pos - 1 (the only positions used)."""
    from llavamod.model.language_model.qwen2_core import rope_tables
    cos, sin = rope_tables(hd, max_pos, 1e6, BF16, "cuda")
    cos[1:max_pos - 1] = NAN
    sin[1:max_pos - 1] = NAN
    return cos, sin


def qkv_fused(a, sa, w, sw, bias, D, nh, nkv, hd, cos, sin, pos):
    from llavamod import kernels as Kk
    M, K = a.shape
    Kk.call("lmod_gemm_e4m3_qkv_rope", Kk.ptr(a), a.stride(0), Kk.ptr(sa), Kk.ptr(w), w.stride(0), Kk.ptr(sw),
            Kk.ptr(bias) if bias is not None else None, Kk.ptr(D), D.stride(0), M, K, nh, nkv, hd, Kk.ptr(cos), Kk.ptr(sin), Kk.ptr(pos))


def swiglu_fused(a, sa, w, sw, act, I):
    from llavamod import kernels as Kk
    M, K = a.shape
    Kk.call("lmod_gemm_e4m3_swiglu", Kk.ptr(a), a.stride(0), Kk.ptr(sa), Kk.ptr(w), w.stride(0), Kk.ptr(sw), Kk.ptr(act), act.stride(0), M, I, K)


@pytest.mark.parametrize("M", [1, 129, 2 * 128 + 127])
@pytest.mark.parametrize("nh,nkv,hd", QKV_HEADS)
def test_fused_qkv_rope_is_bit_identical_to_gemm_then_rope(nh, nkv, hd, M):
    """(3,1,64) N = 320 and (5,1,64) N = 448 end in a partial tile; q|k / v boundaries fall inside tiles and some tiles are v only."""
    from llavamod import kernels as Kk
    N, K, max_pos = (nh + 2 * nkv) * hd, 144, 64
    gen = torch.Generator(device="cuda").manual_seed(nh * 100 + nkv * 10 + hd + M)
    a, sa, w, sw, _ = operands("random", M, N, K, gen)
    bias = torch.randn(N, device="cuda", generator=gen).to(BF16)
    pos = torch.zeros(M, dtype=torch.int64, device="cuda")
    pos[1::2] = max_pos - 1
    cos, sin = rope_tables_poisoned(hd, max_pos)
    av, sav, wv, swv, bv = lay8(a), in_nan(sa), lay8(w), in_nan(sw), in_nan(bias, BF16)
    buf, before = out_buf(M, N)
    qkv_fused(av, sav, wv, swv, bv, buf[:M, :N], nh, nkv, hd, cos, sin, pos)
    two = torch.full((M, N), NAN, dtype=BF16, device="cuda")
    gemm8(av, sav, wv, swv, bv, two)
    with torch.no_grad():
        Kk.rope_(two, cos, sin, pos, nh, nkv, hd)
    torch.cuda.synchronize()
    untouched("qkv", before, buf, keep_mask(buf, M, N))
    _bits_equal("qkv", buf[:M, :N], two)
    assert bool(torch.isfinite(two).all())
    print(f"\nGEMMFP8EXACT qkv_rope M={M} nh={nh} nkv={nkv} hd={hd} N={N}: bit-identical")


@pytest.mark.parametrize("M", [1, 129, 2 * 128 + 127])
@pytest.mark.parametrize("I", [128, 384])
def test_fused_swiglu_is_bit_identical_to_gemm_then_silu_mul(I, M):
    """W [2I, K] (gate rows, then up rows) with NaN rows past 2I; act with ld_act = I + 8 and a sentinel in its gaps."""
    from llavamod import kernels as Kk
    K = 144
    gen = torch.Generator(device="cuda").manual_seed(I + M)
    a, sa, w, sw, _ = operands("random", M, 2 * I, K, gen)
    av, sav, wv, swv = lay8(a), in_nan(sa), lay8(w), in_nan(sw)
    buf, before = out_buf(M, I)
    swiglu_fused(av, sav, wv, swv, buf[:M, :I], I)
    h = torch.full((M, 2 * I), NAN, dtype=BF16, device="cuda")
    gemm8(av, sav, wv, swv, None, h)
    with torch.no_grad():
        want = Kk.silu_mul(h)
    torch.cuda.synchronize()
    untouched("act", before, buf, keep_mask(buf, M, I))
    _bits_equal("act", buf[:M, :I], want)
    assert bool(torch.isfinite(want).all())
    print(f"\nGEMMFP8EXACT swiglu M={M} I={I}: bit-identical")


# ---- alignment of the epilogue's 4-byte reads: refused on the host, before any launch -----------------------------------------------
def test_misaligned_bias_cos_sin_are_refused():
    from llavamod import _C, kernels as Kk
    M, N, K = 8, 384, 128
    a = torch.zeros(M, K, dtype=torch.uint8, device="cuda")
    w = torch.zeros(N, K, dtype=torch.uint8, device="cuda")
    sa, sw = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
    bbuf = torch.zeros(N + 1, dtype=BF16, device="cuda")
    D = torch.zeros(M, N, dtype=BF16, device="cuda")
    with pytest.raises(_C.LmodError, match="4-byte aligned"):
        gemm8(a, sa, w, sw, bbuf[1:], D)
    cos, sin = rope_tables_poisoned(128, 64)
    cbuf = torch.zeros(cos.numel() + 1, dtype=BF16, device="cuda")
    pos = torch.zeros(M, dtype=torch.int64, device="cuda")
    with pytest.raises(_C.LmodError, match="4-byte aligned"):
        qkv_fused(a, sa, w, sw, bbuf[:N], D, 1, 1, 128, cbuf[1:], sin, pos)
    with pytest.raises(_C.LmodError, match="4-byte aligned"):
        qkv_fused(a, sa, w, sw, bbuf[:N], D, 1, 1, 128, cos, cbuf[1:], pos)
    x, wb = torch.zeros(M, K, dtype=BF16, device="cuda"), torch.zeros(N, K, dtype=BF16, device="cuda")
    with pytest.raises(_C.LmodError, match="4-byte aligned"):
        Kk.gemm(x, wb, bias=bbuf[1:])
    with pytest.raises(_C.LmodError, match="4-byte aligned"):
        Kk.call("lmod_gemm_qkv_rope", Kk.ptr(x), K, Kk.ptr(wb), K, Kk.ptr(bbuf), Kk.ptr(D), N, M, K, 1, 1, 128, Kk.ptr(cos), Kk.ptr(cbuf[1:]),
                Kk.ptr(pos))
    gemm8(a, sa, w, sw, bbuf[:N], D)                                    # aligned views still run
    torch.cuda.synchronize()
    assert bool((D == 0).all())


# ---- non-finite rows end to end: a NaN or inf in a row makes that row of every product NaN and leaves the others alone ---------------
def _finite_rows_equal(name, got, want):
    _bits_equal(name, got, want)
    assert bool(torch.isfinite(got).all()), name


def _nan_rows(name, got, rows):
    bad = ~got[rows].isnan()
    assert not bad.any(), f"{name}: rows {rows} must be NaN in every column; {int(bad.sum())} finite elements, first at {torch.nonzero(bad)[0].tolist()}"


def test_quant_rows_then_gemm_with_nan_and_inf_rows():
    from llavamod import kernels as Kk
    M, N, K = 200, 264, 1040
    gen = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(M, K, device="cuda", generator=gen).to(BF16)
    w = Kk.quant_rows((torch.randn(N, K, device="cuda", generator=gen) * 0.03).to(BF16))
    bias = torch.randn(N, device="cuda", generator=gen).to(BF16)
    bad = [3, 130, 199]
    x[3, 500] = NAN
    x[130, 0] = float("inf")
    x[199, K - 1] = float("-inf")
    fin = [i for i in range(M) if i not in bad]
    got = Kk.gemm_fp8(Kk.quant_rows(x), w, bias)
    alone = Kk.gemm_fp8(Kk.quant_rows(x[fin]), w, bias)
    _nan_rows("D", got, bad)
    _finite_rows_equal("D finite rows", got[fin], alone)


def _layer_inputs(H, where, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rows = 150
    x = torch.randn(rows, H, device="cuda", generator=gen).to(BF16)
    res = torch.randn(rows, H, device="cuda", generator=gen).to(BF16)
    wn = (1 + 0.1 * torch.randn(H, device="cuda", generator=gen)).to(BF16)
    bad = [0, 77, 149]
    t = x if where == "x" else res
    t[0, H // 3] = NAN
    t[77, 5] = NAN
    t[149, H - 1] = NAN
    return x, res, wn, bad, [i for i in range(rows) if i not in bad], gen


@pytest.mark.parametrize("where", ["x", "res"])
def test_rmsnorm_quant_then_qkv_rope_with_nan_rows(where):
    from llavamod import kernels as Kk
    H, nh, nkv, hd, max_pos = 256, 5, 1, 64, 64
    N = (nh + 2 * nkv) * hd
    x, res, wn, bad, fin, gen = _layer_inputs(H, where, 21)
    w = Kk.quant_rows((torch.randn(N, H, device="cuda", generator=gen) * 0.05).to(BF16))
    bias = torch.randn(N, device="cuda", generator=gen).to(BF16)
    cos, sin = rope_tables_poisoned(hd, max_pos)
    pos = torch.zeros(x.shape[0], dtype=torch.int64, device="cuda")
    pos[::2] = max_pos - 1

    def qkv(x, res, pos):
        with torch.no_grad():
            a, _ = Kk.rmsnorm_quant(x, wn, 1e-6, res=res)
        out = torch.full((x.shape[0], N), NAN, dtype=BF16, device="cuda")
        qkv_fused(a.q, a.scale, w.q, w.scale, bias, out, nh, nkv, hd, cos, sin, pos)
        return out

    got = qkv(x, res, pos)
    _nan_rows("qkv", got, bad)
    _finite_rows_equal("qkv finite rows", got[fin], qkv(x[fin], res[fin], pos[fin]))


@pytest.mark.parametrize("where", ["x", "res"])
def test_rmsnorm_quant_then_swiglu_with_nan_rows(where):
    from llavamod import kernels as Kk
    H, I = 256, 384
    x, res, wn, bad, fin, gen = _layer_inputs(H, where, 22)
    w = Kk.quant_rows((torch.randn(2 * I, H, device="cuda", generator=gen) * 0.05).to(BF16))

    def act(x, res):
        with torch.no_grad():
            a, _ = Kk.rmsnorm_quant(x, wn, 1e-6, res=res)
        out = torch.full((x.shape[0], I), NAN, dtype=BF16, device="cuda")
        swiglu_fused(a.q, a.scale, w.q, w.scale, out, I)
        return out

    got = act(x, res)
    _nan_rows("act", got, bad)
    _finite_rows_equal("act finite rows", got[fin], act(x[fin], res[fin]))
