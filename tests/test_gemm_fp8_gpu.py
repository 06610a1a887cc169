"""The e4m3 GEMM (csrc/gemm_fp8.cu) element by element against the float64 product of the dequantised operands, so that quantisation
error is excluded and only the accumulation and the final bf16 rounding remain; its fused forms bit for bit against the unfused chain.

Bound: |got - ref| <= 2^-8 |ref| + ACC_EPS * sum_k |a||w| (scaled).  2^-8 |ref| covers the bf16 store; ACC_EPS the accumulator.  The test
prints, per case, the largest (err - 2^-8 |ref|) / sum|a||w| it saw for the e4m3 kernel and for the bf16 kernel on the same values, and
the errors in units of a bf16 ulp of the result; README / DESIGN carry the numbers measured on an H100."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# Accumulator bound, relative to the majorant sum_k |a_k||w_k|.  Hopper's 8-bit MMA truncates its running sum at about 13 fractional bits
# of the largest addend; the kernel therefore promotes the tensor core's partial sum to fp32 registers every 512 elements.  Measured on
# an H100 (80 GB HBM3, 700 W) over the cases below, as (err - 2^-8 |ref|) / majorant: random operands <= 1.1e-4, all-positive
# max-magnitude products 1.2e-3 (K = 4096) to 3.3e-3 (K = 18944), one huge and many tiny products <= 2.3e-3; in bf16 ulps of the result
# a mean of 0.5 - 1.1 (random) and 1.0 - 1.6 (max-magnitude) against 0.25 and <= 0.4 for the bf16 kernel on the same values.  Without the
# promotion the max-magnitude rows were off by 1.65e-2 of the majorant (4 ulps) at K = 4096.  2^-7 is twice the largest value measured.
ACC_EPS = 2.0 ** -7

CASES = [(1, 4096, 4096), (8, 12288, 4096), (100, 4096, 11008), (2048, 4096, 4096), (2048, 12288, 4096), (2048, 4096, 11008),
         (100, 1000, 4096), (2048, 1000, 128), (8, 4096, 18944), (2048, 3584, 18944), (100, 4096, 4112), (7, 264, 48)]


def _e4m3_operand(rows, K, kind, gen):
    """e4m3 bytes [rows, K] (uint8) on the GPU."""
    if kind == "random":
        v = torch.randn(rows, K, device="cuda", generator=gen) * 120
    elif kind == "maxmag":                                  # every element +-448, signs alternating: the sum cancels to (nearly) nothing
        v = torch.full((rows, K), 448.0, device="cuda")
        v[:, 1::2] = -448.0
    else:                                                   # one huge product and many tiny ones per row
        v = torch.randn(rows, K, device="cuda", generator=gen).sign() * 2.0 ** -6
        v[:, K // 3] = 448.0
    return v.clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)


def _f64(q):
    return q.view(torch.float8_e4m3fn).to(torch.float64)


def _errors(got, ref, maj):
    err = (got.double() - ref).abs()
    ulp = torch.maximum(ref.abs(), maj / 256 + 2.0 ** -126).log2().floor().sub(7).exp2()     # bf16 ulp of the result (of majorant / 256 where it cancels)
    excess = ((err - 2.0 ** -8 * ref.abs()).clamp(min=0) / maj.clamp(min=1e-300)).max().item()
    return err, (err / ulp).max().item(), (err / ulp).mean().item(), excess


@pytest.mark.parametrize("kind", ["random", "maxmag", "huge_tiny"])
@pytest.mark.parametrize("M,N,K", CASES)
def test_gemm_e4m3_against_float64_of_the_dequantised_operands(M, N, K, kind):
    from llavamod import kernels as Kk
    gen = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a = Kk.Fp8Rows(_e4m3_operand(M, K, kind, gen), torch.rand(M, device="cuda", generator=gen) * 0.02 + 1e-3)
    w = Kk.Fp8Rows(_e4m3_operand(N, K, "random" if kind == "huge_tiny" else kind, gen), torch.rand(N, device="cuda", generator=gen) * 0.01 + 1e-4)
    bias = torch.randn(N, device="cuda", generator=gen).to(torch.bfloat16)
    got = Kk.gemm_fp8(a, w, bias)
    A, W = _f64(a.q), _f64(w.q)
    sc = a.scale.double()[:, None] * w.scale.double()[None, :]
    ref = (A @ W.t()) * sc + bias.double()
    maj = (A.abs() @ W.abs().t()) * sc + bias.double().abs()
    err, max_ulp, mean_ulp, excess = _errors(got, ref, maj)
    # the bf16 kernel on the same values (e4m3 values are exact in bf16; unit scales, no bias), for comparison only
    ones_m, ones_n = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
    ref1, maj1 = A @ W.t(), A.abs() @ W.abs().t()
    got8 = Kk.gemm_fp8(Kk.Fp8Rows(a.q, ones_m), Kk.Fp8Rows(w.q, ones_n))
    got16 = Kk.gemm(a.q.view(torch.float8_e4m3fn).to(torch.bfloat16), w.q.view(torch.float8_e4m3fn).to(torch.bfloat16))
    _, m8, a8, e8 = _errors(got8, ref1, maj1)
    _, m16, a16, e16 = _errors(got16, ref1, maj1)
    print("\nFP8ACC M=%d N=%d K=%d %s: e4m3 max %.2f mean %.3f bf16-ulp, excess/majorant %.3g | bf16 kernel max %.2f mean %.3f, excess/majorant %.3g"
          % (M, N, K, kind, m8, a8, e8, m16, a16, e16))
    tol = 2.0 ** -8 * ref.abs() + ACC_EPS * maj + 2.0 ** -126
    bad = ~(err <= tol)
    assert not bad.any(), "%d / %d out of bound; max excess/majorant %.3g (bound %.3g), max %.2f ulp" % (int(bad.sum()), bad.numel(), excess, ACC_EPS, max_ulp)


def _quantised(M, N, K, seed):
    from llavamod import kernels as Kk
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    return Kk.quant_rows(x), Kk.quant_rows(w), g


@pytest.mark.parametrize("M", [1, 100, 2048])
@pytest.mark.parametrize("nh,nkv,hd,K", [(32, 32, 128, 4096), (28, 4, 128, 3584), (4, 2, 64, 256)])
def test_qkv_rope_form_is_bit_identical_to_gemm_then_rope(M, nh, nkv, hd, K):
    from llavamod import kernels as Kk
    N = (nh + 2 * nkv) * hd
    a, w, g = _quantised(M, N, K, M + N)
    bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    from llavamod.model.language_model.qwen2_core import rope_tables
    cos, sin = rope_tables(hd, 4096, 1e6, torch.bfloat16, "cuda")
    pos = torch.randint(0, 4096, (M,), device="cuda", generator=g)
    fused = Kk.qkv_rope_fp8(a, w, bias, cos, sin, pos, nh, nkv, hd)
    with torch.no_grad():
        want = Kk.rope_(Kk.gemm_fp8(a, w, bias), cos, sin, pos, nh, nkv, hd)
    assert torch.equal(fused, want)


@pytest.mark.parametrize("M", [1, 100, 2048])
@pytest.mark.parametrize("I,K", [(11008, 4096), (18944, 3584), (256, 128)])
def test_swiglu_form_is_bit_identical_to_gemm_then_silu_mul(M, I, K):
    from llavamod import kernels as Kk
    a, w, _ = _quantised(M, 2 * I, K, M + I)
    act = torch.empty(M, I, dtype=torch.bfloat16, device="cuda")
    Kk.call("lmod_gemm_e4m3_swiglu", Kk.ptr(a.q), K, Kk.ptr(a.scale), Kk.ptr(w.q), K, Kk.ptr(w.scale), Kk.ptr(act), I, M, I, K)
    with torch.no_grad():
        want = Kk.silu_mul(Kk.gemm_fp8(a, w))
    assert torch.equal(act, want)


def test_two_concurrent_streams_give_the_bytes_of_one():
    from llavamod import kernels as Kk
    a, w, _ = _quantised(2048, 4096, 4096, 3)
    b, v, _ = _quantised(2048, 4096, 11008, 4)
    one = (Kk.gemm_fp8(a, w), Kk.gemm_fp8(b, v))
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for _ in range(3):
        with torch.cuda.stream(s1):
            r1 = Kk.gemm_fp8(a, w)
        with torch.cuda.stream(s2):
            r2 = Kk.gemm_fp8(b, v)
    torch.cuda.synchronize()
    assert torch.equal(r1, one[0]) and torch.equal(r2, one[1])


def test_bad_arguments_are_refused():
    from llavamod import _C, kernels as Kk
    q = torch.zeros(8, 40, dtype=torch.uint8, device="cuda")
    s = torch.ones(8, device="cuda")
    with pytest.raises(_C.LmodError, match="multiples of 16"):
        Kk.gemm_fp8(Kk.Fp8Rows(q, s), Kk.Fp8Rows(q, s))
