"""wgmma/TMA GEMM (lmod_gemm_bf16 / lmod_grouped_gemm_bf16) vs an fp32 reference of the same bf16 inputs.
Tolerance: the reference accumulates in fp32 as the kernel does (registers), so the only difference is the summation order and the
final bf16 rounding: |err| <= 2^-8 * |ref| + 2^-8 * sqrt(K) * 2e-2."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def ref_mm(a, b, a_mn, b_mn):
    A = a.float().t() if a_mn else a.float()
    B = b.float() if b_mn else b.float().t()
    return A @ B


def check(out, ref, K, extra=0.0):
    err = (out.float() - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + 2.0 ** -8 * (K ** 0.5) * 2e-2 + extra
    assert bool((err <= tol).all()), f"max err {err.max().item():.4e} (tol {tol.max().item():.4e}), bad {(err > tol).sum().item()} / {err.numel()}"


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 256), (300, 520, 200), (2048, 1024, 1024), (577, 3072, 1024), (64, 8, 72)])
def test_gemm_all_layouts(M, N, K, a_mn, b_mn):
    from llavamod import kernels as Kk
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    pad = lambda n: (n + 7) // 8 * 8          # noqa: E731  row strides must be multiples of 8
    a = torch.randn((K, pad(M)) if a_mn else (M, pad(K)), device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randn((K, pad(N)) if b_mn else (N, pad(K)), device="cuda", generator=g).to(torch.bfloat16)
    a = a[:, :M] if a_mn else a[:, :K]
    b = b[:, :N] if b_mn else b[:, :K]
    out = Kk.gemm(a, b, a_mn=a_mn, b_mn=b_mn)
    torch.cuda.synchronize()
    check(out, ref_mm(a, b, a_mn, b_mn), K)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(2048, 4096, 512), (1900, 3904, 520), (2048, 1024, 2816), (5632, 1024, 2048), (2048, 3072, 1024), (1990, 1000, 520)])
def test_gemm_two_cta_path(M, N, K, a_mn, b_mn):
    """Large problems (what used to run on a two-CTA kernel): 128x256 or 128x128 tiles depending on how well they fill the SMs, with a
    bias epilogue and the fp32-accumulate output."""
    from llavamod import kernels as Kk
    g = torch.Generator(device="cuda").manual_seed(M + N + K + 1)
    pad = lambda n: (n + 7) // 8 * 8          # noqa: E731
    a = torch.randn((K, pad(M)) if a_mn else (M, pad(K)), device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randn((K, pad(N)) if b_mn else (N, pad(K)), device="cuda", generator=g).to(torch.bfloat16)
    a = a[:, :M] if a_mn else a[:, :K]
    b = b[:, :N] if b_mn else b[:, :K]
    bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    out = Kk.gemm(a, b, a_mn=a_mn, b_mn=b_mn, bias=bias)
    torch.cuda.synchronize()
    check(out, ref_mm(a, b, a_mn, b_mn) + bias.float(), K)
    acc = torch.zeros(M, N, device="cuda")
    Kk.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=acc)
    torch.testing.assert_close(acc, ref_mm(a, b, a_mn, b_mn), rtol=1e-4, atol=2e-2)


@pytest.mark.parametrize("M,H,I", [(2048, 512, 2816 + 128 * 10), (300, 256, 384), (2048, 1024, 2816)])
def test_gemm_fused_swiglu_forward_and_backward(M, H, I):
    """One GEMM with the SwiGLU epilogue == GEMM then silu_mul kernel, bit for bit (same bf16 roundings), on the CTA-pair kernel (first
    shape) and the 1-CTA kernel; the saved pre-activations equal the plain GEMM output; the dgrad GEMM with the silu-backward epilogue ==
    dgrad GEMM then silu_mul_bwd kernel, bit for bit.  The weight is the fused gate|up matrix as the checkpoint stores it (no re-layout)."""
    from llavamod import kernels as Kk
    g = torch.Generator(device="cuda").manual_seed(9 + M)
    x = torch.randn(M, H, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(2 * I, H, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    w_dn = (torch.randn(H, I, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    act, h1 = Kk.gemm_swiglu(x, w, True)
    h1_ref = Kk.gemm(x, w)
    assert torch.equal(h1, h1_ref)
    assert torch.equal(act, Kk.silu_mul(h1_ref))
    assert torch.equal(Kk.gemm_swiglu(x, w, False)[0], act)
    ref = torch.nn.functional.silu(x.float() @ w[:I].float().t()) * (x.float() @ w[I:].float().t())
    # vs the un-rounded fp32 formula: gate, up and silu(gate) are each rounded to bf16 on the way (as in the reference's bf16 modules)
    err = (act.float() - ref).abs()
    assert bool((err <= 2.0 ** -6 * ref.abs() + 0.05).all()), err.max().item()
    dy = (torch.randn(M, H, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    dh1 = Kk.gemm_silu_bwd(dy, w_dn, h1)
    assert torch.equal(dh1, Kk.silu_mul_bwd(Kk.gemm(dy, w_dn, b_mn=True), h1))


@pytest.mark.parametrize("M,H,nh,nkv,hd", [(2048, 1024, 16, 16, 64), (300, 256, 4, 2, 128), (2048, 4096, 32, 32, 128), (257, 128, 2, 1, 64)])
def test_qkv_projection_with_fused_rope(M, H, nh, nkv, hd):
    """q|k|v GEMM with bias + RoPE in the epilogue == GEMM(+bias) followed by the in-place rope kernel, bit for bit (1-CTA and CTA-pair
    kernels, MHA and GQA, both head dims), and its autograd (transpose rotation + dgrad / wgrad / bias grad) == the unfused Functions."""
    from llavamod import kernels as Kk
    from llavamod.model.language_model.qwen2_core import rope_tables
    g = torch.Generator(device="cuda").manual_seed(M + hd)
    N = (nh + 2 * nkv) * hd
    x = torch.randn(M, H, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, H, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    b = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    pos = torch.randint(0, 2048, (M,), device="cuda", generator=g)
    cos, sin = rope_tables(hd, 2048, 1e6, torch.bfloat16, "cuda")
    Kk.FUSE_ROPE = "1"                                     # the model path fuses by reduction length; here the fused op itself is under test
    fused = Kk.qkv_rope(x, w, b, cos, sin, pos, nh, nkv, hd)
    two = Kk.rope_(Kk.gemm(x, w, bias=b), cos, sin, pos, nh, nkv, hd)
    assert torch.equal(fused, two)
    assert torch.equal(Kk.qkv_rope(x, w, None, cos, sin, pos, nh, nkv, hd), Kk.rope_(Kk.gemm(x, w), cos, sin, pos, nh, nkv, hd))
    if M <= 512:
        go = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
        res = []
        for fn in (lambda xx, wg, bg: Kk.qkv_rope(xx, w, b, cos, sin, pos, nh, nkv, hd, wg, bg),
                   lambda xx, wg, bg: Kk.rope_(Kk.linear(xx, w, b, wg, bg), cos, sin, pos, nh, nkv, hd)):
            xx = x.clone().requires_grad_(True)
            wg, bg = torch.zeros_like(w), torch.zeros_like(b)
            fn(xx, wg, bg).backward(go.clone())
            res.append((xx.grad, wg, bg))
        for a, c in zip(res[0], res[1]):
            assert torch.equal(a, c)
    Kk.FUSE_ROPE = "auto"


@pytest.mark.parametrize("M,N,K,bias", [(2048, 4096, 4096, False), (2048, 4096, 11008, False), (2048, 1024, 1024, True), (577, 1024, 4096, True),
                                        (300, 520, 200, True), (1154, 1024, 1024, True)])
def test_gemm_with_residual_epilogue_is_gemm_plus_add(M, N, K, bias):
    """o_proj / down_proj (modeling_qwen2.py:796,808) and CLIP out_proj / fc2 with the residual add in the GEMM epilogue: bit-identical to
    GEMM (+bias, rounded to bf16) followed by the bf16 add kernel -- CTA-pair tiles (teacher shapes), 1-CTA tiles, ragged edges, in place."""
    from llavamod import kernels as Kk
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    b = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16) if bias else None
    res = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    y = Kk.gemm(x, w, bias=b)
    want = torch.empty_like(res)
    Kk.call("lmod_add", Kk.ptr(res), Kk.ptr(y), res.numel(), Kk.ptr(want))
    assert torch.equal(want, (res.float() + y.float()).to(torch.bfloat16))          # the add kernel is the reference's bf16 add
    got = Kk.gemm_residual(x, w, b, res)
    assert torch.equal(got, want)
    r2 = res.clone()
    out = Kk.gemm_residual(x, w, b, r2, inplace=True)
    assert out.data_ptr() == r2.data_ptr() and torch.equal(r2, want)


def test_grouped_swiglu_forward_and_backward():
    """Expert form on ragged 128-aligned row groups (one empty group): fused == grouped GEMM + element-wise kernels, bit for bit."""
    from llavamod import kernels as Kk
    E, H, I = 4, 256, 384
    offs = torch.tensor([0, 256, 256, 640, 768], dtype=torch.int32, device="cuda")
    R = 768 + 128
    g = torch.Generator(device="cuda").manual_seed(5)
    xp = torch.randn(R, H, device="cuda", generator=g).to(torch.bfloat16)
    w_gu = (torch.randn(E, 2 * I, H, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    w_dn = (torch.randn(E, H, I, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    act, h1 = Kk.grouped_gemm_swiglu(xp, w_gu, offs, R, True)
    h1_ref = torch.zeros(R, 2 * I, dtype=torch.bfloat16, device="cuda")
    Kk.grouped_gemm(xp, w_gu, h1_ref, offs, 0)
    n = int(offs[-1])
    assert torch.equal(h1[:n], h1_ref[:n]) and torch.equal(act[:n], Kk.silu_mul(h1_ref)[:n])
    dy = (torch.randn(R, H, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    dh1 = Kk.grouped_gemm_silu_bwd(dy, w_dn, h1, offs, R)
    dact = torch.zeros(R, I, dtype=torch.bfloat16, device="cuda")
    Kk.grouped_gemm(dy, w_dn, dact, offs, 1)
    assert torch.equal(dh1[:n], Kk.silu_mul_bwd(dact, h1_ref)[:n])


def test_mlp_function_gradients_match_autograd():
    """K.mlp (fused forward / backward) against fp32 autograd of the plain formula, incl. the in-place weight-gradient accumulation."""
    from llavamod import kernels as Kk
    M, H, I = 384, 256, 512
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(M, H, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    w_gu = (torch.randn(2 * I, H, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    w_dn = (torch.randn(H, I, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    g_gu, g_dn = torch.zeros_like(w_gu), torch.zeros_like(w_dn)
    go = torch.randn(M, H, device="cuda", generator=g).to(torch.bfloat16)
    Kk.FUSE_SWIGLU = "1"                                   # exercise MLPFn (the model path only fuses frozen MLPs with a long reduction)
    y = Kk.mlp(x, w_gu, w_dn, g_gu, g_dn)
    y.backward(go)
    xf = x.detach().float().requires_grad_(True)
    wg, wd = w_gu.float().requires_grad_(True), w_dn.float().requires_grad_(True)
    yr = (torch.nn.functional.silu(xf @ wg[:I].t()) * (xf @ wg[I:].t())) @ wd.t()
    yr.backward(go.float())
    rel = lambda a, b: ((a.float() - b).norm() / b.norm()).item()
    assert rel(y, yr) < 1e-2 and rel(x.grad, xf.grad) < 1.5e-2 and rel(g_gu, wg.grad) < 1.5e-2 and rel(g_dn, wd.grad) < 1.5e-2
    with torch.no_grad():
        assert torch.equal(Kk.mlp(x.detach(), w_gu, w_dn), y.detach())
    Kk.FUSE_SWIGLU = "auto"


def test_gemm_bias_beta_and_f32_accumulate():
    from llavamod import kernels as Kk
    M, N, K = 384, 768, 320
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    ref = ref_mm(a, b, False, False)
    out = Kk.gemm(a, b, bias=bias)
    check(out, ref + bias.float(), K)
    old = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    out2 = Kk.gemm(a, b, out=old.clone(), accumulate=True)
    check(out2, ref + old.float(), K)
    acc = torch.ones(M, N, device="cuda")
    Kk.gemm(a, b, out_f32=acc)
    torch.testing.assert_close(acc, ref + 1.0, rtol=1e-4, atol=1e-2)


def test_grouped_gemm_modes():
    from llavamod import kernels as Kk
    G, H, I = 4, 256, 512
    rows = [256, 0, 384, 128]
    offs = [0]
    for r in rows:
        offs.append(offs[-1] + r)
    R = offs[-1]
    offsets = torch.tensor(offs, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(R + 128, H, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(G, I, H, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    y = torch.zeros(R + 128, I, device="cuda", dtype=torch.bfloat16)
    Kk.grouped_gemm(x, w, y, offsets, 0)                                   # forward
    for e in range(G):
        if rows[e]:
            check(y[offs[e]:offs[e + 1]], x[offs[e]:offs[e + 1]].float() @ w[e].float().t(), H)
    assert bool((y[R:] == 0).all())                                        # rows beyond the last group untouched
    dy = torch.randn(R + 128, I, device="cuda", generator=g).to(torch.bfloat16)
    dx = torch.zeros(R + 128, H, device="cuda", dtype=torch.bfloat16)
    Kk.grouped_gemm(dy, w, dx, offsets, 1)                                 # dgrad: dx = dy @ w[e]
    for e in range(G):
        if rows[e]:
            check(dx[offs[e]:offs[e + 1]], dy[offs[e]:offs[e + 1]].float() @ w[e].float(), I)
    dw = torch.zeros(G, I, H, device="cuda", dtype=torch.bfloat16)
    Kk.grouped_gemm(dy, x, dw, offsets, 2)                                 # wgrad: dw[e] = dy_e^T @ x_e
    for e in range(G):
        ref = dy[offs[e]:offs[e + 1]].float().t() @ x[offs[e]:offs[e + 1]].float()
        check(dw[e], ref, max(rows[e], 1))
    dw2 = dw.clone()
    Kk.grouped_gemm(dy, x, dw2, offsets, 2, accumulate=True)
    check(dw2[0], 2 * dw[0].float(), rows[0], extra=0.05)


def test_gemm_throughput_report():
    """Not a pass/fail perf gate: prints achieved TFLOP/s of the hand-written kernel next to cuBLAS for the path's big shapes."""
    from llavamod import kernels as Kk
    for (M, N, K) in [(2048, 22016, 4096), (2048, 4096, 11008), (2048, 12288, 4096), (2048, 151936, 1024), (2048, 5632, 1024)]:
        a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        res = []
        for fn in (lambda: Kk.gemm(a, b, out=out), lambda: torch.mm(a, b.t(), out=out)):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res.append(2.0 * M * N * K * 10 / (e0.elapsed_time(e1) * 1e-3) / 1e12)
        print(f"GEMM {M}x{N}x{K}: lmod wgmma {res[0]:.0f} TFLOP/s, cuBLAS {res[1]:.0f} TFLOP/s")
