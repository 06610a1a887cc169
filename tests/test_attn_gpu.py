"""wgmma flash-attention forward (lmod_attn_fwd) and backward (lmod_attn_bwd) against the float64 reference of tests/helpers.py, element
by element: out, lse, dq, dk and dv each within the bound derived there from the kernels' arithmetic (bf16 P and dS before their
tensor-core products, fp32 accumulation, ex2 / lg2 approximations).  tests/test_attn_exact_gpu.py adds tile edges, model shapes and
adversarial masked keys."""
import pytest
import torch

from tests.helpers import attn_reference_fp64, check_attn, check_attn_grads

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,T,nh,nkv,hd,causal", [(1, 128, 2, 2, 64, True), (1, 256, 2, 2, 128, True), (2, 300, 4, 2, 64, True),
                                                  (1, 577, 4, 4, 64, False), (2, 1024, 4, 4, 128, True), (1, 2048, 8, 2, 128, True),
                                                  (3, 64, 2, 1, 128, False), (1, 2048, 16, 16, 64, True)])
def test_attn_fwd_matches_sdpa(B, T, nh, nkv, hd, causal):
    from llavamod import kernels as K
    g = torch.Generator(device="cuda").manual_seed(T + nh + hd)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
    scale = hd ** -0.5
    out, lse = K.attention_fwd(qkv, B, T, nh, nkv, hd, causal, scale, need_lse=True)
    torch.cuda.synchronize()
    ref = attn_reference_fp64(qkv, B, T, nh, nkv, hd, causal, scale)
    check_attn("fwd o", out, ref["o"], ref["o_tol"], T, hd)
    check_attn("fwd lse", lse, ref["lse"], ref["lse_tol"], T)


@pytest.mark.parametrize("B,T,nh,nkv,hd,causal", [(2, 384, 4, 2, 64, True), (1, 256, 2, 2, 128, True), (1, 577, 2, 2, 64, False),
                                                  (1, 2048, 4, 4, 128, True), (2, 200, 4, 1, 128, True), (1, 1024, 8, 8, 64, True)])
def test_attn_backward_matches_autograd(B, T, nh, nkv, hd, causal):
    """dq|dk|dv of the wgmma backward against the analytic float64 gradients on the same bf16 inputs, element by element."""
    from llavamod import kernels as K
    g = torch.Generator(device="cuda").manual_seed(T + hd)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    out, lse = K.attention_fwd(qkv, B, T, nh, nkv, hd, causal, hd ** -0.5, need_lse=True)
    dqkv = K.attention_bwd(qkv, out, go, lse, B, T, nh, nkv, hd, causal, hd ** -0.5)      # our wgmma backward
    torch.cuda.synchronize()
    ref = attn_reference_fp64(qkv, B, T, nh, nkv, hd, causal, hd ** -0.5, dout=go, out_kernel=out, lse_kernel=lse)
    check_attn_grads("bwd", dqkv, ref, T, nh, nkv, hd)


def test_attn_fn_default_backward_path():
    """AttnFn (what the student uses): our forward + the default backward, element by element."""
    from llavamod import kernels as K
    B, T, nh, nkv, hd = 2, 384, 4, 2, 64
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    out = K.AttnFn.apply(qkv, B, T, nh, nkv, hd, True, None, None, None)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    out.backward(go)
    ref = attn_reference_fp64(qkv, B, T, nh, nkv, hd, True, hd ** -0.5, dout=go, out_kernel=out.detach())
    check_attn("AttnFn o", out, ref["o"], ref["o_tol"], T, hd)
    check_attn_grads("AttnFn", qkv.grad, ref, T, nh, nkv, hd)


@pytest.mark.parametrize("hd,T,side", [(64, 200, "right"), (128, 333, "right"), (64, 300, "left"), (128, 130, "left"), (64, 64, "right")])
def test_attn_padded_batch_fwd_bwd_matches_masked_reference(hd, T, side):
    """Padded batches stay on the wgmma kernels (per-row key range): forward, LSE and dq|dk|dv against float64 attention under the
    reference's 4-D mask, incl. the un-masked rows in front of a left-padded sequence and a sample that is all padding."""
    from llavamod import kernels as K
    B, nh, nkv = 4, 4, 2
    g = torch.Generator(device="cuda").manual_seed(T + hd)
    lens = [T, max(1, T // 3), T - 5, 0]
    keep = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        if n:
            if side == "right":
                keep[b, :n] = True
            else:
                keep[b, T - n:] = True
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    pad = K.pad_ranges(keep)
    out, lse = K.attention_fwd(qkv, B, T, nh, nkv, hd, True, hd ** -0.5, need_lse=True, pad=pad)
    dqkv = K.attention_bwd(qkv, out, go, lse, B, T, nh, nkv, hd, True, hd ** -0.5, pad=pad)
    torch.cuda.synchronize()
    ref = attn_reference_fp64(qkv, B, T, nh, nkv, hd, True, hd ** -0.5, keep=keep, dout=go, out_kernel=out, lse_kernel=lse)
    check_attn("padded o", out, ref["o"], ref["o_tol"], T, hd)
    check_attn("padded lse", lse, ref["lse"], ref["lse_tol"], T)
    check_attn_grads("padded", dqkv, ref, T, nh, nkv, hd)
    # the un-padded path and the padded path agree bit for bit on a sample without padding
    out0, _ = K.attention_fwd(qkv[:T], 1, T, nh, nkv, hd, True, hd ** -0.5)
    assert torch.equal(out0, out[:T])


@pytest.mark.parametrize("hd", [32, 16, 96, 80])
def test_attn_other_head_dims_run_on_the_same_kernels(hd):
    """head dims that are not 64 / 128 (the reference's tiny test shapes) are zero-padded per head, not sent to a library.  The reference
    runs on the same zero-padded buffer (the zero columns change no score and give zero output columns), so the bounds of the built
    width apply; the padded columns are sliced away from both sides."""
    from llavamod import kernels as K
    B, T, nh, nkv = 2, 150, 4, 2
    hp = 64 if hd < 64 else 128
    g = torch.Generator(device="cuda").manual_seed(hd)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    out = K.attention(qkv, B, T, nh, nkv, hd, True)
    out.backward(go)

    def widen(t, heads):
        return torch.nn.functional.pad(t.detach().view(B * T, heads, hd), (0, hp - hd)).view(B * T, heads * hp)

    def narrow(t, heads):
        return t.view(B * T, heads, hp)[:, :, :hd].reshape(B * T, heads * hd)

    ref = attn_reference_fp64(widen(qkv, nh + 2 * nkv), B, T, nh, nkv, hp, True, hd ** -0.5, dout=widen(go, nh),
                              out_kernel=widen(out, nh))
    check_attn("other hd o", out, narrow(ref["o"], nh), narrow(ref["o_tol"], nh), T, hd)
    check_attn_grads("other hd", qkv.grad, dict(dqkv=narrow(ref["dqkv"], nh + 2 * nkv), dqkv_tol=narrow(ref["dqkv_tol"], nh + 2 * nkv)),
                     T, nh, nkv, hd)


def test_attn_bwd_throughput_report():
    """Prints TFLOP/s of our backward next to PyTorch's SDPA backward on the same inputs (report only)."""
    import torch.nn.functional as F
    from llavamod import kernels as K
    for (B, T, nh, hd) in [(1, 2048, 16, 64), (1, 2048, 32, 128)]:
        qkv = torch.randn(B * T, 3 * nh * hd, device="cuda").to(torch.bfloat16)
        out, lse = K.attention_fwd(qkv, B, T, nh, nh, hd, True, need_lse=True)
        go = torch.randn_like(out)
        q, k, v = [qkv[:, i * nh * hd:(i + 1) * nh * hd].view(B, T, nh, hd).transpose(1, 2).detach().requires_grad_(True) for i in range(3)]
        o_sdpa = F.scaled_dot_product_attention(q, k, v, is_causal=True)
        go_sdpa = go.view(B, T, nh, hd).transpose(1, 2)
        fl = 2.5 * 4.0 * B * nh * T * T * hd * 0.5
        res = []
        for fn in (lambda: K.attention_bwd(qkv, out, go, lse, B, T, nh, nh, hd, True, hd ** -0.5),
                   lambda: torch.autograd.grad(o_sdpa, (q, k, v), go_sdpa, retain_graph=True)):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res.append(fl * 10 / (e0.elapsed_time(e1) * 1e-3) / 1e12)
        print(f"attn bwd T{T} nh{nh} hd{hd}: lmod wgmma {res[0]:.0f} TFLOP/s, torch SDPA {res[1]:.0f} TFLOP/s")


def test_attn_throughput_report():
    """Prints TFLOP/s of our forward next to PyTorch's SDPA forward on the same inputs (report only)."""
    import torch.nn.functional as F
    from llavamod import kernels as K
    for (B, T, nh, hd, causal) in [(1, 2048, 32, 128, True), (1, 2048, 16, 64, True), (1, 577, 16, 64, False), (4, 4096, 32, 128, True)]:
        qkv = torch.randn(B * T, 3 * nh * hd, device="cuda").to(torch.bfloat16)
        q, k, v = [qkv[:, i * nh * hd:(i + 1) * nh * hd].view(B, T, nh, hd).transpose(1, 2) for i in range(3)]
        fl = 4.0 * B * nh * T * T * hd * (0.5 if causal else 1.0)
        res = []
        for fn in (lambda: K.attention_fwd(qkv, B, T, nh, nh, hd, causal), lambda: F.scaled_dot_product_attention(q, k, v, is_causal=causal)):
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res.append(fl * 10 / (e0.elapsed_time(e1) * 1e-3) / 1e12)
        print(f"attn fwd B{B} T{T} nh{nh} hd{hd} causal={causal}: lmod wgmma {res[0]:.0f} TFLOP/s, torch SDPA {res[1]:.0f} TFLOP/s")
