"""wgmma flash-attention forward (lmod_attn_fwd) vs fp32 SDPA on the same bf16 inputs.
Tolerance: P is rounded to bf16 before P*V (as flash-attn 2 does) -> |err| <= 2^-7 * max|out| ; lse within 1e-3."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def ref_attn(qkv, B, T, nh, nkv, hd, causal, scale):
    q = qkv[:, : nh * hd].view(B, T, nh, hd).transpose(1, 2).float()
    k = qkv[:, nh * hd: (nh + nkv) * hd].view(B, T, nkv, hd).transpose(1, 2).float()
    v = qkv[:, (nh + nkv) * hd:].view(B, T, nkv, hd).transpose(1, 2).float()
    rep = nh // nkv
    k = k.repeat_interleave(rep, 1)
    v = v.repeat_interleave(rep, 1)
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = torch.softmax(s, -1) @ v
    return o.transpose(1, 2).reshape(B * T, nh * hd), lse


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
    ref, ref_lse = ref_attn(qkv, B, T, nh, nkv, hd, causal, scale)
    err = (out.float() - ref).abs().max().item()
    assert err <= 2.0 ** -7 * ref.abs().max().item() + 1e-3, err
    torch.testing.assert_close(lse, ref_lse, rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("B,T,nh,nkv,hd,causal", [(2, 384, 4, 2, 64, True), (1, 256, 2, 2, 128, True), (1, 577, 2, 2, 64, False),
                                                  (1, 2048, 4, 4, 128, True), (2, 200, 4, 1, 128, True), (1, 1024, 8, 8, 64, True)])
def test_attn_backward_matches_autograd(B, T, nh, nkv, hd, causal):
    """dq|dk|dv of the wgmma backward vs fp32 autograd of plain attention on the same bf16 inputs: 2% of each gradient's norm
    (P and dS are rounded to bf16 before their tensor-core products, like flash-attn 2)."""
    from llavamod import kernels as K
    g = torch.Generator(device="cuda").manual_seed(T + hd)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    out, lse = K.attention_fwd(qkv.detach(), B, T, nh, nkv, hd, causal, hd ** -0.5, need_lse=True)
    qkv.grad = K.attention_bwd(qkv.detach(), out, go, lse, B, T, nh, nkv, hd, causal, hd ** -0.5)      # our wgmma backward
    torch.cuda.synchronize()
    x = qkv.detach().float().requires_grad_(True)
    ref, _ = ref_attn(x, B, T, nh, nkv, hd, causal, hd ** -0.5)
    ref.backward(go.float())
    for name, sl in (("dq", slice(0, nh * hd)), ("dk", slice(nh * hd, (nh + nkv) * hd)), ("dv", slice((nh + nkv) * hd, None))):
        a, r = qkv.grad[:, sl].float(), x.grad[:, sl]
        rel = (a - r).norm().item() / r.norm().item()
        assert rel < 2e-2, (name, rel)


def test_attn_fn_default_backward_path():
    """AttnFn (what the student uses): our forward + the default backward give gradients that match autograd too."""
    from llavamod import kernels as K
    B, T, nh, nkv, hd = 2, 384, 4, 2, 64
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    out = K.AttnFn.apply(qkv, B, T, nh, nkv, hd, True, None, None, None)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    out.backward(go)
    x = qkv.detach().float().requires_grad_(True)
    ref, _ = ref_attn(x, B, T, nh, nkv, hd, True, hd ** -0.5)
    ref.backward(go.float())
    assert (qkv.grad.float() - x.grad).norm().item() / x.grad.norm().item() < 2e-2


def ref_attn_padded(qkv, B, T, nh, nkv, hd, scale, keep):
    """fp32 attention under the reference's additive 4-D mask (modeling_qwen2.py:1035-1040): causal + key padding, rows with no
    visible key un-masked (HF _unmask_unattended).  keep [B,T] bool."""
    q = qkv[:, : nh * hd].view(B, T, nh, hd).transpose(1, 2).float()
    k = qkv[:, nh * hd: (nh + nkv) * hd].view(B, T, nkv, hd).transpose(1, 2).float().repeat_interleave(nh // nkv, 1)
    v = qkv[:, (nh + nkv) * hd:].view(B, T, nkv, hd).transpose(1, 2).float().repeat_interleave(nh // nkv, 1)
    s = (q @ k.transpose(-1, -2)) * scale
    vis = torch.ones(T, T, dtype=torch.bool, device=s.device).tril()[None, None] & keep[:, None, None, :]
    vis = vis | ~vis.any(-1, keepdim=True)
    s = s.masked_fill(~vis, float("-inf"))
    o = torch.softmax(s, -1) @ v
    return o.transpose(1, 2).reshape(B * T, nh * hd), torch.logsumexp(s, -1)


@pytest.mark.parametrize("hd,T,side", [(64, 200, "right"), (128, 333, "right"), (64, 300, "left"), (128, 130, "left"), (64, 64, "right")])
def test_attn_padded_batch_fwd_bwd_matches_masked_reference(hd, T, side):
    """Padded batches stay on the wgmma kernels (per-row key range): forward, LSE and dq|dk|dv against fp32 attention under the
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
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    pad = K.pad_ranges(keep)
    out, lse = K.attention_fwd(qkv.detach(), B, T, nh, nkv, hd, True, hd ** -0.5, need_lse=True, pad=pad)
    dqkv = K.attention_bwd(qkv.detach(), out, go, lse, B, T, nh, nkv, hd, True, hd ** -0.5, pad=pad)
    torch.cuda.synchronize()
    x = qkv.detach().float().requires_grad_(True)
    ref, ref_lse = ref_attn_padded(x, B, T, nh, nkv, hd, hd ** -0.5, keep)
    ref.backward(go.float())
    assert (out.float() - ref).abs().max().item() <= 2.0 ** -7 * ref.abs().max().item() + 1e-3
    torch.testing.assert_close(lse, ref_lse, rtol=1e-3, atol=1e-3)
    for name, sl in (("dq", slice(0, nh * hd)), ("dk", slice(nh * hd, (nh + nkv) * hd)), ("dv", slice((nh + nkv) * hd, None))):
        a, r = dqkv[:, sl].float(), x.grad[:, sl]
        assert (a - r).norm().item() / r.norm().item() < 2e-2, name
    # the un-padded path and the padded path agree bit for bit on a sample without padding
    out0, _ = K.attention_fwd(qkv.detach()[:T], 1, T, nh, nkv, hd, True, hd ** -0.5)
    assert torch.equal(out0, out[:T])


@pytest.mark.parametrize("hd", [32, 16, 96])
def test_attn_other_head_dims_run_on_the_same_kernels(hd):
    """head dims that are not 64 / 128 (the reference's tiny test shapes) are zero-padded per head, not sent to a library."""
    from llavamod import kernels as K
    B, T, nh, nkv = 2, 150, 4, 2
    g = torch.Generator(device="cuda").manual_seed(hd)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    go = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    out = K.attention(qkv, B, T, nh, nkv, hd, True)
    out.backward(go)
    x = qkv.detach().float().requires_grad_(True)
    ref, _ = ref_attn(x, B, T, nh, nkv, hd, True, hd ** -0.5)
    ref.backward(go.float())
    assert (out.float() - ref).abs().max().item() <= 2.0 ** -7 * ref.abs().max().item() + 1e-3
    assert (qkv.grad.float() - x.grad).norm().item() / x.grad.norm().item() < 2e-2


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
