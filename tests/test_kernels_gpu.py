"""GPU parity tests: every kernel is called through the C ABI (llavamod._C / llavamod.kernels) and compared with the
CPU oracle (oracle/restated.py) on the same seeded inputs.  Integer outputs must be bit-exact; floating point within the
tolerance written next to each assertion (bf16 outputs: one bf16 ulp of the value plus a small absolute term)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restated as R  # noqa: E402
from tests.helpers import (check_dlogits, check_moe_stages, check_row_out, kl_reference_fp64, moe_reference_fp64,  # noqa: E402
                           moe_run_stages)

BF16_EPS = 2.0 ** -8


def dev():
    return torch.device("cuda:0")


def bf16_close(a, b, rtol=2 * BF16_EPS, atol=1e-6, msg=""):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = err > tol
    assert not bad.any(), f"{msg} mismatch: max err {err.max().item():.3e} at {int(bad.sum())} / {bad.numel()} elems (max tol {tol.max().item():.3e})"


def make_logits(N, V, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    s = (torch.randn(N, V, generator=g) * scale).to(torch.bfloat16)
    t = (torch.randn(N, V, generator=g) * scale + 0.5 * s.float()).to(torch.bfloat16)
    return s, t


def oracle_kl(s, t, labels, B, T, V, w_ce, distill_all=False):
    sl = s.float().view(B, T, -1).requires_grad_(True)
    tl = t.float().view(B, T, -1)
    logp = R.get_logp(sl, V)
    p = R.get_p(tl, V)
    align = R.compute_align_loss(logp, p, labels.view(B, T), distill_all)
    ce = R.shifted_ce(sl[..., :V], labels.view(B, T), V)
    (align + w_ce * ce).backward()
    return align.detach(), ce.detach(), sl.grad.view(B * T, -1)


@pytest.mark.parametrize("B,T,V,w_ce", [(2, 16, 512, 1.0), (1, 24, 4136, 0.0), (2, 8, 151936, 1.0), (1, 7, 1024, 1.0)])
def test_kl_fused_matches_oracle(B, T, V, w_ce):
    from llavamod import kernels as K
    s, t = make_logits(B * T, V, seed=V + T)
    g = torch.Generator().manual_seed(1)
    labels = torch.randint(0, V, (B, T), generator=g)
    labels[:, : T // 3] = -100
    labels[0, T // 2] = -100
    a_ref, ce_ref, g_ref = oracle_kl(s, t, labels, B, T, V, w_ce)
    sd, td, ld = s.to(dev()), t.to(dev()), labels.to(dev()).reshape(-1)
    d = torch.empty_like(sd)
    out4, row_out = K.kl_fused(sd, td, ld, T, V, 1.0, w_ce, False, dlogits=d)
    torch.cuda.synchronize()
    # loss scalars: fp32 math on both sides, different summation order / ex2.approx -> 2e-5 relative
    assert abs(out4[0].item() - a_ref.item()) <= 2e-5 * abs(a_ref.item()) + 1e-6
    assert abs(out4[1].item() - ce_ref.item()) <= 2e-5 * abs(ce_ref.item()) + 1e-6
    # gradient: element-wise against the float64 reference, bound scaled by the two terms the kernel combines (tests/helpers.py)
    ref = kl_reference_fp64(sd, td, ld, T, V, 1.0, w_ce)
    check_dlogits(d, ref, "dlogits")
    check_row_out(row_out, ref)
    assert (g_ref - ref["g"].cpu()).abs().max() <= 1e-5 * g_ref.abs().max()     # the fp32 oracle and the fp64 reference agree
    # in-place (dlogits aliases the student logits) gives the same bytes
    s2 = sd.clone()
    K.kl_fused(s2, td, ld, T, V, 1.0, w_ce, False, dlogits=s2)
    torch.cuda.synchronize()
    assert torch.equal(s2, d)


def test_kl_fused_wide_teacher_row_stride_and_distill_all():
    """teacher vocab 152064 > slice 151936 (Qwen-2-7B teacher, align_trainer.py:473) handled by the row stride."""
    from llavamod import kernels as K
    B, T, V, Vt = 1, 6, 1024, 1152
    s, _ = make_logits(B * T, V, 5)
    _, t = make_logits(B * T, Vt, 6)
    labels = torch.full((B, T), -100)
    labels[0, 3:] = torch.tensor([5, 9, 1000])
    a_ref, ce_ref, g_ref = oracle_kl(s, t[:, :V].contiguous(), labels, B, T, V, 1.0, distill_all=True)
    d = torch.empty(B * T, V, dtype=torch.bfloat16, device=dev())
    out4, _ = K.kl_fused(s.to(dev()), t.to(dev()), labels.to(dev()).reshape(-1), T, V, 1.0, 1.0, True, dlogits=d)
    assert abs(out4[0].item() - a_ref.item()) <= 2e-5 * abs(a_ref.item())
    bf16_close(d, g_ref.to(torch.bfloat16), atol=2e-7, msg="dlogits(distill_all)")


def test_kl_known_answers_and_all_masked():
    from llavamod import kernels as K
    B, T, V = 1, 8, 2048
    labels = torch.arange(T).view(B, T).to(dev())
    z = torch.zeros(B * T, V, dtype=torch.bfloat16, device=dev())
    out4, _ = K.kl_fused(z, z, labels.reshape(-1), T, V, 1.0, 1.0)
    assert abs(out4[0].item() - math.log(V)) < 1e-4              # uniform logits -> log V
    s, _ = make_logits(B * T, V, 3)
    sd = s.to(dev())
    out4, _ = K.kl_fused(sd, sd, labels.reshape(-1), T, V, 1.0, 1.0)
    p = torch.softmax(s.float(), -1)
    ent = -(p * torch.log_softmax(s.float(), -1)).sum(-1).mean()
    assert abs(out4[0].item() - ent.item()) < 2e-5 * ent.item() + 1e-6    # student == teacher -> teacher entropy
    masked = torch.full((B * T,), -100, device=dev())
    out4, _ = K.kl_fused(sd, sd, masked, T, V, 1.0, 1.0)
    assert math.isnan(out4[0].item())                             # 0/0 kept (align_trainer.py:526)


def test_kl_minus_inf_student_logit_is_dropped():
    from llavamod import kernels as K
    B, T, V = 1, 4, 512
    s, t = make_logits(B * T, V, 11)
    s[:, 7] = float("-inf")
    labels = torch.tensor([[3, 4, 5, 6]])
    a_ref, _, _ = oracle_kl(s, t, labels, B, T, V, 0.0)
    out4, _ = K.kl_fused(s.to(dev()), t.to(dev()), labels.to(dev()).reshape(-1), T, V, 1.0, 0.0)
    assert abs(out4[0].item() - a_ref.item()) <= 2e-5 * abs(a_ref.item())


@pytest.mark.parametrize("B,T,V", [(2, 12, 1000), (1, 5, 151936), (3, 9, 4104)])
def test_logp_gather_matches_oracle(B, T, V):
    from llavamod import kernels as K
    Vp = (V + 7) // 8 * 8
    g = torch.Generator().manual_seed(V)
    full = (torch.randn(B, T, Vp, generator=g) * 2).to(torch.bfloat16)
    logits = full[..., :V]
    labels = torch.randint(0, V, (B, T), generator=g)
    labels[:, :2] = -100
    lf = logits.float().clone().requires_grad_(True)
    ref = R.dpo_get_logp(lf, labels)
    gs = torch.randn(B, generator=g)
    (ref * gs).sum().backward()
    ld = full.to(dev())[..., :V]
    seq, tok, lse = K.logp_gather(ld, labels.to(dev()))
    torch.testing.assert_close(seq.cpu(), ref.detach(), rtol=2e-5, atol=2e-4)
    d = torch.empty(B, T, Vp, dtype=torch.bfloat16, device=dev())[..., :V]
    lab_d, gs_d = labels.to(dev()), gs.to(dev())          # keep the device buffers alive across the raw-pointer call
    K.call("lmod_logp_gather_bwd", K.ptr(ld), ld.stride(1), K.ptr(lab_d), B, T, V, K.ptr(lse), K.ptr(gs_d), 0, K.ptr(d), d.stride(1))
    torch.cuda.synchronize()
    bf16_close(d, lf.grad.to(torch.bfloat16), atol=2e-7, msg="dlogits(logp)")


def test_dense_compat_kernels():
    from llavamod import kernels as K
    N, V = 6, 1000
    s, t = make_logits(N, V, 21)
    labels = torch.tensor([-100, 3, 4, -100, 7, 8])
    logp = K.softmax_rows(s.to(dev()), V, True)
    p = K.softmax_rows(t.to(dev()), V, False)
    torch.testing.assert_close(logp.cpu(), torch.log_softmax(s.float(), -1), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(p.cpu(), torch.softmax(t.float(), -1), rtol=1e-4, atol=1e-8)
    loss = K.align_loss_dense(logp, p, labels.to(dev()))
    ref = R.compute_align_loss(torch.log_softmax(s.float(), -1)[None], torch.softmax(t.float(), -1)[None], labels[None])
    assert abs(loss.item() - ref.item()) < 1e-5 * abs(ref.item())


# ---------------------------------------------------------------------------------------------------------------------
# MoE router / scatter / combine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,H,E,cf,padded", [(64, 128, 4, 1.5, True), (333, 256, 4, 1.0, False), (2048, 1024, 4, 1.5, True),
                                             (500, 128, 8, 0.5, False), (16, 64, 2, 2.0, True), (2048, 1024, 4, 1.5, "aligned"),
                                             (700, 128, 4, 0.75, "aligned"), (4096, 2048, 8, 1.5, "aligned"), (20001, 64, 4, 1.25, "aligned"),
                                             (17, 64, 4, 1.5, False), (320, 128, 4, 0.3, "aligned"), (1040, 256, 8, 1.1, "aligned"),
                                             (335, 64, 2, 0.7, False)])
def test_route_scatter_bit_exact(S, H, E, cf, padded):
    from llavamod import kernels as K
    g = torch.Generator().manual_seed(S + E)
    x = torch.randn(S, H, generator=g).to(torch.bfloat16)
    wg = torch.randn(E, H, generator=g) * 0.2
    noise = R.gumbel_noise((S, E), g)
    layout = K.LAYOUT_ALIGNED if padded == "aligned" else (K.LAYOUT_SLABS if padded else K.LAYOUT_COMPACT)
    r = K.moe_route_scatter(x.to(dev()), wg.to(dev()), noise.to(dev()), cf, 0, layout=layout)
    torch.cuda.synchronize()
    logits = r["logits"].cpu()
    torch.testing.assert_close(logits, x.float() @ wg.t(), rtol=1e-4, atol=1e-4)        # fp32 gate GEMV, different sum order
    o = R.top2gating(logits, noise, cf, 0)                                              # oracle on the SAME fp32 logits
    C = o["capacity"]
    assert r["capacity"] == C
    idx = r["idx"].cpu().long()
    assert torch.equal(idx[:, 0], o["idx1"]) and torch.equal(idx[:, 1], o["idx2"])       # bit exact
    row = r["row"].cpu().long()
    keep1, keep2 = row[:, 0] >= 0, row[:, 1] >= 0
    assert torch.equal(keep1, o["keep1"]) and torch.equal(keep2, o["keep2"])
    off = r["offsets"].cpu().long()
    slot1 = row[:, 0] - off[idx[:, 0]]
    slot2 = row[:, 1] - off[idx[:, 1]]
    assert torch.equal(slot1[keep1], o["slot1"][keep1]) and torch.equal(slot2[keep2], o["slot2"][keep2])
    w = r["w"].cpu()
    torch.testing.assert_close(w[:, 0], o["g1"], rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(w[:, 1], o["g2"], rtol=1e-5, atol=1e-7)
    meta = r["meta"].cpu()
    assert abs(meta[0].item() - o["l_aux"].item()) < 1e-5 * abs(o["l_aux"].item())
    assert torch.equal(meta[4:4 + E].long(), o["exp_counts"])
    if padded == "aligned":
        cnt = torch.minimum(torch.bincount(idx[:, 0], minlength=E) + torch.bincount(idx[:, 1], minlength=E), torch.tensor(C))
        assert bool((off % 128 == 0).all()) and torch.equal(off[1:] - off[:-1], (cnt + 127) // 128 * 128)
        assert int(meta[2].item()) == int(cnt.sum()) and int(meta[3].item()) == int(off[-1]) and off[-1] <= r["xp"].shape[0]
        unused = torch.ones(r["xp"].shape[0], dtype=torch.bool)
        unused[torch.cat([row[:, 0][keep1], row[:, 1][keep2]])] = False
        unused[int(off[-1]):] = False                                    # rows past offsets[E] are never read by a GEMM (uninitialised)
        assert bool((r["xp"].cpu()[unused] == 0).all())                  # the op zeroes the alignment rows (inert in the grouped wgrad)
    elif padded:
        assert torch.equal(off, torch.arange(E + 1) * C)
    else:
        cnt = torch.minimum(torch.bincount(idx[:, 0], minlength=E) + torch.bincount(idx[:, 1], minlength=E), torch.tensor(C))
        assert torch.equal(off, torch.cat([torch.zeros(1, dtype=torch.long), cnt.cumsum(0)]))
        assert int(meta[2].item()) == int(cnt.sum())
    xp = r["xp"].cpu()
    assert torch.equal(xp[row[:, 0][keep1]], x[keep1]) and torch.equal(xp[row[:, 1][keep2]], x[keep2])   # token scatter bit exact
    # every kept row is written exactly once
    used = torch.cat([row[:, 0][keep1], row[:, 1][keep2]])
    assert used.unique().numel() == used.numel()


def test_route_scatter_concurrent_streams_do_not_share_state():
    """Two routers in flight on two streams (student on the main stream, a sparse teacher on the side stream): the op owns its scratch
    per call, so both produce what they produce alone (the round-1 kernel shared one grid-barrier word per device)."""
    from llavamod import kernels as K
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(2048, 1024, generator=g).to(torch.bfloat16).to(dev()) for _ in range(2)]
    wg = (torch.randn(4, 1024, generator=g) * 0.2).to(dev())
    noise = R.gumbel_noise((2048, 4), g).to(dev())
    alone = [K.moe_route_scatter(x, wg, noise, 1.5, 0) for x in xs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    both = [None, None]
    for rep in range(20):
        for i, st in enumerate(streams):
            with torch.cuda.stream(st):
                both[i] = K.moe_route_scatter(xs[i], wg, noise, 1.5, 0)
        torch.cuda.synchronize()
        for a, b in zip(alone, both):
            n = int(a["offsets"][-1])
            assert torch.equal(a["row"], b["row"]) and torch.equal(a["offsets"], b["offsets"]) and torch.equal(a["xp"][:n], b["xp"][:n])
            assert torch.equal(a["meta"], b["meta"]) and torch.equal(a["w"], b["w"])


def test_moe_layer_forward_backward_vs_oracle():
    from llavamod import kernels as K
    S, H, I, E, cf = 96, 128, 256, 4, 1.5
    g = torch.Generator().manual_seed(7)
    cfg = R.LMCfg(hidden=H, inter=I, layers=1, heads=4, kv_heads=4, vocab=64, moe_layers=[0], num_experts=E, capacity_factor=cf)
    sd = {}
    pre = "m."
    sd[pre + "gate.wg.weight"] = torch.randn(E, H, generator=g) * 0.3
    for e in range(E):
        sd[pre + f"experts.deepspeed_experts.{e}.gate_proj.weight"] = (torch.randn(I, H, generator=g) * 0.05).to(torch.bfloat16).float()
        sd[pre + f"experts.deepspeed_experts.{e}.up_proj.weight"] = (torch.randn(I, H, generator=g) * 0.05).to(torch.bfloat16).float()
        sd[pre + f"experts.deepspeed_experts.{e}.down_proj.weight"] = (torch.randn(H, I, generator=g) * 0.05).to(torch.bfloat16).float()
    x = torch.randn(S, H, generator=g).to(torch.bfloat16)
    res = torch.randn(S, H, generator=g).to(torch.bfloat16)
    noise = R.gumbel_noise((S, E), g)
    # device side
    xd = x.to(dev()).requires_grad_(True)
    rd = res.to(dev()).requires_grad_(True)
    wg = sd[pre + "gate.wg.weight"].to(dev())
    w_gu = torch.stack([torch.cat([sd[pre + f"experts.deepspeed_experts.{e}.gate_proj.weight"], sd[pre + f"experts.deepspeed_experts.{e}.up_proj.weight"]]) for e in range(E)]).to(torch.bfloat16).to(dev())
    w_dn = torch.stack([sd[pre + f"experts.deepspeed_experts.{e}.down_proj.weight"] for e in range(E)]).to(torch.bfloat16).to(dev())
    grads = dict(wg=torch.zeros_like(wg), w_gu=torch.zeros_like(w_gu), w_dn=torch.zeros_like(w_dn))
    out, l_aux = K.MoEFn.apply(xd, rd, wg, w_gu, w_dn, noise.to(dev()), cf, 0, grads)
    go = torch.randn(S, H, generator=g).to(torch.bfloat16)
    (out.float() * go.to(dev()).float()).sum().add(0.37 * l_aux).backward()
    # oracle side (fp32 on the bf16-rounded values; routing decided from the KERNEL's logits to remove fp32 tie noise)
    xo = x.float().requires_grad_(True)
    ro = res.float().requires_grad_(True)
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    y, la, _ = R.moe_layer(sdo, pre, cfg, xo, noise)
    outo = ro + y
    (outo * go.float()).sum().add(0.37 * la).backward()
    assert abs(l_aux.item() - la.item()) < 1e-4 * abs(la.item())
    bf16_close(rd.grad, ro.grad, rtol=2 * BF16_EPS, atol=1e-6, msg="moe dres")
    # element by element: every stage against the float64 reference from the kernels' previous stage (tests/helpers.py), and MoEFn
    # gives the stage functions' bytes
    zeros = {k: torch.zeros_like(v) for k, v in grads.items()}
    k = moe_run_stages(xd.detach(), rd.detach(), wg, w_gu, w_dn, noise.to(dev()), cf, 0, go.to(dev()), 0.37, zeros, False)
    assert torch.equal(out, k["out"]) and torch.equal(xd.grad, k["dx"])
    for name in ("wg", "w_gu", "w_dn"):
        assert torch.equal(grads[name], k["g_" + name]), name
    ref = moe_reference_fp64(xd.detach(), rd.detach(), wg, w_gu, w_dn, noise, cf, 0, dout=go.to(dev()), g_laux=0.37, old=zeros, k=k)
    check_moe_stages(k, ref, E, zeros)


# ---------------------------------------------------------------------------------------------------------------------
# element-wise / norm / rope / splice / optimizer
# ---------------------------------------------------------------------------------------------------------------------
def test_rmsnorm_fwd_bwd():
    from llavamod import kernels as K
    rows, H = 37, 256
    g = torch.Generator().manual_seed(0)
    x = torch.randn(rows, H, generator=g).to(torch.bfloat16)
    res = torch.randn(rows, H, generator=g).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16)
    xd, rd = x.to(dev()).requires_grad_(True), res.to(dev()).requires_grad_(True)
    y, s = K.rmsnorm(xd, w.to(dev()), 1e-6, res=rd)
    ref_s = (x + res)                                           # bf16 add like the reference's residual add
    ref_y = R.rmsnorm(ref_s, w, 1e-6)
    assert torch.equal(s.cpu(), ref_s) and torch.equal(y.cpu(), ref_y)      # same roundings -> bit exact
    gy = torch.randn(rows, H, generator=g).to(torch.bfloat16)
    gs = torch.randn(rows, H, generator=g).to(torch.bfloat16)
    (y.float() * gy.to(dev()).float()).sum().add((s.float() * gs.to(dev()).float()).sum()).backward()
    so = ref_s.float().requires_grad_(True)
    yo = R.rmsnorm(so, w.float(), 1e-6)
    (yo * gy.float()).sum().add((so * gs.float()).sum()).backward()
    bf16_close(xd.grad, so.grad, rtol=2 * BF16_EPS, atol=1e-3, msg="rmsnorm dx")
    assert torch.equal(xd.grad, rd.grad)


def test_rope_matches_reference_rounding():
    from llavamod import kernels as K
    from llavamod.model.language_model.qwen2_core import rope_tables
    B, T, nh, nkv, hd = 2, 9, 4, 2, 32
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, generator=g).to(torch.bfloat16)
    pos = torch.arange(T).repeat(B)
    cos, sin = R.rope_cache(hd, 64, 1e6, torch.bfloat16)
    q = qkv[:, : nh * hd].view(B, T, nh, hd).transpose(1, 2)
    k = qkv[:, nh * hd:(nh + nkv) * hd].view(B, T, nkv, hd).transpose(1, 2)
    qr, kr = R.apply_rope(q, k, cos, sin, pos.view(B, T))
    cd, sn = rope_tables(hd, 64, 1e6, torch.bfloat16, dev())
    assert torch.equal(cd.cpu(), cos) and torch.equal(sn.cpu(), sin)
    d = qkv.to(dev()).clone()
    K.rope_(d, cd, sn, pos.to(dev()), nh, nkv, hd)
    out = d.cpu()
    assert torch.equal(out[:, : nh * hd].view(B, T, nh, hd).transpose(1, 2), qr)                 # bit exact (same bf16 roundings)
    assert torch.equal(out[:, nh * hd:(nh + nkv) * hd].view(B, T, nkv, hd).transpose(1, 2), kr)
    assert torch.equal(out[:, (nh + nkv) * hd:], qkv[:, (nh + nkv) * hd:])                       # v untouched
    # backward = transpose rotation: <rope(x), y> == <x, rope_bwd(y)>
    y = torch.randn_like(qkv.float()).to(torch.bfloat16)
    yb = y.to(dev()).clone()
    pos_d = pos.to(dev())
    K.call("lmod_rope", K.ptr(yb), yb.shape[1], nh, yb.data_ptr() + nh * hd * 2, yb.shape[1], nkv, hd, K.ptr(cd), K.ptr(sn), K.ptr(pos_d), B * T, 1)
    lhs = (out[:, :(nh + nkv) * hd].float() * y[:, :(nh + nkv) * hd].float()).sum()
    rhs = (qkv[:, :(nh + nkv) * hd].float() * yb.cpu()[:, :(nh + nkv) * hd].float()).sum()
    assert abs(lhs - rhs) < 2e-2 * abs(lhs) + 0.5


def test_silu_mul_gelu_layernorm():
    from llavamod import kernels as K
    rows, I = 19, 64
    g = torch.Generator().manual_seed(2)
    gu = torch.randn(rows, 2 * I, generator=g).to(torch.bfloat16)
    gd = gu.to(dev()).requires_grad_(True)
    out = K.silu_mul(gd)
    ref = torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]
    assert torch.equal(out.cpu(), ref) or (out.cpu().float() - ref.float()).abs().max() <= 2 * BF16_EPS * ref.float().abs().max()
    go = torch.randn(rows, I, generator=g).to(torch.bfloat16)
    (out.float() * go.to(dev()).float()).sum().backward()
    gf = gu.float().requires_grad_(True)
    (torch.nn.functional.silu(gf[:, :I]) * gf[:, I:] * go.float()).sum().backward()
    bf16_close(gd.grad, gf.grad, rtol=2 * BF16_EPS, atol=1e-3, msg="silu_mul bwd")
    x = torch.randn(rows, I, generator=g).to(torch.bfloat16)
    xd = x.to(dev()).requires_grad_(True)
    y = K.gelu(xd)
    bf16_close(y, torch.nn.functional.gelu(x.float()), atol=1e-3, msg="gelu")
    (y.float() * go.to(dev()).float()).sum().backward()
    xf = x.float().requires_grad_(True)
    (torch.nn.functional.gelu(xf) * go.float()).sum().backward()
    bf16_close(xd.grad, xf.grad, atol=1e-3, msg="gelu bwd")
    q = K.bias_act(x.to(dev()), None, K.ACT_QUICK_GELU)
    bf16_close(q, x.float() * torch.sigmoid(1.702 * x.float()), atol=1e-3, msg="quick_gelu")
    w = torch.randn(I, generator=g).to(torch.bfloat16)
    b = torch.randn(I, generator=g).to(torch.bfloat16)
    ln = K.layernorm(x.to(dev()), w.to(dev()), b.to(dev()), 1e-5)
    bf16_close(ln, torch.nn.functional.layer_norm(x.float(), (I,), w.float(), b.float(), 1e-5), atol=2e-3, msg="layernorm")


def test_splice_gather_and_plan_bit_exact():
    from llavamod import kernels as K
    from llavamod.model.llava_arch import splice_plan
    g = torch.Generator().manual_seed(3)
    B, Tt, V, H, P = 3, 14, 50, 64, 4
    ids = torch.randint(0, V, (B, Tt), generator=g)
    ids[0, 2] = -200; ids[2, 0] = -200; ids[2, 9] = -200
    mask = torch.ones(B, Tt, dtype=torch.bool); mask[1, 10:] = False
    labels = ids.clone(); labels[:, :4] = -100
    for side in ("right", "left"):
        o = R.splice_plan(ids, mask, labels, P, side)
        p = splice_plan(ids.numpy(), mask.numpy(), labels.numpy(), P, side)
        for a, b in zip(o, p):
            a = a.clone()
            if a.dtype == torch.int64:
                a[a == -(1 << 40)] = -(1 << 40)
            assert torch.equal(a, torch.from_numpy(b)), side                                  # integer plan bit exact
    src, nl, nm, pos, img = [torch.from_numpy(a) for a in splice_plan(ids.numpy(), mask.numpy(), labels.numpy(), P)]
    emb = torch.randn(V, H, generator=g).to(torch.bfloat16)
    feats = torch.randn(4, P, H, generator=g).to(torch.bfloat16)
    ref = R.splice_embed(emb, feats, src, img)
    fd = feats.to(dev()).requires_grad_(True)
    out = K.splice_embed(fd, emb.to(dev()), src.to(dev()), img.to(dev()), P)
    assert torch.equal(out.cpu(), ref)
    go = torch.randn_like(ref.float()).to(torch.bfloat16)
    (out.float() * go.to(dev()).float()).sum().backward()
    ff = feats.float().requires_grad_(True)
    (R.splice_embed(emb.float(), ff, src, img) * go.float()).sum().backward()
    assert torch.equal(fd.grad.cpu().float(), ff.grad)


def test_adamw_matches_oracle():
    from llavamod import kernels as K
    n = 1000
    g = torch.Generator().manual_seed(4)
    p = torch.randn(n, generator=g)
    m, v = torch.zeros(n), torch.zeros(n)
    pd, md, vd = p.to(dev()), m.to(dev()), v.to(dev())
    model = torch.empty(n, dtype=torch.bfloat16, device=dev())
    for step in range(1, 4):
        grad = (torch.randn(n, generator=g) * 3).to(torch.bfloat16)
        gs = 0.125
        geff = grad.float() * gs
        total = R.clip_grad_norm([geff], 1.0)
        R.adamw_step([p], [geff], [m], [v], step, 1e-3, wd=0.01)
        nsq = torch.zeros(1, device=dev())
        K.sumsq_(grad.to(dev()), nsq)
        assert abs(math.sqrt(nsq.item()) * gs - total.item()) < 1e-3 * total.item()
        K.adamw_(pd, md, vd, grad.to(dev()), model, 1e-3, 0.9, 0.999, 1e-8, 0.01, step, nsq, 1.0, gs)
        torch.testing.assert_close(pd.cpu(), p, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(model.cpu(), p.to(torch.bfloat16), rtol=2 * BF16_EPS, atol=1e-6)
