"""CPU pins of the float64 references of the norm / rotary / activation / splice / embedding-gradient / optimizer kernels (tests/helpers.py):
they agree with the oracle (oracle/restated.py) and with torch autograd of the bf16 formulas, and their bounds catch the defects a subtly
wrong kernel would have -- each planted defect below must fail its check while the unperturbed output passes."""
import math

import pytest
import torch

from oracle import restated as R
from tests.helpers import (BF16_U, accumulate_tol, adamw_reference_fp64, bias_act_reference_fp64, check_bound,
                           embed_grad_reference_fp64, gelu_bwd_reference_fp64, layernorm_reference_fp64, rmsnorm_bwd_reference_fp64,
                           rmsnorm_reference_fp64, rmsnorm_wgrad_reference_fp64, rope_bwd_reference_fp64, silu_mul_reference_fp64,
                           splice_bwd_reference, splice_reference)

bf16 = torch.bfloat16


def fails(fn):
    with pytest.raises(AssertionError):
        fn()


def rand(*shape, seed=0, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(bf16)


def rstd32(s, eps):
    return torch.rsqrt(s.float().pow(2).mean(-1) + eps)       # the fp32 rstd of R.rmsnorm


@pytest.mark.parametrize("H", [64, 1024, 1032])
def test_rmsnorm_reference_matches_oracle_and_catches_defects(H):
    rows, eps = 9, 1e-6
    x, res, w = rand(rows, H, seed=1), rand(rows, H, seed=2), (1 + 0.1 * rand(H, seed=3).float()).to(bf16)
    s = x + res
    r32 = rstd32(s, eps)
    ref = rmsnorm_reference_fp64(x, w, eps, res=res, rstd_k=r32)
    assert torch.equal(ref["s"], s)
    assert torch.equal(ref["y"], R.rmsnorm(s, w, eps))                        # y from the fp32 rstd: the oracle's bytes
    check_bound("rstd", r32, ref["rstd"], ref["rstd_tol"])
    check_bound("y", ref["y"], ref["y"])
    # a row's last 16-byte vector dropped
    y = ref["y"].clone(); y[3, -8:] = 0
    fails(lambda: check_bound("y", y, ref["y"]))
    # H - 8 used as the width
    fails(lambda: check_bound("rstd", rstd32(s[:, :-8], eps), ref["rstd"], ref["rstd_tol"]))
    # a neighbouring row's rstd applied to y
    y = rmsnorm_reference_fp64(x, w, eps, res=res, rstd_k=r32.roll(1))["y"]
    fails(lambda: check_bound("y", y, ref["y"]))


@pytest.mark.parametrize("H", [64, 1024])
def test_rmsnorm_backward_references_match_autograd_and_catch_defects(H):
    rows, eps = 300, 1e-6
    s, w = rand(rows, H, seed=4), (1 + 0.1 * rand(H, seed=5).float()).to(bf16)
    dy, dres = rand(rows, H, seed=6), rand(rows, H, seed=7)
    r32 = rstd32(s, eps)
    # autograd of the bf16 module (w * h.to(bf16)), plus the residual stream's gradient
    sa, wa = s.clone().requires_grad_(True), w.clone().requires_grad_(True)
    R.rmsnorm(sa, wa, eps).backward(dy)
    ref = rmsnorm_bwd_reference_fp64(dy, s, w, r32, dres)
    check_bound("dx (autograd)", sa.grad.double() + dres.double(), ref["dx"], ref["tol"] + ref["tol_g"] + BF16_U * (ref["dx"].abs() + dres.double().abs()))
    ref0 = rmsnorm_bwd_reference_fp64(dy, s, w, r32)
    check_bound("dx (autograd, no dres)", sa.grad, ref0["dx"], ref0["tol"] + ref0["tol_g"])
    old = rand(H, seed=8, scale=0.1)
    wg = rmsnorm_wgrad_reference_fp64(dy, s, r32, old)
    check_bound("wgrad (autograd)", (old.float() + wa.grad.float()).to(bf16), wg["want"], wg["tol"])
    # a kernel that matches the float64 formula passes; dres missing on one 16-byte vector fails
    dx = ref["dx"].to(bf16)
    check_bound("dx", dx, ref["dx"], ref["tol"])
    bad = dx.clone(); bad[5, 8:16] = ref["dx"][5, 8:16].sub(dres[5, 8:16].double()).to(bf16)
    fails(lambda: check_bound("dx", bad, ref["dx"], ref["tol"]))
    # a neighbouring row's rstd in the backward
    fails(lambda: check_bound("dx", rmsnorm_bwd_reference_fp64(dy, s, w, r32.roll(1), dres)["dx"].to(bf16), ref["dx"], ref["tol"]))


def rope_setup(nh, nkv, hd, rows, P, seed):
    qkv = rand(rows, (nh + 2 * nkv) * hd, seed=seed)
    pos = torch.randint(0, P, (rows,), generator=torch.Generator().manual_seed(seed))
    cos, sin = R.rope_cache(hd, P, 1e6, bf16)
    return qkv, pos, cos, sin


def rope_fwd_torch(x, cos, sin, pos, hd, swap_head=None):
    """the kernels' forward written with torch bf16 ops: o1 = bf16(bf16(x1 c) + bf16(-x2 s)), o2 = bf16(bf16(x2 c) + bf16(x1 s))"""
    rows = x.shape[0]
    v = x.view(rows, -1, hd)
    c, s = cos[pos][:, None, : hd // 2], sin[pos][:, None, : hd // 2]
    x1, x2 = v[..., : hd // 2], v[..., hd // 2:]
    if swap_head is not None:
        x1, x2 = x1.clone(), x2.clone()
        x1[:, swap_head], x2[:, swap_head] = v[:, swap_head, hd // 2:], v[:, swap_head, : hd // 2]
    return torch.cat([x1 * c + (-x2) * s, x2 * c + x1 * s], -1).reshape(rows, -1)


@pytest.mark.parametrize("hd", [64, 128])
def test_rope_references_match_oracle_and_autograd(hd):
    nh, nkv, rows, P = 4, 2, 40, 4096
    qkv, pos, cos, sin = rope_setup(nh, nkv, hd, rows, P, hd)
    B, T = 2, rows // 2
    q = qkv[:, : nh * hd].view(B, T, nh, hd).transpose(1, 2)
    k = qkv[:, nh * hd:(nh + nkv) * hd].view(B, T, nkv, hd).transpose(1, 2)
    qr, kr = R.apply_rope(q, k, cos, sin, pos.view(B, T))
    qk = qkv[:, :(nh + nkv) * hd]
    mine = rope_fwd_torch(qk, cos, sin, pos, hd)
    assert torch.equal(mine[:, : nh * hd], qr.transpose(1, 2).reshape(rows, -1))
    assert torch.equal(mine[:, nh * hd:], kr.transpose(1, 2).reshape(rows, -1))
    # q/k halves swapped in one head: the forward's bytes change
    assert not torch.equal(rope_fwd_torch(qk, cos, sin, pos, hd, swap_head=1), mine)
    # backward: autograd of the oracle in bf16 within one ulp of the float64 transpose rotation
    dy = rand(rows, (nh + nkv) * hd, seed=hd + 1)
    qa = q.detach().clone().requires_grad_(True)
    ka = k.detach().clone().requires_grad_(True)
    qo, ko = R.apply_rope(qa, ka, cos, sin, pos.view(B, T))
    (qo.float() * dy[:, : nh * hd].view(B, T, nh, hd).transpose(1, 2).float()).sum().add(
        (ko.float() * dy[:, nh * hd:].view(B, T, nkv, hd).transpose(1, 2).float()).sum()).backward()
    ag = torch.cat([qa.grad.transpose(1, 2).reshape(rows, -1), ka.grad.transpose(1, 2).reshape(rows, -1)], 1)
    ref = rope_bwd_reference_fp64(dy, cos, sin, pos, hd)
    check_bound("rope bwd (autograd)", ag, ref["d"], ref["tol_ag"])
    check_bound("rope bwd", ref["d"].to(bf16), ref["d"], ref["tol"])
    # the sine's sign flipped in the backward
    flipped = rope_bwd_reference_fp64(dy, cos, -sin, pos, hd)["d"].to(bf16)
    fails(lambda: check_bound("rope bwd", flipped, ref["d"], ref["tol"]))
    # q/k halves swapped in one head of the backward
    sw = ref["d"].to(bf16).view(rows, -1, hd).clone()
    sw[:, 2] = sw[:, 2].roll(hd // 2, -1)
    fails(lambda: check_bound("rope bwd", sw.view(rows, -1), ref["d"], ref["tol"]))


def test_activation_references_match_torch():
    rows, I = 16, 64
    g = torch.Generator().manual_seed(9)
    gu = (torch.randn(rows, 2 * I, generator=g) * 4).to(bf16)
    gu[0, :8] = torch.tensor([100, -100, 88, -88, -89, 20, -20, 0.0]).to(bf16)
    ref = silu_mul_reference_fp64(gu, I)
    out = torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]                    # the module: bf16(bf16(silu(g)) u)
    check_bound("silu_mul (torch bf16)", out, ref["out"], ref["out_tol"])
    d = rand(rows, I, seed=10)
    gf = gu.double().requires_grad_(True)
    (torch.nn.functional.silu(gf[:, :I]) * gf[:, I:] * d.double()).sum().backward()
    b = ref["bwd"](d)
    assert torch.allclose(gf.grad[:, :I], b["dg"], rtol=1e-12, atol=1e-300) and torch.allclose(gf.grad[:, I:], b["du"], rtol=1e-12, atol=1e-300)
    x = (torch.randn(rows, I, generator=g) * 3).to(bf16)
    bias = rand(I, seed=11)
    for act, fn in ((0, lambda z: torch.nn.functional.gelu(z)), (1, lambda z: z * torch.sigmoid(1.702 * z)), (2, lambda z: z)):
        for bb in (None, bias):
            ref = bias_act_reference_fp64(x, bb, act)
            z = x if bb is None else x + bb
            check_bound(f"act {act} (torch fp32)", fn(z.float()), ref["y"], ref["tol"])
    xf = x.double().requires_grad_(True)
    torch.nn.functional.gelu(xf).backward(d.double())
    assert torch.allclose(xf.grad, gelu_bwd_reference_fp64(d, x)["dx"], rtol=1e-12, atol=1e-300)


def test_layernorm_reference_matches_torch():
    H = 1024
    x = rand(6, H, seed=12)
    x[1] = (100 + 0.01 * torch.randn(H, generator=torch.Generator().manual_seed(1))).to(bf16)
    x[2] = (100 + 2 * torch.randn(H, generator=torch.Generator().manual_seed(2))).to(bf16)
    w, b = rand(H, seed=13), rand(H, seed=14)
    ref = layernorm_reference_fp64(x, w, b, 1e-5)
    check_bound("layernorm (torch fp32)", torch.nn.functional.layer_norm(x.float(), (H,), w.float(), b.float(), 1e-5), ref["y"], ref["tol"])
    bad = ref["y"].to(bf16).clone(); bad[4, -8:] = 0
    fails(lambda: check_bound("layernorm", bad, ref["y"], ref["tol"]))


def test_splice_references_match_oracle():
    from llavamod.model.llava_arch import splice_plan
    g = torch.Generator().manual_seed(3)
    B, Tt, V, H, P = 3, 20, 50, 64, 4
    ids = torch.randint(0, V, (B, Tt), generator=g)
    ids[0, 2] = -200; ids[1, 5] = -200; ids[1, 11] = -200; ids[2, 0] = -200
    mask = torch.ones(B, Tt, dtype=torch.bool); mask[2, 15:] = False
    src, _, _, _, img = [torch.from_numpy(a) for a in splice_plan(ids.numpy(), mask.numpy(), None, P, "left")]
    emb, feats = rand(V, H, seed=15), rand(4, P, H, seed=16)
    assert torch.equal(splice_reference(emb, feats, src, img, P).view(B, -1, H), R.splice_embed(emb, feats, src, img))
    ff = feats.float().requires_grad_(True)
    d = rand(*src.shape, H, seed=17)
    (R.splice_embed(emb.float(), ff, src, img) * d.float()).sum().backward()
    assert torch.equal(splice_bwd_reference(d, src, img, 4, P).float(), ff.grad)


def test_embed_grad_reference_matches_autograd_and_catches_defects():
    from llavamod.model.llava_arch import embed_grad_order
    g = torch.Generator().manual_seed(18)
    V, H = 300, 64
    src = torch.cat([torch.randperm(V, generator=g)[:40], torch.full((64,), 7), torch.full((8,), 11), torch.full((5,), -3)])
    src = src[torch.randperm(src.numel(), generator=g)].view(3, -1)
    d = rand(src.numel(), H, seed=19).view(3, -1, H)
    old = rand(V, H, seed=20, scale=0.1)
    ref = embed_grad_reference_fp64(d, src, old)
    # nn.Embedding backward (fp32 sums), then the bf16 accumulation into .grad
    w = torch.zeros(V, H, requires_grad=True)
    torch.nn.functional.embedding(src.clamp(min=0), w).mul((src >= 0)[..., None]).backward(d.float())
    got = (old.float() + w.grad.to(bf16).float()).to(bf16)
    check_bound("embed grad (autograd)", got[ref["toks"]], ref["want"], ref["tol"])
    untouched = torch.ones(V, dtype=torch.bool); untouched[ref["toks"]] = False
    assert torch.equal(got[untouched], old[untouched])
    # the order groups rows by token, stable, image / padding rows last
    o = torch.from_numpy(embed_grad_order(src.numpy())).reshape(-1)
    fs = src.reshape(-1)[o]
    n_text = int((src >= 0).sum())
    assert bool((fs[:n_text] >= 0).all()) and bool((fs[n_text:] < 0).all()) and bool((fs[1:n_text] >= fs[:n_text - 1]).all())
    same = fs[1:n_text] == fs[:n_text - 1]
    assert bool((o[1:n_text][same] > o[:n_text - 1][same]).all())
    # the kernel's algorithm (fp32 sum per token, one rounding) passes
    i7 = int((ref["toks"] == 7).nonzero())
    rows7 = (src.reshape(-1) == 7).nonzero()[:, 0]
    f32 = torch.zeros(H)
    for r in rows7:
        f32 += d.reshape(-1, H)[r].float()
    check_bound("fp32 sum", (old[7].float() + f32.to(bf16).float()).to(bf16), ref["want"][i7], ref["tol"][i7])
    # one duplicate row lost
    lost = (old[7].float() + (f32 - d.reshape(-1, H)[rows7[-1]].float()).to(bf16).float()).to(bf16)
    fails(lambda: check_bound("lost row", lost, ref["want"][i7], ref["tol"][i7]))
    # bf16 atomics: every duplicate rounded into the bf16 gradient in turn
    seq = old[7].clone()
    for r in rows7[torch.randperm(rows7.numel(), generator=g)]:
        seq = seq + d.reshape(-1, H)[r]
    fails(lambda: check_bound("bf16 sequential", seq, ref["want"][i7], ref["tol"][i7]))


def test_accumulate_tol_is_one_rounding_plus_the_sum():
    S = torch.tensor([1.0, 1000.0, -3.0], dtype=torch.float64)
    t = accumulate_tol(torch.zeros(3, dtype=torch.float64), S, torch.zeros(3, dtype=torch.float64))
    assert bool((t < 2.05 * BF16_U * S.abs() + 1e-20).all()) and bool((t >= 2 * BF16_U * S.abs()).all())


@pytest.mark.parametrize("max_norm,step,wd", [(1.0, 1, 0.01), (1e4, 3, 0.0), (0.0, 10000, 0.01)])
def test_adamw_reference_matches_oracle_and_catches_missing_bias_correction(max_norm, step, wd):
    n = 4000
    g = torch.Generator().manual_seed(step)
    p = torch.randn(n, generator=g)
    m, v = torch.randn(n, generator=g) * 0.01, torch.rand(n, generator=g) * 1e-4
    grad = (torch.randn(n, generator=g) * 3).to(bf16)
    gs = 0.125
    nsq = float((grad.double() ** 2).sum())
    ref = adamw_reference_fp64(p, m, v, grad, step, 1e-3, 0.9, 0.999, 1e-8, wd, nsq, max_norm, gs)
    geff = grad.float() * gs
    if max_norm > 0:
        total = R.clip_grad_norm([geff], max_norm)
        assert abs(total.item() - math.sqrt(nsq) * gs) <= 1e-6 * total.item()
    pr, mr, vr = p.clone(), m.clone(), v.clone()
    R.adamw_step([pr], [geff], [mr], [vr], step, 1e-3, wd=wd)
    # the fp32 oracle makes the same kind of roundings as the kernel: within the bound (2x: its own fp32 errors plus the kernel's), with
    # the hyperparameters as the Python floats it uses
    py = adamw_reference_fp64(p, m, v, grad, step, 1e-3, 0.9, 0.999, 1e-8, wd, nsq, max_norm, gs, fp32_hyper=False)
    check_bound("m", mr, py["m"], 2 * py["m_tol"])
    check_bound("v", vr, py["v"], 2 * py["v_tol"])
    check_bound("master", pr, py["master"], 2 * py["master_tol"])
    # and the kernel's fp32 hyperparameters move the result by far less than the update itself
    assert float((py["master"] - ref["master"]).abs().max()) <= 1e-4 * 1e-3
    if step < 100:
        nb = adamw_reference_fp64(p, m, v, grad, step, 1e-3, 0.9, 0.999, 1e-8, wd, nsq, max_norm, gs, bias_correction=False)
        fails(lambda: check_bound("master", nb["master"].float(), ref["master"], ref["master_tol"]))
