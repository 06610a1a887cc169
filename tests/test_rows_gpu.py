"""Active-row compaction of the loss head (csrc/rows.cu, lmod_gemm_bf16_dyn, lmod_kl_fwd_bwd_rows): integer index work bit-exact
against numpy/torch, the compact KL kernel bit-identical to the dense one on the rows that matter, dynamic-extent GEMMs equal to the
static GEMM on the effective sub-problem, and the whole compact head equal to the dense head."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _labels(B, T, V, frac, seed, tail_pad=0):
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (B, T), generator=g)
    lab[:, : int(frac * T)] = -100
    if tail_pad:
        lab[:, T - tail_pad:] = -100
    return lab


def _active_ref(lab):
    B, T = lab.shape
    m_kd = lab != -100
    m_ce = torch.cat([lab[:, 1:] != -100, torch.zeros(B, 1, dtype=torch.bool)], 1)
    return (m_kd | m_ce).reshape(-1)


@pytest.mark.parametrize("B,T,frac,pad", [(1, 2048, 0.57, 0), (3, 333, 0.4, 7), (2, 64, 1.0, 0), (1, 5000, 0.0, 0), (4, 17, 0.5, 3)])
def test_active_rows_gather_scatter_bit_exact(B, T, frac, pad):
    from llavamod import kernels as K
    lab = _labels(B, T, 1000, frac, seed=B * T, tail_pad=pad)
    act = _active_ref(lab)
    perm, count = K.active_rows(lab.reshape(-1).cuda(), T)
    n = int(act.sum())
    assert int(count) == n
    idx = torch.nonzero(act).reshape(-1).to(torch.int32)
    assert torch.equal(perm[:n].cpu(), idx) and bool((perm[n:] == -1).all())
    # distill_all: every row is active
    perm_all, count_all = K.active_rows(lab.reshape(-1).cuda(), T, True)
    assert int(count_all) == B * T and torch.equal(perm_all.cpu(), torch.arange(B * T, dtype=torch.int32))
    x = torch.randn(B * T, 64, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).cuda()
    xc = K.gather_rows(x, perm, count)
    assert xc.shape[0] % K.ROW_PAD == 0 and xc.shape[0] >= B * T
    assert torch.equal(xc[:n].cpu(), x.cpu()[idx.long()])
    padded = (n + K.ROW_PAD - 1) // K.ROW_PAD * K.ROW_PAD
    assert bool((xc[n:padded] == 0).all())
    back = K.scatter_rows(xc, perm, count, B * T)
    ref = torch.zeros_like(x)
    ref[idx.long().cuda()] = x[idx.long().cuda()]
    assert torch.equal(back, ref)
    # identity gather = dynamic-count row copy (pipeline hand-over)
    out = torch.full_like(xc, 7.0)
    K.gather_rows(xc, None, count, out=out)
    assert torch.equal(out[:padded], xc[:padded]) and bool((out[padded:] == 7.0).all())


@pytest.mark.parametrize("N,V,frac,w_ce", [(96, 4136, 0.5, 1.0), (64, 151936, 0.6, 1.0), (40, 1024, 0.3, 0.0),
                                          (600, 151936, 0.3, 1.0)])   # several rows per cluster: compact and dense clusters see other rows
def test_compact_kl_equals_dense_kl(N, V, frac, w_ce):
    """Same kernel, same per-row arithmetic: the compact call must reproduce the dense call's loss numbers exactly and its gradient rows
    bit for bit."""
    from llavamod import kernels as K
    g = torch.Generator().manual_seed(N + V)
    s = (torch.randn(N, V, generator=g) * 2).to(torch.bfloat16).cuda()
    t = (torch.randn(N, V, generator=g) * 2).to(torch.bfloat16).cuda()
    lab = _labels(1, N, V, frac, seed=3, tail_pad=5).reshape(-1).cuda()
    d_dense = torch.empty_like(s)
    out_dense, _ = K.kl_fused(s, t, lab, N, V, 1.0, w_ce, False, dlogits=d_dense)
    perm, count = K.active_rows(lab, N)
    n = int(count)
    sc, tc = K.gather_rows(s, perm, count), K.gather_rows(t, perm, count)
    d_c = torch.full_like(sc, float("nan"))
    out_c, _ = K.kl_fused(sc, tc, lab, N, V, 1.0, w_ce, False, dlogits=d_c, rows=(perm, count))
    assert torch.equal(out_c, out_dense)
    assert torch.equal(d_c[:n], d_dense[perm[:n].long()])
    inactive = torch.ones(N, dtype=torch.bool, device="cuda")
    inactive[perm[:n].long()] = False
    assert bool((d_dense[inactive] == 0).all())             # what the compact path never has to write


@pytest.mark.parametrize("count", [0, 1, 255, 256, 700, 2048])
def test_dynamic_extent_gemms_match_static_subproblem(count):
    """M from device memory (forward / dgrad) and K from device memory (wgrad), incl. the empty problem."""
    from llavamod import kernels as K
    g = torch.Generator().manual_seed(count)
    M, Kd, N = 2048, 256, 2048 + 512
    a = torch.randn(M, Kd, generator=g).to(torch.bfloat16).cuda()
    a[count:] = 0                                                           # what gather_rows guarantees up to the tile boundary
    w = torch.randn(N, Kd, generator=g).to(torch.bfloat16).cuda()
    cnt = torch.tensor([count], dtype=torch.int32, device="cuda")
    full = K.gemm(a, w)
    out = torch.full((M, N), 3.0, dtype=torch.bfloat16, device="cuda")
    K.gemm(a, w, out=out, m_dev=cnt)
    assert torch.equal(out[:count], full[:count])
    tile_end = (count + 255) // 256 * 256
    assert bool((out[tile_end:] == 3.0).all())                              # tiles past the extent are not touched
    # dgrad form (B MN-major); N = 2560 stays below mm_nn's split-K threshold (N >= 16384), which test_loss_head_gpu.py covers
    dx = K.mm_nn(full, w, m_dev=cnt)
    ref = K.mm_nn(full, w)
    assert torch.allclose(dx[:count].float(), ref[:count].float(), rtol=2e-2, atol=2e-2 * ref.float().abs().max().item())
    # wgrad form: reduction over the first `count` rows only
    gacc = torch.zeros(N, Kd, dtype=torch.bfloat16, device="cuda")
    K.mm_tn_acc(full, a, gacc, k_dev=cnt)
    gref = torch.zeros(N, Kd, dtype=torch.bfloat16, device="cuda")
    if count:
        K.mm_tn_acc(full[:tile_end if tile_end <= M else M], a[:tile_end if tile_end <= M else M], gref)
    err = (gacc.float() - gref.float()).abs().max().item()
    assert err <= 2e-2 * max(1.0, gref.float().abs().max().item()), err


def test_compact_head_equals_dense_head():
    """DistillHeadFn with and without row compaction: same losses, same d hidden, same lm_head gradient."""
    from llavamod import kernels as K
    g = torch.Generator().manual_seed(5)
    B, T, H, V = 2, 96, 128, 4096
    hid = torch.randn(B, T, H, generator=g).to(torch.bfloat16).cuda()
    w = (torch.randn(V, H, generator=g) * 0.05).to(torch.bfloat16).cuda()
    th = torch.randn(B * T, H, generator=g).to(torch.bfloat16).cuda()
    wt = (torch.randn(V, H, generator=g) * 0.05).to(torch.bfloat16).cuda()
    lab = _labels(B, T, V, 0.55, seed=9, tail_pad=4).cuda()
    res = []
    for compact in (False, True):
        h = hid.clone().requires_grad_(True)
        hg = torch.zeros(V, H, dtype=torch.bfloat16, device="cuda")
        rows = K.active_rows(lab.reshape(-1), T) if compact else None
        t_logits = K.gemm(K.gather_rows(th, *rows) if compact else th, wt, m_dev=rows[1] if compact else None)
        total, align, ce = K.distill_head(h, w, t_logits, lab, V, 1.0, 1.0, False, hg, rows=rows)
        (total * 0.5).backward()
        res.append((float(total), float(align), float(ce), h.grad.clone(), hg))
    a, b = res
    assert a[:3] == b[:3]
    assert torch.allclose(a[3].float(), b[3].float(), rtol=2e-2, atol=1e-5)
    assert torch.allclose(a[4].float(), b[4].float(), rtol=2e-2, atol=2e-2 * a[4].float().abs().max().item())
    act = _active_ref(lab.cpu()).reshape(B, T)
    assert bool((b[3][~act.cuda()] == 0).all())
