"""tests/helpers.distill_head_reference_fp64, the float64 stages of kernels.DistillHeadFn, against autograd of the oracle's own formulas
(R.get_logp, R.get_p, R.compute_align_loss and R.shifted_ce over h W^T, scaled by an upstream g != 1), in the compact and the dense row
layout and with a student vocabulary wider than the KD slice.  No GPU."""
import math

import pytest
import torch

from oracle import restated as R
from tests.helpers import IGNORE_INDEX, distill_head_reference_fp64, kl_row_masks

F64 = torch.float64


@pytest.mark.parametrize("g", [1.0 / 3.0, -0.37])
@pytest.mark.parametrize("Vs,vocab,w_ce", [(96, 96, 1.3), (104, 96, 0.0)], ids=["ce", "slice"])
@pytest.mark.parametrize("distill_all", [False, True])
@pytest.mark.parametrize("compact", [False, True], ids=["dense", "compact"])
def test_reference_matches_oracle_autograd(compact, distill_all, Vs, vocab, w_ce, g):
    B, T, H, w_kd = 2, 12, 16, 0.7
    N = B * T
    gen = torch.Generator().manual_seed(Vs + 2 * distill_all + compact)
    h = torch.randn(N, H, generator=gen, dtype=F64)
    W = torch.randn(Vs, H, generator=gen, dtype=F64) * (3 / math.sqrt(H))
    t = torch.randn(N, vocab, generator=gen, dtype=F64) * 3 + 0.5 * (h @ W[:vocab].t())
    labels = torch.randint(0, vocab, (B, T), generator=gen)
    labels[0, :3] = labels[0, 7:9] = labels[1, 5] = labels[1, T - 1] = IGNORE_INDEX
    labels[1, :4] = IGNORE_INDEX                                       # rows 12, 13 inactive, 14 CE-only, 4 KD-only
    flat = labels.reshape(-1)
    old = torch.randn(Vs, H, generator=gen, dtype=F64) * 0.01
    m_kd, m_ce, _ = kl_row_masks(flat, T, distill_all)
    act = torch.nonzero(m_kd | m_ce)[:, 0]
    assert distill_all or act.numel() < N
    rows, t_in = None, t
    if compact:                                                        # the layout kernels.active_rows and the trainer's teacher give
        n = act.numel()
        perm = torch.full((N,), -1, dtype=torch.int32)
        perm[:n] = act.to(torch.int32)
        rows = (perm, torch.tensor([n], dtype=torch.int32))
        t_in = torch.full((n + 5, vocab + 8), float("nan"), dtype=F64)
        t_in[:n, :vocab] = t[act]
    ref = distill_head_reference_fp64(h, W, t_in, flat, T, vocab, w_kd, w_ce, distill_all, g, rows=rows, old=old)

    hh, WW = h.clone().requires_grad_(True), W.clone().requires_grad_(True)
    s = (hh @ WW.t()).view(B, T, Vs)
    align = R.compute_align_loss(R.get_logp(s, vocab), R.get_p(t.view(B, T, vocab), vocab), labels, distill_all)
    total = w_kd * align
    if w_ce != 0.0:
        ce = R.shifted_ce(s, labels, vocab)
        total = total + w_ce * ce
        assert abs(ref["ce"] - ce.item()) <= 1e-5 * abs(ce.item())
    (g * total).backward()

    assert torch.equal(ref["act"], act)
    torch.testing.assert_close(ref["logits"], (h @ W.t())[act], rtol=1e-12, atol=0)
    assert abs(ref["align"] - align.item()) <= 1e-5 * abs(align.item())
    assert abs(ref["total"] - total.item()) <= 1e-5 * abs(total.item())
    # R.get_logp / get_p work in fp32: the oracle's gradients carry fp32 roundings of q and p
    for name, got, want in (("dh", ref["dh"], hh.grad), ("dW", ref["dW"] - old, WW.grad)):
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6 * float(want.abs().max()), msg=name)
    assert torch.equal(ref["dh"][~(m_kd | m_ce)], torch.zeros(N - act.numel(), H, dtype=F64))
    assert torch.equal(ref["dW"][vocab:], old[vocab:]) and bool((ref["dW_tol"][vocab:] == 0).all())
    for key in ("logits_tol", "dh_tol", "dW_tol"):
        assert bool((ref[key] >= 0).all() and torch.isfinite(ref[key]).all()), key
    assert bool((ref["dW_tol"][:vocab] > 0).all())
