"""The exact designs of test_decode_exact_gpu.py and test_spec_accept_exact_gpu.py checked on the CPU: their expected values equal the float64
references (decode_reference_fp64 after bf16 rounding, spec_oracle.accept), and every planted kernel defect changes at least one
expected byte or token of the designed sweep, so the GPU tests would see it."""
import numpy as np
import pytest
import torch

from tests import decode_exact as D
from tests import spec_exact as E
from tests import spec_oracle as SO

SMS = 132                        # an H100 SXM; the GPU tests take the SM count from the device


def _design(hd, nh, nkv, max_len, T=1, tier=1, mult=1, seed=0):
    sk = D.decode_splits(max_len, nkv, SMS)[1] * D.BK
    ring = D.NST[D.head_dim_padded(hd)] * D.BK
    lens = [n for n in D.edge_lengths(max_len, sk, ring) if n >= T]
    return D.Design(len(lens), T, nh, nkv, hd, lens, max_len, sk, seed=seed, tier=tier, mult=mult)


@pytest.mark.parametrize("hd,nh,nkv,max_len,tier,mult", [(64, 4, 2, 1024, 1, 1), (128, 6, 2, 1024, 1, 1), (80, 7, 1, 512, 1, 1),
                                                         (64, 8, 2, 2048, 1, 2), (128, 4, 2, 1024, 2, 1), (64, 16, 2, 1024, 2, 2)])
def test_exact_expectation_equals_fp64_reference(hd, nh, nkv, max_len, tier, mult):
    d = _design(hd, nh, nkv, max_len, tier=tier, mult=mult, seed=hd + nh)
    out, lse, lse_tol = d.expected()
    ref, ref_lse, tol, _ = D.decode_reference_fp64(d.q, d.k, d.v, d.lens, nh, nkv, hd, d.scale)
    ref = ref.view(d.B, -1)
    # where the exact sum is 0 the reference leaves rounding noise (1e-16), and at tier 2 the 3e-9 relative gap between scale and fp32 ln 2
    # in its exponents (1e-9); every nonzero exact output is at least 2^-3 / (8 len) > 1e-5
    ref = torch.where(ref.abs() < 1e-6, torch.zeros_like(ref), ref)
    assert torch.equal(ref.float().to(torch.bfloat16).view(torch.int16), out.view(torch.int16))
    assert bool(((out.double() - ref).abs() <= tol.view(d.B, -1)).all())
    # the reference takes softmax over scale * s in natural units; the kernel's exponent is exactly mult * s, scaled by fp32 ln 2
    assert bool(((lse - ref_lse).abs() <= lse_tol + 1e-5 * ref_lse.abs()).all())
    assert bool((lse_tol <= 8 * 2.0 ** -24 * (1 + lse.abs()) + 2.0 ** -20).all())              # a few ulp


def test_chunk_expectation_is_the_single_query_one_at_each_row_limit():
    T = 5
    d = _design(128, 6, 2, 1024, T=T, seed=3)
    out, lse, _ = d.expected()
    for t in range(T):
        one = D.Design.__new__(D.Design)
        one.__dict__.update(d.__dict__)
        one.T, one.q, one.col = 1, d.q.view(d.B, T, -1)[:, t], d.col.view(d.B, T, -1)[:, t]
        one.lims = [n - T + t + 1 for n in d.lens]
        o1, l1, _ = one.expected()
        assert torch.equal(out.view(d.B, T, -1)[:, t], o1) and torch.equal(lse.view(d.B, T, -1)[:, t], l1)


def _changed(d, defect, want):
    out, lse, _ = d.expected(defect)
    return not torch.equal(out.view(torch.int16), want[0].view(torch.int16)) or not torch.equal(lse, want[1])


@pytest.mark.parametrize("hd", [64, 128])
def test_planted_decode_defects_change_the_expectation(hd):
    """One key dropped at each edge class, a neighbour's score or V row, the wrong KV head, a lost split: each changes at least one
    expected output of the sweep."""
    d = _design(hd, 4, 2, 1024, seed=11)
    want = d.expected()
    sk, ring = d.sk, D.NST[d.hp] * D.BK
    classes = {"first key": 0, "block last": D.BK - 1, "block first": D.BK, "ring last": ring - 1, "ring first": ring,
               "split last": sk - 1, "split first": sk, "second ring pass of split 1": sk + ring, "second split last": 2 * sk - 1}
    for name, p in classes.items():
        assert _changed(d, ("drop", p), want), name
    for p in (0, D.BK - 1, ring - 1, sk - 1):
        assert _changed(d, ("score", p), want), ("score", p)
        assert _changed(d, ("vrow", p), want), ("vrow", p)
    assert _changed(d, ("kvhead",), want)
    for i in range(3):
        assert _changed(d, ("split", i), want), ("split", i)
    for n in d.lens:                                                # the last key of each length
        assert _changed(d, ("drop", n - 1), want), ("drop last", n)


def test_spec_expectation_equals_fp64_restatement():
    for V in (1, 4, 4095, 4096, 4097, 152064):
        m = 0 if V == 1 else (2 if V < 16 else 4)
        P, Q, d, u = E.bonus_sweep(V, m, seed=V)
        for b in range(len(u)):
            assert E.expected(P[b], Q[b], d[b], u[b]) == SO.accept(P[b], d[b], Q[b], u[b].double()), (V, b)
            S = (P[b, 1] == 0).nonzero()[:, 0].tolist()
            assert E.expected(P[b], Q[b], d[b], u[b])[1] == S[int(np.floor(float(u[b, 1]) * (1 << m)))]
    for bd in (False, True):
        for V_t, V_d, k in ((5000, 4097, 7), (8200, 8193, 64)):
            P, Q, d, u = E.residual_design(V_t, V_d, k, 16, seed=V_t + k + bd, boundary=bd)
            for b in range(16):
                assert E.expected(P[b], Q[b], d[b], u[b]) == SO.accept(P[b], d[b], Q[b], u[b].double()), (bd, V_t, k, b)


def test_planted_spec_defects_change_a_token():
    seqs = []
    for V in (4095, 4096, 4097, 152064):
        P, Q, d, u = E.bonus_sweep(V, 4, seed=V)
        seqs += [(P[b], Q[b], d[b], u[b]) for b in range(len(u))]
    P, Q, d, u = E.residual_design(5000, 4097, 7, 64, seed=5000 + 7 + 1, boundary=True)
    seqs += [(P[b], Q[b], d[b], u[b]) for b in range(64)]
    want = [E.expected(*s) for s in seqs]
    for defect in ("ge", "lt", "late"):
        assert any(E.expected(*s, defect=defect) != w for s, w in zip(seqs, want)), defect
