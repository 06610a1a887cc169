"""lmod_spec_accept (csrc/spec.cu) on designs that make it exact (tests/spec_exact.py): logits 0 on 2^m ids and -inf elsewhere, so every
probability and every running sum is exact in fp32 and the accepted count and the token are functions of u alone.  The inverse CDF is
checked at u = j / 2^m and its fp32 neighbours (the strict > picks element j at u = j / 2^m) with the set on the thread-item, tile and
vocabulary edges; the acceptance test at u = p(x) / q(x) and the next fp32 above; the residual draw with a draft vocabulary smaller than
the target's; k = 1, 7 and 64 (the largest the kernel takes) and thousands of sequences in one launch.  Both cache lengths must be rolled
back by exactly k - n_acc."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from llavamod import kernels as K  # noqa: E402
from tests import spec_exact as E  # noqa: E402
from tests.helpers import poisoned_uninitialised_memory  # noqa: E402


def _run_and_check(name, P, Q, d, u):
    B, k = d.shape
    want = [E.expected(P[b], Q[b], d[b], u[b]) for b in range(B)]
    lt = torch.arange(B, dtype=torch.int32, device="cuda") + 1000
    ld = torch.arange(B, dtype=torch.int32, device="cuda") + 500
    with poisoned_uninitialised_memory():
        n_acc, nxt = K.spec_accept(P.cuda(), d.cuda(), Q.cuda(), u.cuda(), len_target=lt, len_draft=ld)
    got = list(zip(n_acc.tolist(), nxt.tolist()))
    bad = [(b, got[b], want[b], float(u[b, -1])) for b in range(B) if got[b] != want[b]]
    assert not bad, "%s: %d / %d sequences differ; first (b, got, want, u_k) = %s" % (name, len(bad), B, bad[:3])
    drop = torch.tensor([k - n for n, _ in want], dtype=torch.int32)
    assert torch.equal(lt.cpu(), torch.arange(B, dtype=torch.int32) + 1000 - drop), name
    assert torch.equal(ld.cpu(), torch.arange(B, dtype=torch.int32) + 500 - drop), name
    return want


@pytest.mark.parametrize("V", [1, 4, 4095, 4096, 4097, 151936, 152064])
def test_inverse_cdf_at_every_boundary(V):
    m = 0 if V == 1 else (2 if V < 16 else 4)
    P, Q, d, u = E.bonus_sweep(V, m, seed=V)
    want = _run_and_check("bonus V%d" % V, P, Q, d, u)
    assert all(n == 1 for n, _ in want)


@pytest.mark.parametrize("V_t,V_d,k,B", [(5000, 4097, 7, 64), (152064, 151936, 1, 16), (8200, 8193, 64, 8), (4097, 4096, 1, 4096)])
def test_residual_and_acceptance_boundary(V_t, V_d, k, B):
    P, Q, d, u = E.residual_design(V_t, V_d, k, B, seed=V_t + k)
    want = _run_and_check("residual %d/%d k%d" % (V_t, V_d, k), P, Q, d, u)
    assert {n for n, _ in want} == set(range(min(k, B - 1) + 1))
    P, Q, d, u = E.residual_design(V_t, V_d, k, B, seed=V_t + k + 1, boundary=True)
    want = _run_and_check("boundary %d/%d k%d" % (V_t, V_d, k), P, Q, d, u)
    for b, (n, _) in enumerate(want):               # u = p/q accepts the boundary draft, the next fp32 above rejects it
        if b % (k + 1) < k:
            assert (n > b % (k + 1)) == ((b // (k + 1)) % 2 == 0), (b, n)
