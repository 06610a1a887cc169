"""The float64 restatement of assisted decoding's acceptance step (tests/spec_oracle.py) yields exactly the target distribution p.

Checked by enumeration, not by sampling: the restatement's output is a step function of the uniforms, so its distribution is the sum, over
the draft token d ~ q and over the intervals between the breakpoints of u_0 (the acceptance test) and u_1 (the inverse CDF), of the interval
lengths.  It must equal P(out = x) = q(x) min(1, p(x)/q(x)) + (1 - sum_y min(p(y), q(y))) r(x) = p(x), r = normalize(max(0, p - q))."""
import math

import pytest
import torch

from tests import spec_oracle as SO


def _logits(p):
    return torch.tensor([math.log(v) if v > 0 else -math.inf for v in p.tolist()], dtype=torch.float64)


def _intervals(points):
    pts = sorted({0.0, 1.0} | {float(x) for x in points if 0.0 < float(x) < 1.0})
    return [((a + b) / 2, b - a) for a, b in zip(pts[:-1], pts[1:])]


def _distribution(p, q):
    """P(first token of a round = x) with k = 1, by enumeration over d and the breakpoints of u_0 and u_1."""
    V_t = p.numel()
    pl, ql = _logits(p), _logits(q)
    P = torch.cat([pl[None], pl[None]])                      # rows 0 (scores d) and 1 (bonus); both the same target position here
    out = torch.zeros(V_t, dtype=torch.float64)
    qp = SO.softmax64(ql, V_t)
    for d in range(q.numel()):
        qd = float(SO.softmax64(ql)[d])
        if qd == 0:
            continue
        pd = float(SO.softmax64(pl)[d]) if d < V_t else 0.0
        u0s = _intervals([pd / qd])
        pp = SO.softmax64(pl)
        r = (pp - qp).clamp(min=0)
        cuts = list((torch.cumsum(r, 0) / r.sum()).tolist()) if r.sum() > 0 else []
        cuts += list(torch.cumsum(pp, 0).tolist())
        for u0, l0 in u0s:
            for u1, l1 in _intervals(cuts):
                n, x = SO.accept(P, torch.tensor([d]), ql[None], torch.tensor([u0, u1], dtype=torch.float64))
                out[d if n == 1 else x] += qd * l0 * l1          # the round's first token: the kept draft, or the resample
    return out


CASES = [
    ([0.5, 0.3, 0.2, 0.0], [0.1, 0.1, 0.8, 0.0]),
    ([0.25, 0.25, 0.25, 0.25], [0.7, 0.1, 0.1, 0.1]),
    ([0.0, 0.0, 1.0, 0.0], [0.3, 0.3, 0.2, 0.2]),
    ([0.4, 0.1, 0.3, 0.2], [0.4, 0.1, 0.3, 0.2]),           # q == p: every draft is kept
    ([0.1, 0.2, 0.3, 0.25, 0.15], [0.5, 0.3, 0.2]),        # V_d < V_t: the draft never proposes ids 3, 4
]


@pytest.mark.parametrize("p,q", CASES)
def test_restatement_yields_exactly_p(p, q):
    p = torch.tensor(p, dtype=torch.float64)
    q = torch.tensor(q, dtype=torch.float64)
    got = _distribution(p, q)
    assert torch.allclose(got, p, atol=1e-12, rtol=0), (got.tolist(), p.tolist())


def test_restatement_yields_exactly_p_random():
    g = torch.Generator().manual_seed(0)
    for _ in range(20):
        V = int(torch.randint(2, 7, (1,), generator=g))
        p = torch.rand(V, generator=g, dtype=torch.float64) * (torch.rand(V, generator=g) > 0.3)
        q = torch.rand(V, generator=g, dtype=torch.float64) * (torch.rand(V, generator=g) > 0.3)
        if p.sum() == 0 or q.sum() == 0:
            continue
        p, q = p / p.sum(), q / q.sum()
        assert torch.allclose(_distribution(p, q), p, atol=1e-12, rtol=0)


def test_greedy_restatement():
    P = torch.tensor([[0.0, 2.0, 2.0, 1.0], [5.0, 1.0, 5.0, 0.0], [0.0, 0.0, 0.0, 9.0]])
    assert SO.accept(P, torch.tensor([1, 0])) == (2, 3)        # ties take the first index, as torch.argmax
    assert SO.accept(P, torch.tensor([2, 0])) == (0, 1)
    assert SO.accept(P, torch.tensor([1, 2])) == (1, 0)
