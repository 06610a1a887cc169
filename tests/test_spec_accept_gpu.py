"""lmod_spec_accept (csrc/spec.cu): greedy acceptance equals torch.argmax including planted ties; sampling matches the float64
restatement (tests/spec_oracle.py) given the same uniforms, a different decision allowed only within fp32 rounding of its boundary; the
bonus token, rejection at row 0, -inf entries, a draft vocabulary smaller than the target's, and the rollback of both cache lengths."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from llavamod import kernels as K  # noqa: E402
from tests import spec_oracle as SO  # noqa: E402


def _lens(B, base=100):
    return torch.arange(B, dtype=torch.int32, device="cuda") + base


@pytest.mark.parametrize("V,k", [(1000, 4), (151936, 4), (777, 1), (4099, 7)])
def test_greedy_equals_argmax_with_ties(V, k):
    B = 2 * (k + 1)
    g = torch.Generator(device="cuda").manual_seed(V + k)
    logits = torch.randn(B, k + 1, V, device="cuda", generator=g) * 3
    for b in range(B):                                          # ties at the maximum in every other row: the first index wins
        for j in range(0, k + 1, 2):
            i1, i2 = sorted(torch.randint(0, V, (2,), generator=g, device="cuda").tolist())
            if i1 != i2:
                logits[b, j, i1] = logits[b, j, i2] = logits[b, j].max() + 1
    logits[0, 0, : V // 2] = float("-inf")
    a = logits.argmax(-1)
    d = torch.randint(0, V, (B, k), generator=g, device="cuda")
    want_n = [b % (k + 1) for b in range(B)]
    for b, n in enumerate(want_n):
        d[b, :n] = a[b, :n]
        if n < k:
            d[b, n] = (a[b, n] + 1) % V
    lt, ld = _lens(B), _lens(B, 50)
    lt0, ld0 = lt.clone(), ld.clone()
    n_acc, nxt = K.spec_accept(logits, d, len_target=lt, len_draft=ld)
    assert n_acc.tolist() == want_n
    assert nxt.tolist() == [int(a[b, n]) for b, n in enumerate(want_n)]
    drop = torch.tensor([k - n for n in want_n], dtype=torch.int32, device="cuda")
    assert torch.equal(lt, lt0 - drop) and torch.equal(ld, ld0 - drop)
    for b in range(B):
        assert SO.accept(logits[b].cpu(), d[b].cpu()) == (want_n[b], int(a[b, want_n[b]]))


def _check_sampling(P, Q, d, u):
    B, k = d.shape
    lt = _lens(B)
    n_acc, nxt = K.spec_accept(P, d, Q, u, len_target=lt)
    n_acc, nxt = n_acc.tolist(), nxt.tolist()
    exact = 0
    for b in range(B):
        err = SO.explain_sample(P[b].cpu(), d[b].cpu(), Q[b].cpu(), u[b].cpu().double(), n_acc[b], nxt[b])
        assert err is None, (b, err)
        exact += SO.accept(P[b].cpu(), d[b].cpu(), Q[b].cpu(), u[b].cpu().double()) == (n_acc[b], nxt[b])
    assert exact >= B - 1
    assert lt.tolist() == [100 + b - (k - n_acc[b]) for b in range(B)]
    return n_acc, nxt


@pytest.mark.parametrize("V_t,V_d,k", [(1000, 1000, 4), (152064, 151936, 4), (5000, 4097, 2), (300, 300, 7)])
def test_sampling_matches_fp64_restatement(V_t, V_d, k):
    B = 16
    g = torch.Generator(device="cuda").manual_seed(V_t + V_d + k)
    P = torch.randn(B, k + 1, V_t, device="cuda", generator=g) * 2
    Q = P[:, :k, :V_d] + 0.7 * torch.randn(B, k, V_d, device="cuda", generator=g)          # a draft near the target
    P[:, :, 7::5] = float("-inf")                                                           # filtered entries
    Q[:, :, 11::7] = float("-inf")
    d = torch.multinomial(Q.reshape(B * k, V_d).softmax(-1), 1, generator=g).view(B, k)
    u = torch.rand(B, k + 1, device="cuda", generator=g)
    n_acc, _ = _check_sampling(P, Q, d, u)
    assert 0 < sum(n_acc) < B * k
    # q == p: every draft is kept, the bonus token comes from row k
    Q2 = P[:, :k].clone()
    d2 = torch.multinomial(Q2[..., :min(V_t, V_d)].reshape(B * k, -1).softmax(-1), 1, generator=g).view(B, k)
    n2, _ = _check_sampling(P, Q2, d2, u)
    assert n2 == [k] * B
    # rejection at row 0: the target gives the first draft probability 0
    P3 = P.clone()
    P3[torch.arange(B), 0, d[:, 0]] = float("-inf")
    n3, nx3 = _check_sampling(P3, Q, d, u)
    assert n3 == [0] * B
    assert all(int(x) != int(d[b, 0]) for b, x in enumerate(nx3))


def test_sampling_is_deterministic_and_stays_in_the_vocabulary():
    B, k, V = 8, 3, 2000
    g = torch.Generator(device="cuda").manual_seed(1)
    P = torch.randn(B, k + 1, V, device="cuda", generator=g)
    P[..., 100:] = float("-inf")                                # a narrowed vocabulary
    Q = P[:, :k].clone()
    Q += torch.randn_like(Q)
    d = torch.multinomial(Q.reshape(B * k, V).softmax(-1), 1, generator=g).view(B, k)
    u = torch.rand(B, k + 1, device="cuda", generator=g)
    a = K.spec_accept(P, d, Q, u)
    b = K.spec_accept(P, d, Q, u)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert int(a[1].max()) < 100
