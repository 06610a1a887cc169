"""Designs that make lmod_spec_accept (csrc/spec.cu) exact, and their expected results.  Pure torch / numpy: the CPU tests check them.

Every row's logits are 0 on a set of 2^m ids and -inf elsewhere.  The kernel's softmax is then exactly 2^-m on the set (ex2(0) = 1, a sum
of 2^m ones, an IEEE divide), the residual max(0, p - q) of two such rows is a difference of powers of two, and every running sum of the
inverse CDF is exact in fp32.  So the drawn token is a function of u alone:
  * q = p (every draft kept, the bonus row sampled): the token is element floor(u 2^m) of the set -- the running sum passes u at element j
    exactly when u < (j + 1) 2^-m, and u = j 2^-m picks element j because the comparison is strict;
  * residual: the first id whose exact running sum exceeds fp32(u * total), the product the kernel forms;
  * acceptance: u q(x) <= p(x) with both sides exact, so u = p(x) / q(x) accepts and the next fp32 above rejects.
`expected` restates the kernel's decisions on these designs; its `defect` argument plants a kernel defect, for the CPU check that the
designs see it: "ge" (>= for > in the inverse CDF), "lt" (< for <= in the acceptance test), "late" (a crossing at the last of a thread's
four ids reported one id late)."""
import numpy as np
import torch

ITEMS = 4                        # SA_ITEMS: consecutive ids per thread
TILE = 1024 * ITEMS              # SA_TILE


def edge_set(V, m, rng):
    """2^m ids in [0, V) with the thread-item edges 3 | 4, the tile edges 4095 | 4096 and 8191 | 8192 and V - 1 among them."""
    n = 1 << m
    assert n <= V
    want = [i for i in (3, 4, 4095, 4096, 8191, 8192, V - 1, 0) if i < V]
    s = list(dict.fromkeys(want))[:n]
    rest = np.setdiff1d(np.arange(V), s)
    s += rng.choice(rest, n - len(s), replace=False).tolist()
    return sorted(int(i) for i in s)


def u_sweep(m):
    """u = j / 2^m, its fp32 neighbours, 0 and the largest fp32 below 1."""
    us = {np.float32(0.0), np.nextafter(np.float32(1.0), np.float32(0.0))}
    for j in range(1 << m):
        x = np.float32(j / (1 << m))
        us |= {x, np.nextafter(x, np.float32(1.0))}
        if j:
            us.add(np.nextafter(x, np.float32(0.0)))
    return sorted(us)


def row(V, ids):
    x = torch.full((V,), float("-inf"))
    x[list(ids)] = 0.0
    return x


def _probs(x):
    """The kernel's fp32 softmax of a design row: 2^-m on the set."""
    fin = np.isfinite(x)
    p = np.zeros(len(x), dtype=np.float32)
    p[fin] = np.float32(1.0) / np.float32(fin.sum())
    return p


def inverse_cdf(w, u, defect=None):
    """sample_inverse_cdf of csrc/spec.cu on exact fp32 weights w: the first id whose running sum exceeds fp32(u * total)."""
    c = np.cumsum(w.astype(np.float64))
    total = np.float32(c[-1])
    assert float(total) == c[-1]
    target = float(np.float32(np.float32(u) * total))
    hit = (c >= target) if defect == "ge" else (c > target)
    hit &= w > 0
    idx = np.nonzero(hit)[0]
    i = int(idx[0]) if len(idx) else int(np.nonzero(w > 0)[0][-1])
    if defect == "late" and i % ITEMS == ITEMS - 1:
        i += 1
    return i


def expected(P, Q, d, u, defect=None):
    """One sequence of a design: P [k + 1, V_t], Q [k, V_d] logits, d [k] drafts, u [k + 1] fp32.  -> (n_acc, next)."""
    P, Q, d, u = P.numpy(), Q.numpy(), d.tolist(), np.asarray(u, dtype=np.float32)
    k, V_t = len(d), P.shape[1]
    V_d = Q.shape[1]
    for j in range(k):
        p = _probs(P[j])
        q = np.zeros(V_t, dtype=np.float32)
        q[:min(V_t, V_d)] = _probs(Q[j])[:V_t]
        x = d[j]
        pd = p[x] if x < V_t else np.float32(0)
        qd = q[x] if x < V_d else np.float32(0)
        lhs = np.float32(u[j] * qd)
        if (lhs < pd) if defect == "lt" else (lhs <= pd):
            continue
        w = np.maximum(np.float32(0), p - q)
        if not (w > 0).any():
            w = p
        return j, inverse_cdf(w, u[k], defect)
    return k, inverse_cdf(_probs(P[k]), u[k], defect)


def bonus_sweep(V, m, seed):
    """q = p: every draft kept, the bonus row sampled at every u of u_sweep(m).  -> (P [B, 2, V], Q [B, 1, V], d [B, 1], u [B, 2])."""
    rng = np.random.default_rng(seed)
    us = u_sweep(m)
    B = len(us)
    S = edge_set(V, m, rng)
    S0 = edge_set(V, min(m, 1), rng)
    P = torch.stack([torch.stack([row(V, S0), row(V, S)]) for _ in range(B)])
    Q = P[:, :1].clone()
    d = torch.tensor([[S0[b % len(S0)]] for b in range(B)], dtype=torch.int64)
    u = torch.tensor([[0.5, float(x)] for x in us], dtype=torch.float32)
    return P, Q, d, u


def residual_design(V_t, V_d, k, B, seed, boundary=False):
    """k rows per sequence; sequence b keeps its first n_b = b % (k + 1) drafts (q = p there) and rejects draft n_b (when n_b < k).
    Rejection row: p uniform on S (2^a ids), q uniform on S' (2^(a+1) ids, inside [0, V_d)), S and S' partly overlapping, with S' holding
    ids the target set does not.  boundary: q on S' of 2^(a-1) ids inside S and the draft in both, so p(x) / q(x) = 1/2; u = 1/2 must accept
    and the next fp32 above it must reject (sequences b with b // (k + 1) odd take the latter).  u of the bonus / residual draw: 12-bit dyadics, so
    fp32(u * total) is exact."""
    rng = np.random.default_rng(seed)
    a = 3
    P = torch.full((B, k + 1, V_t), float("-inf"))
    Q = torch.full((B, k, V_d), float("-inf"))
    d = torch.zeros(B, k, dtype=torch.int64)
    u = torch.zeros(B, k + 1, dtype=torch.float32)
    for b in range(B):
        n = b % (k + 1)
        for j in range(k + 1):
            S = edge_set(V_d if j < n else V_t, a, rng)
            P[b, j] = row(V_t, S)
            if j < k:
                if j < n:
                    Q[b, j] = row(V_d, S)
                    d[b, j] = S[rng.integers(len(S))]
                    u[b, j] = float(np.float32(rng.integers(0, 1 << 12) / (1 << 12)))
                elif j == n:
                    if boundary:
                        Sq = sorted(rng.choice([s for s in S if s < V_d], 1 << (a - 1), replace=False).tolist())
                        Q[b, j] = row(V_d, Sq)
                        d[b, j] = Sq[rng.integers(len(Sq))]
                        u[b, j] = 0.5 if (b // (k + 1)) % 2 == 0 else float(np.nextafter(np.float32(0.5), np.float32(1.0)))
                    else:
                        inS = [s for s in S if s < V_d]
                        keep = rng.choice(inS, max(1, len(inS) // 2), replace=False).tolist()
                        outS = np.setdiff1d(np.arange(V_d), S)
                        Sq = sorted(keep + rng.choice(outS, (1 << (a + 1)) - len(keep), replace=False).tolist())
                        Q[b, j] = row(V_d, Sq)
                        d[b, j] = [s for s in Sq if s not in S][rng.integers((1 << (a + 1)) - len(keep))]
                        u[b, j] = float(np.float32((rng.integers(1, 1 << 12)) / (1 << 12)))
                else:
                    Sq = edge_set(V_d, a, rng)
                    Q[b, j] = row(V_d, Sq)
                    d[b, j] = Sq[0]
                    u[b, j] = 0.25
        u[b, k] = float(np.float32(rng.integers(0, 1 << 12) / (1 << 12)))
    return P, Q, d, u
