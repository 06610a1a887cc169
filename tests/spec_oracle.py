"""The acceptance step of assisted decoding restated in float64 on the CPU (what lmod_spec_accept computes, csrc/spec.cu).

Greedy (HF _assisted_decoding): a_j = argmax of target row j, first index on ties; the drafts are kept while d_{j+1} == a_j; the next token
is a_{n_acc}.  Sampling (Leviathan et al., HF _speculative_sampling): with p_j = softmax(target row j) and q_j = softmax(draft row j)
(probability 0 at -inf and, for q, at ids >= V_d), d_{j+1} is kept while u_j * q_j(d_{j+1}) <= p_j(d_{j+1}); at the first rejection the next
token is drawn from normalize(max(0, p_j - q_j)), after k acceptances from p_k, both by inverse CDF with u_k: the first id whose running sum
exceeds u_k times the total."""
import torch


def softmax64(logits, V=None):
    """float64 softmax of one row of logits (-inf -> 0), zero-padded to V entries."""
    x = logits.double()
    p = torch.softmax(x, 0) if bool(torch.isfinite(x).any()) else torch.zeros_like(x)
    if V is not None and V > p.numel():
        p = torch.cat([p, p.new_zeros(V - p.numel())])
    return p[:V] if V is not None else p


def inverse_cdf(w, u):
    c = torch.cumsum(w, 0)
    hit = (c > u * c[-1]).nonzero()
    return int(hit[0]) if hit.numel() else int((w > 0).nonzero()[-1])


def accept(p_logits, d, q_logits=None, u=None):
    """One sequence.  p_logits [k+1, V_t]; d [k] draft ids; q_logits [k, V_d] and u [k+1] for sampling (None: greedy).
    -> (n_acc, next)."""
    k = len(d)
    V_t = p_logits.shape[1]
    if u is None:
        for j in range(k + 1):
            a = int(torch.argmax(p_logits[j]))
            if j < k and int(d[j]) == a:
                continue
            return j, a
    for j in range(k):
        p = softmax64(p_logits[j])
        q = softmax64(q_logits[j], V_t)
        x = int(d[j])
        pd = float(p[x]) if x < V_t else 0.0
        qd = float(q[x]) if x < q_logits.shape[1] else 0.0
        if float(u[j]) * qd <= pd:
            continue
        return j, inverse_cdf((p - q).clamp(min=0), float(u[k]))
    return k, inverse_cdf(softmax64(p_logits[k]), float(u[k]))


def explain_sample(p_logits, d, q_logits, u, n_got, next_got, tol=1e-4):
    """Check a kernel's sampling result (n_got, next_got) against the float64 restatement, allowing a different decision only where u
    lies within tol of the decision's boundary.  -> None, or a string saying what is wrong."""
    k = len(d)
    V_t = p_logits.shape[1]
    for j in range(k + 1):
        p = softmax64(p_logits[j])
        if j < k:
            q = softmax64(q_logits[j], V_t)
            x = int(d[j])
            pd = float(p[x]) if x < V_t else 0.0
            qd = float(q[x]) if x < q_logits.shape[1] else 0.0
            acc = float(u[j]) * qd <= pd
            near = abs(float(u[j]) * qd - pd) <= tol * max(pd, qd)
            if j < n_got:
                if not (acc or near):
                    return "row %d accepted, u*q = %g > p = %g" % (j, float(u[j]) * qd, pd)
                continue
            if acc and not near:
                return "row %d rejected, u*q = %g <= p = %g" % (j, float(u[j]) * qd, pd)
            w = (p - q).clamp(min=0)
            if not bool((w > 0).any()):
                w = p
        else:
            w = p
        if next_got < 0 or next_got >= V_t or not float(w[next_got]) > 0:
            return "row %d: token %d has weight 0" % (j, next_got)
        c = torch.cumsum(w, 0) / w.sum()
        lo = float(c[next_got - 1]) if next_got > 0 else 0.0
        hi = float(c[next_got])
        if not (lo - tol <= float(u[k]) <= hi + tol):
            return "row %d: token %d covers [%g, %g), u = %g" % (j, next_got, lo, hi, float(u[k]))
        return None
    return "unreachable"
