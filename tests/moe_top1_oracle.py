"""TEST INFRASTRUCTURE ONLY -- restatement of DeepSpeed 0.9.5's top1gating (random token selection, RTS) and the MoE layer built on it,
next to oracle/restated.py's top2gating (SURVEY.md Appendix A, "top-1").

top1gating(logits, cf, min_capacity, used_token=None, noisy_gate_policy=None, drop_tokens=True, use_rts=True), the defaults MoE passes:
  gates = softmax(logits); idx1 = argmax(gates) (the first maximal gate); C = ceil(S/E * cf) raised to min_capacity (no factor 2);
  exp_counts and l_aux = E * sum_e mean_s(gates) mean_s(mask1) before any drop; u = Uniform(0, 1) [S, E] on every call; per expert the
  routed tokens with the C largest u[s, idx1[s]] keep their seat (topk(mask1 * u, C, dim=0)); seats are cumsum(kept) - 1 in token order;
  the combine weight is the raw gate of a kept token (no renormalisation).  torch.topk leaves ties unspecified; the build's rule, restated
  here, keeps the lower token index among equal keys, and a routed token with u = 0.0 outranks every unrouted token (whose key is 0 in
  mask1 * u).  S < min_capacity (DeepSpeed's assert) and C > S (topk's k > S) raise ValueError.

The uniform is an explicit input so both sides route identically.  ``llava_forward`` runs oracle/restated.py's model forward with top-1 MoE
layers when ``cfg.top_k == 1``."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import restated as R


def top1_checks(S, E, cf, min_cap):
    if S < min_cap:
        raise ValueError("top1gating: %d tokens < min_capacity %d" % (S, min_cap))
    C = R.moe_capacity(S, E, cf, min_cap, 1)
    if C > S:
        raise ValueError("top1gating: capacity %d > %d tokens" % (C, S))
    return C


def top1gating(logits, uniform, capacity_factor, min_capacity):
    """logits fp32 [S,E]; uniform fp32 [S,E] in [0, 1).  Returns the record keys of R.top2gating (second choice empty: idx2 = -1,
    keep2 = False, g2 = 0)."""
    S, E = logits.shape
    C = top1_checks(S, E, capacity_factor, min_capacity)
    gates = F.softmax(logits, dim=1)
    idx1 = torch.argmax(gates, dim=1)
    mask1 = F.one_hot(idx1, num_classes=E)
    exp_counts = torch.sum(mask1, dim=0).detach()
    me = torch.mean(gates, dim=0)
    ce = torch.mean(mask1.float(), dim=0)
    l_aux = torch.sum(me * ce) * E
    # topk(mask1 * u, C, dim=0) with the tie rule: a stable descending sort keeps the lower index first among equal keys, and unrouted
    # tokens sort below every routed one (key -1 instead of 0)
    key = torch.where(mask1.bool(), uniform, torch.full_like(uniform, -1.0))
    top_idx = torch.sort(key, dim=0, descending=True, stable=True).indices[:C]
    mask1 = mask1 * torch.zeros_like(mask1).scatter_(0, top_idx, 1)
    loc1 = torch.cumsum(mask1, dim=0) - 1
    slot1 = torch.sum(loc1 * mask1, dim=1)
    m1f = mask1.float()
    g1 = torch.einsum("se,se->s", gates, m1f)
    combine = torch.einsum("se,sc->sec", gates * m1f, F.one_hot(slot1, num_classes=C).float())
    return dict(l_aux=l_aux, combine=combine, dispatch=combine.bool(), exp_counts=exp_counts,
                idx1=idx1, idx2=torch.full_like(idx1, -1), slot1=slot1, slot2=torch.zeros_like(slot1),
                keep1=mask1.sum(1).bool(), keep2=torch.zeros(S, dtype=torch.bool), g1=g1, g2=torch.zeros_like(g1), capacity=C,
                gates=gates)


def simulate_top1(logits, uniform, capacity_factor, min_capacity):
    """Token by token, independent of top1gating's tensor formulation: per expert, sort its routed tokens by (-u, index), keep the first
    C, seat the kept ones in token order.  Returns (idx1, keep1, slot1, w1, l_aux, exp_counts, C) as Python lists / floats."""
    S, E = logits.shape
    C = top1_checks(S, E, capacity_factor, min_capacity)
    gates = F.softmax(logits.float(), dim=1)
    idx1 = []
    for s in range(S):
        row = gates[s].tolist()
        best = 0
        for e in range(1, E):
            if row[e] > row[best]:
                best = e
        idx1.append(best)
    counts = [idx1.count(e) for e in range(E)]
    keep = [False] * S
    for e in range(E):
        toks = [s for s in range(S) if idx1[s] == e]
        toks.sort(key=lambda s: (-float(uniform[s, e]), s))
        for s in toks[:C]:
            keep[s] = True
    slot = [0] * S
    seen = [0] * E
    for s in range(S):
        if keep[s]:
            slot[s] = seen[idx1[s]]
            seen[idx1[s]] += 1
    w = [float(gates[s, idx1[s]]) if keep[s] else 0.0 for s in range(S)]
    gm = gates.double().mean(0)
    l_aux = float(E * sum(float(gm[e]) * counts[e] / S for e in range(E)))
    return idx1, keep, slot, w, l_aux, counts, C


def moe_layer_top1(sd, pre, cfg, x, uniform, record=None):
    """R.moe_layer with top1gating: dispatch einsum, the experts, combine einsum; returns (out, l_aux, exp_counts)."""
    shp = x.shape
    xs = x.reshape(-1, shp[-1])
    logits = F.linear(xs.float(), sd[pre + "gate.wg.weight"].float())
    r = top1gating(logits, uniform, cfg.capacity_factor, cfg.min_capacity)
    if record is not None:
        record.append({k: v for k, v in r.items() if k not in ("combine", "dispatch")} | {"logits": logits})
    dispatched = torch.einsum("sec,sm->ecm", r["dispatch"].type_as(xs), xs)
    outs = [R.mlp(sd, pre + f"experts.deepspeed_experts.{e}.", dispatched[e]) for e in range(cfg.num_experts)]
    combined = torch.einsum("sec,ecm->sm", r["combine"].type_as(xs), torch.stack(outs, 0))
    return combined.reshape(shp), r["l_aux"], r["exp_counts"]


def moe_layer(sd, pre, cfg, x, noise, record=None):
    """Dispatch on cfg.top_k: 1 -> top1gating (noise is the uniform), 2 -> R.moe_layer (noise is the Gumbel noise)."""
    if getattr(cfg, "top_k", 2) == 1:
        return moe_layer_top1(sd, pre, cfg, x, noise, record)
    return _R_MOE_LAYER(sd, pre, cfg, x, noise, record)


_R_MOE_LAYER = R.moe_layer


@contextlib.contextmanager
def dispatching_moe_layer():
    """oracle/restated.py's model forwards with moe_layer dispatching on cfg.top_k."""
    R.moe_layer = moe_layer
    try:
        yield
    finally:
        R.moe_layer = _R_MOE_LAYER


def llava_forward(sd, cfg, clip_cfg, input_ids, attention_mask, labels, images, moe_noise=None, record=None):
    with dispatching_moe_layer():
        return R.llava_forward(sd, cfg, clip_cfg, input_ids, attention_mask, labels, images, moe_noise, record)
