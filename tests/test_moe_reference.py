"""CPU checks of the sparse-MoE block's yardsticks: the float64 reference of tests/helpers.py (moe_reference_fp64) against float64
autograd of the oracle's MoE layer, the library's capacity rule against the oracle's, and the oracle's tie rules, which the kernels'
routing must follow."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restated as R
from tests import helpers as Hh

# non-dyadic capacity factors: not exact in binary, so a factor rounded to fp32 before the product can land on the other side of an integer
NON_DYADIC_CF = [0.05, 0.1, 0.3, 0.35, 0.6, 0.7, 0.9, 1.1, 1.2, 1.3, 1.7, 2.3]


def test_capacity_matches_oracle_for_non_dyadic_factors():
    from llavamod import kernels as K
    sizes = list(range(16, 8193, 16)) + [1, 7, 17, 333, 2047, 4095, 6001]
    bad = []
    for E in range(2, 9):
        for cf in NON_DYADIC_CF + [0.5, 0.75, 1.0, 1.25, 1.5, 2.0]:
            for S in sizes:
                for mc in (0, 4):
                    got, want = K.moe_capacity(S, E, cf, mc), R.moe_capacity(S, E, cf, mc, 2)
                    if got != want:
                        bad.append((S, E, cf, mc, got, want))
    assert not bad, f"{len(bad)} disagreements, e.g. (S, E, cf, min_capacity, library, oracle) {bad[:5]}"
    # min_capacity above the ceil rule wins; the documented example of a factor that fp32 moves: S 320, E 4, cf 0.3 -> 48
    assert K.moe_capacity(64, 4, 0.3, 50) == R.moe_capacity(64, 4, 0.3, 50) == 50
    assert K.moe_capacity(320, 4, 0.3, 0) == 48


def test_oracle_tie_rules():
    """idx1 is the first maximal GATE (softmax can tie where the logits do not); idx2 the first maximum of logits + noise without idx1."""
    nt = float(torch.nextafter(torch.tensor(0.1, dtype=torch.float32), torch.tensor(1.0)))
    logits = torch.tensor([[0.1, nt, -1.0, -2.0], [0.5] * 4, [1.0, 0.5, 0.25, -1.0], [0.0, 2.0, 2.0, 1.0]], dtype=torch.float32)
    noise = torch.tensor([[0.0, 0.0, 10.0, 0.0], [0.0, 3.0, 3.0, 0.0], [0.0, 1.0, 1.25, 0.0], [0.0, 0.0, 0.0, 1.0]])
    assert logits[0, 1] > logits[0, 0]
    gates = torch.softmax(logits, 1)
    assert gates[0, 0] == gates[0, 1]                          # the gates tie although the logits differ by one ulp
    o = R.top2gating(logits, noise, 2.0, 0)
    assert o["idx1"].tolist() == [0, 0, 0, 1]
    assert o["idx2"].tolist() == [2, 1, 1, 2]                  # row 3: logits + noise 2 (expert 2) ties 2 (expert 3) -> the first


def _pin_case(S, H, I, E, cf, mc, n1, n2, specials, seed, clamp_to=None):
    rows = [r for r in Hh.moe_special_rows(E, S, clamp_to) if r[4] in specials]
    pairs = Hh.moe_force_pairs(Hh.moe_plan_pairs(S, E, n1, n2, seed), rows)
    x, wg, noise = Hh.moe_planted_inputs(pairs, E, H, [(s, l, n) for s, l, n, _, _ in rows], seed)
    g = torch.Generator().manual_seed(seed + 1)
    w_gu = (torch.randn(E, 2 * I, H, generator=g) * 0.3).to(torch.bfloat16)
    w_dn = (torch.randn(E, H, I, generator=g) * 0.3).to(torch.bfloat16)
    res = torch.randn(S, H, generator=g).to(torch.bfloat16)
    go = torch.randn(S, H, generator=g).to(torch.bfloat16)
    return rows, pairs, x, wg, noise, w_gu, w_dn, res, go


PIN_CASES = [
    # S, H, I, E, cf, min_cap, first-choice counts, second-choice counts, planted edges, clamp_to
    (48, 64, 24, 4, 1.0, 0, [28, 8, 8, 4], [3, 26, 9, 10], ("equal logits", "1-ulp near tie", "tie in logits + noise",
                                                             "dropped first, clamped second", "both dropped"), None),
    (40, 32, 16, 2, 0.6, 0, [26, 14], [14, 26], ("equal logits", "1-ulp near tie", "both dropped"), None),
    (64, 64, 32, 8, 1.1, 20, [30, 10, 8, 6, 4, 3, 3, 0], [2, 20, 10, 10, 8, 8, 6, 0],
     ("equal logits", "1-ulp near tie", "tie in logits + noise", "dropped first, clamped second", "both dropped"), 3),
]


@pytest.mark.parametrize("S,H,I,E,cf,mc,n1,n2,specials,clamp_to", PIN_CASES)
def test_reference_matches_float64_autograd_of_the_oracle(S, H, I, E, cf, mc, n1, n2, specials, clamp_to):
    rows, pairs, x, wg, noise, w_gu, w_dn, res, go = _pin_case(S, H, I, E, cf, mc, n1, n2, specials, S + E, clamp_to)
    f64 = torch.float64
    pre = "m."
    cfg = R.LMCfg(hidden=H, inter=I, layers=1, heads=4, kv_heads=4, vocab=64, moe_layers=[0], num_experts=E, capacity_factor=cf,
                  min_capacity=mc)
    sd = {pre + "gate.wg.weight": wg.to(f64).requires_grad_(True)}
    for e in range(E):
        ep = pre + f"experts.deepspeed_experts.{e}."
        sd[ep + "gate_proj.weight"] = w_gu[e, :I].to(f64).requires_grad_(True)
        sd[ep + "up_proj.weight"] = w_gu[e, I:].to(f64).requires_grad_(True)
        sd[ep + "down_proj.weight"] = w_dn[e].to(f64).requires_grad_(True)
    xo, ro = x.to(f64).requires_grad_(True), res.to(f64).requires_grad_(True)
    y, la, _ = R.moe_layer(sd, pre, cfg, xo, noise.to(f64))
    out = ro + y
    ((out * go.to(f64)).sum() + 0.37 * la).backward()
    # the reference chained from its own float64 stages; routing from the oracle's fp32 logits; the model's rounding of the combine
    # weights to the activations' dtype does not happen in float64
    ref = Hh.moe_reference_fp64(x, res, wg, w_gu, w_dn, noise, cf, mc, dout=go, g_laux=0.37, k=dict(logits=F.linear(x.float(), wg.float())),
                                w_bf16=False)
    rec = ref["rec"]
    assert torch.equal(rec["idx"], pairs)
    C = rec["capacity"]
    assert C == R.moe_capacity(S, E, cf, mc)
    for s, _, _, _, what in rows:                               # the planted edges happen
        k1, k2 = bool(rec["keep"][s, 0]), bool(rec["keep"][s, 1])
        if what == "both dropped":
            assert not k1 and not k2
            assert torch.equal(ref["out"][0][s], res[s].to(f64))
            assert torch.allclose(ref["dx"][0][s], ref["dx_gate"][s], rtol=0, atol=0)
        if what == "dropped first, clamped second":
            assert not k1 and k2 and float(torch.softmax(ref["logits"][0][s], 0)[rec["idx"][s, 1]]) < Hh.FLT_EPS
    assert int((~rec["keep"][:, 0]).sum()) > 0 and int((~rec["keep"][:, 1]).sum()) > 0

    def close(name, got, want):
        want = want.detach().to(f64)
        err = (got.to(f64) - want).abs()
        tol = 1e-5 * want.abs() + 1e-5 * want.abs().max() + 1e-12
        assert bool((err <= tol).all()), f"{name}: max err {float(err.max()):.3g} (scale {float(want.abs().max()):.3g})"

    close("out", ref["out"][0], out)
    close("l_aux", ref["l_aux"][0], la)
    close("dx", ref["dx"][0], xo.grad)
    close("dwg", ref["g_wg"][0], sd[pre + "gate.wg.weight"].grad)
    for e in range(E):
        ep = pre + f"experts.deepspeed_experts.{e}."
        close(f"dW_gu[{e}]", ref["g_w_gu"][0][e], torch.cat([sd[ep + "gate_proj.weight"].grad, sd[ep + "up_proj.weight"].grad]))
        close(f"dW_dn[{e}]", ref["g_w_dn"][0][e], sd[ep + "down_proj.weight"].grad)
    if 0 in n1 and 0 in n2:                                     # an expert without tokens: zero gradient
        e = n1.index(0)
        assert float(ref["g_w_gu"][0][e].abs().max()) == 0.0 and float(ref["g_w_dn"][0][e].abs().max()) == 0.0


def test_reference_bounds_hold_for_its_own_rounded_stages():
    """The bounds are not vacuous and not violated by plain bf16 rounding: a reference stage rounded to bf16 stays within its bound, and a
    stage perturbed by 1 % of its largest element does not."""
    S, H, I, E = 48, 64, 24, 4
    rows, pairs, x, wg, noise, w_gu, w_dn, res, go = _pin_case(S, H, I, E, 1.0, 0, [28, 8, 8, 4], [3, 26, 9, 10], ("equal logits",), 7)
    ref = Hh.moe_reference_fp64(x, res, wg, w_gu, w_dn, noise, 1.0, 0, dout=go, g_laux=0.37)
    routed = ref["rec"]["tok"] >= 0
    for name in ("h1", "y", "dact", "dxp", "dh1"):
        want, tol = ref[name]
        Hh.check_moe(name, want.to(torch.bfloat16), want, tol, rows=routed)
        bumped = want.clone()
        bumped[routed.nonzero()[0, 0], 0] += 0.01 * float(want.abs().max())
        with pytest.raises(AssertionError, match=name):
            Hh.check_moe(name, bumped, want, tol, rows=routed)
