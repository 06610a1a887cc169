"""The sparse-MoE block (router, token scatter, grouped expert GEMMs, combine and the five backward kernels) element by element against
the float64 reference of tests/helpers.py, with every routing edge planted exactly; and the grouped GEMM on its own.

Routing is planted, not sampled: column e < E of x and wg[e, e] = 4 make expert e the first choice, the noise (an input tensor) adds 10
to the second choice, and special tokens are one-hot rows of x that select a column of wg holding their exact fp32 logits (equal
logits, a 1-ulp near tie, a tie in logits + noise, a dropped first choice with a second gate below FLT_EPSILON, both choices dropped).
The first- and second-choice counts per expert are chosen so that experts overflow, receive exactly C tokens, counts that are 0 or 1
mod 128, or no token at all."""
import math

import pytest
import torch

from oracle import restated as R
from tests import helpers as Hh

pytestmark = pytest.mark.gpu

ALL = ("equal logits", "1-ulp near tie", "tie in logits + noise", "dropped first, clamped second", "both dropped")
CASES = [
    # id, S, H, I, E, cf, min_cap, first-choice counts, second-choice counts, planted edges, clamp_to, l_aux weight
    # config 2: experts 0 and 1 overflow (first / second choices dropped), expert 2 gets 513 = 1 mod 128 rows, expert 3 256 = 0 mod 128
    ("config2", 2048, 1024, 2816, 4, 1.5, 0, [1600, 200, 120, 128], [27, 1500, 393, 128], ALL, None, 0.37),
    ("1.8B-4E-S2048", 2048, 2048, 5504, 4, 1.5, 0, [1600, 200, 120, 128], [27, 1500, 393, 128], ALL, None, 0.37),
    ("1.8B-4E-S4096", 4096, 2048, 5504, 4, 1.5, 0, [3200, 400, 300, 196], [40, 2900, 340, 816], ALL, None, 0.0),
    # E = 8 with an empty expert and min_capacity 800 above the ceil rule (768)
    ("E8", 2048, 1024, 1408, 8, 1.5, 800, [900, 300, 200, 200, 150, 129, 169, 0], [10, 600, 200, 300, 300, 300, 338, 0], ALL, 3, 0.0),
    # unfused (I = 320 is not a multiple of 128), E = 2
    ("I320-E2", 333, 256, 320, 2, 0.6, 0, [220, 113], [113, 220], ("equal logits", "1-ulp near tie", "both dropped"), None, 0.37),
    # ragged S, non-dyadic cf: expert 1 receives exactly C = 1126 rows
    ("S2047", 2047, 1024, 2816, 4, 1.1, 0, [1200, 400, 247, 200], [30, 726, 400, 891], ALL[:4], 2, 0.37),
    # non-dyadic factors where a factor rounded to fp32 gives another capacity (48 and 573; fp32 gives 49 and 572)
    ("cf0.3", 320, 256, 384, 4, 0.3, 0, [150, 80, 70, 20], [10, 150, 132, 28], ALL, 3, 0.37),
    ("cf1.1", 1040, 512, 512, 4, 1.1, 0, [700, 140, 100, 100], [20, 500, 300, 220], ALL, 3, 0.37),
]
STAGES_FWD = ("logits", "gates", "h1", "act", "y")
STAGES_BWD = ("dw", "dact", "dh1", "dxp", "dlogits", "dx", "g_wg", "g_w_gu", "g_w_dn")
REPORT = {}


def _inputs(S, H, I, E, cf, mc, n1, n2, specials, clamp_to, seed):
    rows = [r for r in Hh.moe_special_rows(E, S, clamp_to) if r[4] in specials]
    pairs = Hh.moe_force_pairs(Hh.moe_plan_pairs(S, E, n1, n2, seed), rows)
    x, wg, noise = Hh.moe_planted_inputs(pairs, E, H, [(s, l, n) for s, l, n, _, _ in rows], seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    w_gu = (torch.randn(E, 2 * I, H, device=dev, generator=g) / math.sqrt(H)).to(torch.bfloat16)
    w_dn = (torch.randn(E, H, I, device=dev, generator=g) / math.sqrt(I)).to(torch.bfloat16)
    res = torch.randn(S, H, device=dev, generator=g).to(torch.bfloat16)
    dout = (torch.randn(S, H, device=dev, generator=g) * 0.1).to(torch.bfloat16)
    old = dict(wg=torch.randn(E, H, device=dev, generator=g) * 1e-2,                 # the dtypes TrainState hands out: fp32 router,
               w_gu=(torch.randn(E, 2 * I, H, device=dev, generator=g) * 1e-2).to(torch.bfloat16),   # bf16 experts
               w_dn=(torch.randn(E, H, I, device=dev, generator=g) * 1e-2).to(torch.bfloat16))
    return rows, pairs, x.cuda(), wg.cuda(), noise.cuda(), w_gu, w_dn, res, dout, old


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_moe_block_stage_by_stage(case):
    from llavamod import kernels as K
    name, S, H, I, E, cf, mc, n1, n2, specials, clamp_to, g_laux = case
    rows, pairs, x, wg, noise, w_gu, w_dn, res, dout, old = _inputs(S, H, I, E, cf, mc, n1, n2, specials, clamp_to, S + H + E)
    assert K.moe_capacity(S, E, cf, mc) == R.moe_capacity(S, E, cf, mc)
    paths = [False, True] if I % 128 == 0 else [False]
    runs = {}
    report = REPORT.setdefault(name, {})
    for fused in paths:
        k = Hh.moe_run_stages(x, res, wg, w_gu, w_dn, noise, cf, mc, dout, g_laux, old, fused)
        ref = Hh.moe_reference_fp64(x, res, wg, w_gu, w_dn, noise, cf, mc, dout=dout, g_laux=g_laux, old=old, k=k, store=torch.float32)
        assert torch.equal(ref["rec"]["idx"].cpu(), pairs)           # the planted routing is the oracle's
        Hh.check_moe_stages(k, ref, E, old, report)
        rec = ref["rec"]
        for s, _, _, _, what in rows:
            if what == "both dropped":
                assert int(k["row"][s, 0]) == -1 and int(k["row"][s, 1]) == -1
                Hh.check_moe("out (both dropped)", k["out"][s], res[s])
            if what == "dropped first, clamped second":
                assert int(k["row"][s, 0]) == -1 and int(k["row"][s, 1]) >= 0
                assert float(k["gates"][s, rec["idx"][s, 1]]) < Hh.FLT_EPS
        assert int((~rec["keep"][:, 0]).sum()) > 0 and int((~rec["keep"][:, 1]).sum()) > 0
        del ref
        # a second launch gives the same bytes (no float atomics on the path: integer shared-memory counters, fixed-order sums)
        k2 = Hh.moe_run_stages(x, res, wg, w_gu, w_dn, noise, cf, mc, dout, g_laux, old, fused)
        n = int(k["offsets"][-1])                                    # rows past offsets[E] are never written (uninitialised)
        for key, v in k.items():
            if isinstance(v, torch.Tensor):
                v, v2 = (v[:n], k2[key][:n]) if v.shape[0] == k["max_rows"] else (v, k2[key])
                assert torch.equal(v, v2), f"{key} differs between two launches"
        del k2
        runs[fused] = k
    if len(paths) == 2:                                              # fused and unfused SwiGLU agree bit for bit
        a, b = runs[False], runs[True]
        n = int(a["offsets"][-1])
        for key in ("out", "h1", "act", "y", "dy", "dw", "dh1", "dxp", "dlogits", "dx", "g_wg", "g_w_gu", "g_w_dn"):
            va, vb = (a[key][:n], b[key][:n]) if a[key].shape[0] == a["max_rows"] else (a[key], b[key])
            assert torch.equal(va, vb), f"{key}: fused and unfused SwiGLU differ"
    # MoEFn (FUSE_SWIGLU auto, and "1") and the no-grad eval path give the stage functions' bytes
    saved = K.FUSE_SWIGLU
    try:
        for mode in ("auto", "1") if I % 128 == 0 else ("auto",):
            K.FUSE_SWIGLU = mode
            fused = K.swiglu_fusable(I, H, training=True)
            want = runs[fused]
            grads = {kk: v.clone() for kk, v in old.items()}
            xd, rd = x.clone().requires_grad_(True), res.clone().requires_grad_(True)
            out, l_aux = K.MoEFn.apply(xd, rd, wg, w_gu, w_dn, noise, cf, mc, grads)
            ((out.float() * dout.float()).sum() + g_laux * l_aux).backward()
            assert torch.equal(out, want["out"]) and torch.equal(l_aux, want["meta"][0])
            assert torch.equal(xd.grad, want["dx"]) and torch.equal(rd.grad, dout)
            for gname in ("wg", "w_gu", "w_dn"):
                assert torch.equal(grads[gname], want["g_" + gname]), gname
        K.FUSE_SWIGLU = saved
        with torch.no_grad():
            out_ng, la_ng, _ = K.moe_forward_nograd(x, res, wg, w_gu, w_dn, noise, cf, mc)
        assert torch.equal(out_ng, runs[False]["out"]) and torch.equal(la_ng, runs[False]["meta"][0])
    finally:
        K.FUSE_SWIGLU = saved
    print(f"\n{name}: max err/bound " + ", ".join(f"{k} {v:.3g}" for k, v in report.items() if v) +
          f"; peak allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


# ---------------------------------------------------------------------------------------------------------------------
# grouped GEMM on its own (lmod_grouped_gemm_bf16 modes 0 / 1 / 2)
# ---------------------------------------------------------------------------------------------------------------------
def _grouped_case(sizes, align, K_, N, seed):
    offs = [0]
    for n in sizes:
        offs.append(offs[-1] + -(-n // align) * align)
    g = torch.Generator(device="cuda").manual_seed(seed)
    R_ = offs[-1] + 128
    a = torch.randn(R_, K_, device="cuda", generator=g).to(torch.bfloat16)
    for i, n in enumerate(sizes):                                   # rows past a group's real size are zero, as the router leaves them
        a[offs[i] + n:offs[i + 1]] = 0
    return offs, a


def _pick_bn(m_tiles, N):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 256 if (m_tiles * -(-N // 256) >= sms * 3 // 2 or N <= 128) else 128


@pytest.mark.parametrize("wide", [False, True], ids=["bn128", "bn256"])
def test_grouped_gemm_ragged_eight_groups(wide):
    """G = 8 ragged 128-aligned groups, two of them empty; N on both sides of pick_bn's 1.5-wave rule (computed from this device)."""
    from llavamod import kernels as Kk
    G, K_ = 8, 384
    sizes = [300, 0, 128, 1, 513, 0, 256, 77]
    offs, a = _grouped_case(sizes, 128, K_, 0, 11)
    m_tiles = (len(a) + 127) // 128
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = 256 * -(-(sms * 3 // 2) // m_tiles) if wide else 256
    assert (_pick_bn(m_tiles, N) == 256) == wide
    g = torch.Generator(device="cuda").manual_seed(12)
    w = (torch.randn(G, N, K_, device="cuda", generator=g) / math.sqrt(K_)).to(torch.bfloat16)
    offsets = torch.tensor(offs, dtype=torch.int32, device="cuda")
    y = torch.full((len(a), N), 7.0, device="cuda", dtype=torch.bfloat16)
    Kk.grouped_gemm(a, w, y, offsets, 0)
    f64 = torch.float64
    for e in range(G):
        r0, r1 = offs[e], offs[e + 1]
        if r1 > r0:
            A, B = a[r0:r1].to(f64), w[e].to(f64).t()
            ref = A @ B
            Hh.check_moe(f"mode 0 group {e}", y[r0:r1], ref, Hh._gemm_tol(ref, A.abs() @ B.abs(), K_))
    assert bool((y[offs[-1]:] == 7.0).all())                        # rows past the last group untouched
    dy = (torch.randn(len(a), N, device="cuda", generator=g)).to(torch.bfloat16)
    dx = torch.full((len(a), K_), 7.0, device="cuda", dtype=torch.bfloat16)
    Kk.grouped_gemm(dy, w, dx, offsets, 1)                          # mode 1: dx = dy @ w[e] (w stored [G, N, K] = [G, K_red, N_out])
    for e in range(G):
        r0, r1 = offs[e], offs[e + 1]
        if r1 > r0:
            A, B = dy[r0:r1].to(f64), w[e].to(f64)
            ref = A @ B
            Hh.check_moe(f"mode 1 group {e}", dx[r0:r1], ref, Hh._gemm_tol(ref, A.abs() @ B.abs(), N))


def test_grouped_wgrad_on_64_aligned_bounds_into_a_prefilled_buffer():
    """Mode 2 on group bounds that are multiples of 64 but not of 128 (its documented requirement), accumulating into a non-zero bf16
    buffer; empty groups keep their bytes."""
    from llavamod import kernels as Kk
    G, M, N = 8, 256, 384
    sizes = [64, 0, 192, 320, 64, 0, 448, 1]
    offs, a = _grouped_case(sizes, 64, M, 0, 21)
    assert any(o % 128 for o in offs)
    g = torch.Generator(device="cuda").manual_seed(22)
    b = torch.randn(len(a), N, device="cuda", generator=g).to(torch.bfloat16)
    offsets = torch.tensor(offs, dtype=torch.int32, device="cuda")
    old = torch.randn(G, M, N, device="cuda", generator=g).to(torch.bfloat16)
    dw = old.clone()
    Kk.grouped_gemm(a, b, dw, offsets, 2, max_rows=offs[-1], accumulate=True)
    f64 = torch.float64
    for e in range(G):
        r0, r1 = offs[e], offs[e + 1]
        if r1 == r0:
            Hh.check_moe(f"mode 2 empty group {e}", dw[e], old[e])
            continue
        A, B = a[r0:r1].to(f64), b[r0:r1].to(f64)
        ref = A.t() @ B + old[e].to(f64)
        Hh.check_moe(f"mode 2 group {e}", dw[e], ref, Hh._gemm_tol(ref, A.abs().t() @ B.abs(), r1 - r0) + 2.0 ** -23 * ref.abs())
