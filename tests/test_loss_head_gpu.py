"""The loss head at full vocabulary, element by element: the streaming KL+CE kernel (csrc/kl.cu kl_stream_kernel) with many rows per
cluster, its numeric edges and its documented variants against the float64 reference of tests/helpers.py, and the split-K lm_head dgrad
(kernels.mm_nn) against a float64 GEMM.

The stream kernel gives each cluster of two CTAs the rows cid, cid + ncl, ... (ncl = co-resident clusters, ~66 on an H100), and carries
its ring stage / phase counters, the held pass-1 chunks and the alternating exchange slot from one active row to the next; a test with
fewer rows than clusters sees one row per cluster and none of that state.  Every test here runs several rows per cluster.

Bounds (derived in tests/helpers.py): dlogits |g_k - g| <= 2^-8 |g| + 2e-5 (ca q + cb p); row_out lse / nll within 1e-5 + 2e-6 |lse|,
x within 2e-5 |x| + 1e-5; the loss scalars within 2e-5 relative."""
import os
import re
import subprocess
import sys

import pytest
import torch

from oracle import restated as R
from tests.helpers import (IGNORE_INDEX, check_dlogits, check_out4, check_row_out, kl_reference_fp64, kl_row_masks)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200")

V_FULL = 151936
KS_CH = 8192                 # csrc/kl.cu: logit pairs per ring stage
N_MANY, T_MANY = 720, 240    # rows of the many-rows tests (three sequences): >= 3x the co-resident clusters, checked below


def dev():
    return torch.device("cuda:0")


def half_start(V, cs=2):
    """First vocabulary column of the second CTA of a row (kl_stream_kernel's v0 of rank 1)."""
    per = (V + cs - 1) // cs
    return (per + 7) // 8 * 8


def make_logits(N, V, seed, scale=3.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = torch.randn(N, V, device="cuda", generator=g) * scale
    t = torch.randn(N, V, device="cuda", generator=g) * scale + 0.5 * s
    return s.to(torch.bfloat16), t.to(torch.bfloat16)


def run_labels(N, T, V, seed):
    """Labels in runs: a leading ignored run longer than two cluster strides (every cluster meets consecutive inactive rows), then runs of
    labelled and ignored positions of mixed lengths, so that clusters meet KD-only rows (next label ignored or sequence end), CE-only rows
    (own label ignored, next one set) and inactive rows between active ones.  Some labels sit at v0 - 1, v0 (the half boundary), 0, V - 1."""
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (N,), generator=g)
    lab[:150] = IGNORE_INDEX
    i, on = 150, True
    while i < N:
        n = int(torch.randint(1, 9 if on else 5, (1,), generator=g))
        if not on:
            lab[i:i + n] = IGNORE_INDEX
        i, on = i + n, not on
    v0 = half_start(V)
    special = [v for v in (v0 - 1, v0, 0, V - 1) if 0 <= v < V]
    valid = torch.nonzero(lab != IGNORE_INDEX).reshape(-1)
    for j, k in enumerate(valid[:: max(1, len(valid) // 40)].tolist()):
        lab[k] = special[j % len(special)]
    return lab


def run_and_check(s, t, lab, T, V, w_ce, distill_all, w_kd=1.0, msg=""):
    """One launch against the reference, then in-place and repeat launches against the first one's bytes."""
    from llavamod import kernels as K
    ld = lab.to(dev())
    d = torch.empty_like(s)
    out4, row_out = K.kl_fused(s, t, ld, T, V, w_kd, w_ce, distill_all, dlogits=d)
    ref = kl_reference_fp64(s, t, ld, T, V, w_kd, w_ce, distill_all, g_dtype=torch.float32)
    check_out4(out4, ref, msg)
    check_row_out(row_out, ref, msg)
    check_dlogits(d, ref, msg)
    m_kd, m_ce, _ = kl_row_masks(ld, T, distill_all)
    inactive = ~(m_kd | m_ce)
    assert bool((d[inactive] == 0).all()) and bool((row_out[inactive] == 0).all()), msg
    del ref
    # in place (dlogits aliases the student logits) and a second launch: the same bytes (no atomics on this path; a difference is a race)
    s2 = s.clone()
    out4_b, row_b = K.kl_fused(s2, t, ld, T, V, w_kd, w_ce, distill_all, dlogits=s2)
    assert torch.equal(s2, d) and torch.equal(row_b, row_out) and torch.equal(out4_b, out4), msg
    del s2
    d2 = torch.full_like(d, float("nan"))
    out4_c, row_c = K.kl_fused(s, t, ld, T, V, w_kd, w_ce, distill_all, dlogits=d2)
    assert torch.equal(d2, d) and torch.equal(row_c, row_out) and torch.equal(out4_c, out4), msg
    return d, out4, row_out


def child(code, env_extra, *args, timeout=600):
    """Runs `code` in a fresh interpreter with the package importable and `env_extra` in its environment; waits for it."""
    env = dict(os.environ, **env_extra)
    return subprocess.run([sys.executable, "-c", f"import sys; sys.path[:0] = [{ROOT!r}, {PKG!r}]\n" + code, *map(str, args)], env=env,
                          capture_output=True, text=True, timeout=timeout, check=True)


# ---------------------------------------------------------------------------------------------------------------------
# the reference itself, pinned to the oracle (no GPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("distill_all", [False, True])
def test_reference_fp64_matches_oracle(distill_all):
    B, T, V, w_kd, w_ce = 2, 12, 96, 0.7, 1.3
    g = torch.Generator().manual_seed(7)
    s = torch.randn(B * T, V, generator=g) * 3
    t = torch.randn(B * T, V, generator=g) * 3 + 0.5 * s
    s[1, 5] = s[4, 0] = s[13, 95] = float("-inf")            # -inf student logits: dropped from x
    s[9, 40:48] = float("-inf")
    t[9, 41] = t[20, 3] = float("-inf")                       # -inf teacher logits (one under a -inf student logit)
    labels = torch.randint(48, V - 1, (B, T), generator=g)    # never on a -inf student column (the nll would be inf)
    labels[0, :3] = labels[0, 7:9] = labels[1, 5] = labels[1, T - 1] = IGNORE_INDEX
    flat = labels.reshape(-1)
    m_kd, m_ce, nxt = kl_row_masks(flat, T, distill_all)
    assert not torch.isinf(s[m_ce, nxt[m_ce]]).any()
    ref = kl_reference_fp64(s, t, flat, T, V, w_kd, w_ce, distill_all)

    sl = s.view(B, T, V).clone().requires_grad_(True)
    logp, p = R.get_logp(sl, V), R.get_p(t.view(B, T, V), V)
    align = R.compute_align_loss(logp, p, labels, distill_all)
    ce = R.shifted_ce(sl, labels, V)
    (w_kd * align + w_ce * ce).backward()
    assert abs(ref["align"] - align.item()) <= 1e-5 * abs(align.item())
    assert abs(ref["ce"] - ce.item()) <= 1e-5 * abs(ce.item())
    assert ref["n_kd"] == float(m_kd.sum()) and ref["n_ce"] == float(m_ce.sum())
    # per row: x = -(align over that row alone), nll = CE over that row's next label alone, lse from the oracle's log-softmax
    for r in range(B * T):
        if not (m_kd[r] or m_ce[r]):
            assert torch.equal(ref["row"][r], torch.zeros(4, dtype=torch.float64))
            continue
        one = torch.full((B * T,), IGNORE_INDEX)
        one[r] = 0
        x = -R.compute_align_loss(logp.detach(), p, one.view(B, T))
        assert abs(ref["row"][r, 0].item() - x.item()) <= 1e-5 * abs(x.item()) + 1e-6, r
        if m_ce[r]:
            one = torch.full((B * T,), IGNORE_INDEX)
            one[r + 1] = nxt[r]
            nll = R.shifted_ce(s.view(B, T, V), one.view(B, T), V)
            assert abs(ref["row"][r, 1].item() - nll.item()) <= 1e-5 * abs(nll.item()) + 1e-6, r
        else:
            assert ref["row"][r, 1].item() == 0.0
        j = int(torch.nonzero(torch.isfinite(s[r]))[0])
        assert abs(ref["row"][r, 2].item() - (s[r, j] - logp.view(-1, V)[r, j]).item()) <= 1e-5
        assert abs(ref["row"][r, 3].item() - torch.logsumexp(t[r], 0).item()) <= 1e-5
    # gradient: autograd on the rows where the student logits are finite; on the others autograd's ckd (q sum_kept p - p [kept]) and the
    # kernel's ckd (q - p) differ by ckd (q sum_dropped p - p [dropped]) exactly
    got = sl.grad.view(B * T, V).double()
    dropped = torch.isinf(s)
    q, pd = torch.softmax(s.double(), -1), torch.softmax(t.double(), -1)
    ckd = w_kd / ref["n_kd"] * m_kd.double()
    fix = ckd[:, None] * (q * (pd * dropped).sum(-1, keepdim=True) - pd * dropped)
    torch.testing.assert_close(ref["g"], got + fix, rtol=1e-5, atol=1e-8)
    a = (w_kd / ref["n_kd"] * m_kd.double() + w_ce / ref["n_ce"] * m_ce.double())[:, None]
    torch.testing.assert_close(ref["gscale"], a * q + ckd[:, None] * pd, rtol=1e-12, atol=0)


# ---------------------------------------------------------------------------------------------------------------------
# many rows per cluster, default path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_many_row_tests_give_every_cluster_several_rows():
    """The stream kernel's grid is min(rows, co-resident clusters); the kernel reports the cluster count under LMOD_KL_VERBOSE=1."""
    r = child("import torch\nfrom llavamod import kernels as K\n"
              "s = torch.zeros(4, 1024, dtype=torch.bfloat16, device='cuda')\n"
              "K.kl_fused(s, s, torch.arange(4, device='cuda'), 4, 1024, 1.0, 1.0, dlogits=torch.empty_like(s))\n"
              "torch.cuda.synchronize()\n", {"LMOD_KL_VERBOSE": "1"})
    m = re.search(r"kl_stream_kernel<[^>]*>: cluster (\d+), \d+ B smem, (\d+) co-resident clusters", r.stderr)
    assert m, r.stderr
    cs, ncl = int(m.group(1)), int(m.group(2))
    assert cs == 2 and ncl > 0
    assert N_MANY >= 3 * ncl, (N_MANY, ncl)
    assert VARIANT_N >= 3 * ncl                                # the variant tests and the 600-row compact case of test_rows_gpu


# V and the chunking case it forces: per half of the row (length, chunks, chunks held in the ring into pass 2, chunks re-fetched from L2)
VOCABS = [
    (151936, [(75968, 10, 6, 4), (75968, 10, 6, 4)]),
    (114688, [(57344, 7, 6, 1), (57344, 7, 6, 1)]),
    (98304, [(49152, 6, 6, 0), (49152, 6, 6, 0)]),        # exactly KS_STAGES chunks: all held
    (16392, [(8200, 2, 2, 0), (8192, 1, 1, 0)]),          # halves with different chunk counts
    (1000, [(504, 1, 1, 0), (496, 1, 1, 0)]),             # second half shorter
    (8, [(8, 1, 1, 0), (0, 0, 0, 0)]),                    # second half empty
]


@pytest.mark.gpu
@pytest.mark.parametrize("w_ce,distill_all", [(1.0, False), (0.0, False), (1.0, True)])
@pytest.mark.parametrize("V", [v for v, _ in VOCABS])
def test_stream_kernel_many_rows_per_cluster(V, w_ce, distill_all):
    s, t = make_logits(N_MANY, V, seed=V)
    lab = run_labels(N_MANY, T_MANY, V, seed=V + 1)
    m_kd, m_ce, _ = kl_row_masks(lab, T_MANY, distill_all)
    if not distill_all:                                        # the mixture the labels are built for
        assert bool((m_kd & ~m_ce).any() and (m_ce & ~m_kd).any() and (~m_kd & ~m_ce).any())
    run_and_check(s, t, lab, T_MANY, V, w_ce, distill_all, msg=f"V={V} w_ce={w_ce} distill_all={distill_all}")


def kernel_constant(name):
    src = open(os.path.join(PKG, "csrc", "kl.cu")).read()
    m = re.search(r"constexpr int %s = (\d+);" % name, src)
    assert m, name
    return int(m.group(1))


def test_vocab_cases_force_their_chunking():
    """The VOCABS table against the stream kernel's own constants (csrc/kl.cu) and its per-CTA rules: slice = round_up(ceil(V / KS_CS), 8),
    len = clamp(V - rank * slice, 0, slice), nchunks = ceil(len / KS_CH), held = min(KS_STAGES, nchunks), pass 2 re-fetches the rest."""
    assert kernel_constant("KS_CH") == KS_CH
    cs, stages = kernel_constant("KS_CS"), kernel_constant("KS_STAGES")
    assert cs == 2
    for V, halves in VOCABS:
        slice_ = half_start(V, cs)
        got = []
        for rank in range(cs):
            n = max(0, min(slice_, V - rank * slice_))
            nchunks = -(-n // KS_CH)
            held = min(stages, nchunks)
            got.append((n, nchunks, held, nchunks - held))
        assert got == halves, (V, got)


# ---------------------------------------------------------------------------------------------------------------------
# numeric edges at V = 151936
# ---------------------------------------------------------------------------------------------------------------------
EDGE_ROWS = dict(inf_student=(3, 140), inf_teacher=(7, 201), peaked_teacher=(20, 150, 299), all_equal=(50, 230))


def edge_inputs(target, c):
    """300 rows at the full vocabulary with edge rows on first and later rows of the clusters; c added to every student (target 's') or
    teacher ('t') logit.  Every edge row carries its own label (KD mask set), so the kernel computes it."""
    N, T, V = 300, 100, V_FULL
    s, t = make_logits(N, V, seed=17)
    s, t = s.float(), t.float()
    v0 = half_start(V)
    held0, refetch0 = 5 * KS_CH, 0                             # of a half's 10 chunks, 4..9 stay in the ring for pass 2, 0..3 are re-fetched
    for r in EDGE_ROWS["inf_student"]:
        for base in (0, v0):
            s[r, base + refetch0 + 100] = float("-inf")
            s[r, base + held0 + 37] = float("-inf")
            s[r, base + 3 * KS_CH + 5] = float("-inf")
        s[r, 2 * KS_CH: 2 * KS_CH + 8] = float("-inf")          # a whole 16-byte vector, re-fetched chunk of the first half
        s[r, v0 + 9 * KS_CH + 8: v0 + 9 * KS_CH + 16] = float("-inf")   # a whole vector in the last (held, partial) chunk of the second half
    for r in EDGE_ROWS["inf_teacher"]:                          # -inf teacher logits in both halves, re-fetched and held chunks, a whole vector
        t[r, 11] = t[r, 4 * KS_CH + 64: 4 * KS_CH + 72] = t[r, v0 + 7 * KS_CH + 3] = t[r, v0 + 2 * KS_CH + 9] = float("-inf")
    for r in EDGE_ROWS["peaked_teacher"]:                       # sharply peaked teacher, maximum in the last chunk of the second half
        t[r, V - 5] = t[r].max() + 40.0
    for r in EDGE_ROWS["all_equal"]:                            # every logit equal
        s[r] = 1.5
        t[r] = -2.0
    if target == "s":
        s += c
    else:
        t += c
    s, t = s.to(torch.bfloat16), t.to(torch.bfloat16)
    g = torch.Generator().manual_seed(5)
    lab = torch.randint(0, V, (N,), generator=g)
    for b in range(N // T):
        lab[b * T + 60: b * T + 70] = IGNORE_INDEX             # inactive rows between active ones, away from the edge rows
    lab[[150 - 2, 150 + 1]] = torch.tensor([v0, V - 1])
    bad = torch.isinf(s.float().cpu()[torch.arange(N).roll(1), lab.clamp_min(0)])   # no next label on a -inf student logit
    lab[bad & (lab >= 0)] = 1
    m_kd, _, _ = kl_row_masks(lab, T)
    edge = [r for rows in EDGE_ROWS.values() for r in rows]
    assert bool(m_kd[edge].all()) and not bool(m_kd.all()), "every edge row must be a KD row, and some rows inactive"
    return s, t, lab, T, V


@pytest.mark.gpu
@pytest.mark.parametrize("target,c", [("s", 0.0), ("s", 8.0), ("s", 32.0), ("s", 96.0), ("t", 8.0), ("t", 32.0), ("t", 96.0)])
def test_stream_kernel_numeric_edges(target, c):
    s, t, lab, T, V = edge_inputs(target, c)
    run_and_check(s, t, lab, T, V, 1.0, False, msg=f"offset {c} on {target}")


# ---------------------------------------------------------------------------------------------------------------------
# the documented A/B variants (README), each in its own process: the kernel reads these variables once into statics
# ---------------------------------------------------------------------------------------------------------------------
# name: (environment, the launch line the kernel prints under LMOD_KL_VERBOSE=1 for it -- proof that the variant, not the default, ran)
VARIANTS = {
    "stream1": ({"LMOD_KL_MODE": "stream1"},         # one CTA per row: the single-CTA exchange (named barrier)
                r"kl_stream_kernel<0,0,512>: cluster 1, .* keep_tail 1"),
    "stream4": ({"LMOD_KL_MODE": "stream4"}, r"kl_stream_kernel<0,0,512>: cluster 4, .* keep_tail 1"),
    "sb128": ({"LMOD_KL_MODE": "sb128"},             # the shared-memory-resident 8-CTA kernel
              r"kl_fused_kernel<128,1>: cluster 8,"),
    "keep0": ({"LMOD_KL_KEEP": "0"},                 # nothing held over: pass 2 re-fetches every chunk
              r"kl_stream_kernel<0,0,512>: cluster 2, .* keep_tail 0"),
    "poly33": ({"LMOD_KL_POLY": "33"},               # 3/8 of the exponentials by polynomial
               r"kl_stream_kernel<3,3,512>: cluster 2, .* keep_tail 1"),
    "threads256": ({"LMOD_KL_THREADS": "256"}, r"kl_stream_kernel<0,0,256>: cluster 2, .* keep_tail 1"),
    "threads768": ({"LMOD_KL_THREADS": "768"}, r"kl_stream_kernel<0,0,768>: cluster 2, .* keep_tail 1"),
}
VARIANT_N, VARIANT_T = 600, 200

CHILD_RUN = """import torch
from llavamod import kernels as K
x = torch.load(sys.argv[1])
s, t, lab = x["s"].cuda(), x["t"].cuda(), x["lab"].cuda()
d = torch.empty_like(s)
out4, row_out = K.kl_fused(s, t, lab, x["T"], x["V"], 1.0, 1.0, False, dlogits=d)
torch.cuda.synchronize()
torch.save({"out4": out4.cpu(), "row_out": row_out.cpu(), "d": d.cpu(), "peak": torch.cuda.max_memory_allocated()}, sys.argv[2])
"""


@pytest.fixture(scope="module")
def variant_inputs(tmp_path_factory):
    V = V_FULL
    s, t = make_logits(VARIANT_N, V, seed=23)
    lab = run_labels(VARIANT_N, VARIANT_T, V, seed=24)
    path = tmp_path_factory.mktemp("kl_variants") / "inputs.pt"
    torch.save({"s": s.cpu(), "t": t.cpu(), "lab": lab, "T": VARIANT_T, "V": V}, path)
    ref = kl_reference_fp64(s, t, lab.to(dev()), VARIANT_T, V, 1.0, 1.0, False, g_dtype=torch.float32)
    return path, ref, lab


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VARIANTS))
def test_stream_kernel_variants(name, variant_inputs, tmp_path):
    inputs, ref, lab = variant_inputs
    out = tmp_path / f"{name}.pt"
    env, launch = VARIANTS[name]
    r = child(CHILD_RUN, dict(env, LMOD_KL_VERBOSE="1"), inputs, out)
    assert re.search(launch, r.stderr), (name, r.stderr)
    got = torch.load(out)
    print(f"{name}: child peak GPU memory {got['peak'] / 2**30:.2f} GiB")
    check_out4(got["out4"], ref, name)
    check_row_out(got["row_out"], ref, name)
    d = got["d"].to(dev())
    check_dlogits(d, ref, name)
    m_kd, m_ce, _ = kl_row_masks(lab, VARIANT_T)
    assert bool((d[~(m_kd | m_ce).to(dev())] == 0).all()), name


# ---------------------------------------------------------------------------------------------------------------------
# split-K lm_head dgrad: dx[M, H] = dy[M, 151936] @ w[151936, H]
# ---------------------------------------------------------------------------------------------------------------------
def dgrad_ref_fp64(dy, w, block=16384):
    acc = torch.zeros(dy.shape[0], w.shape[1], dtype=torch.float64, device=dy.device)
    for k0 in range(0, dy.shape[1], block):
        acc += dy[:, k0:k0 + block].double() @ w[k0:k0 + block].double()
    return acc


def accumulation_extra(ref, split, K=V_FULL, BK=64):
    """Absolute error of the wgmma fp32 accumulator over a long reduction, the `extra` of test_gemm_gpu.check: every k=16 step adds into the
    accumulator truncating toward zero, up to one ulp (2^-23 relative) of a partial sum of the order of rms(ref), so the error grows with the
    k-steps ONE accumulator takes (K / split), not with sqrt(K).  Measured on an H100 (random bf16 operands, K = 151936, split 1..16): max
    error 0.78 x (K/split/16) 2^-23 rms(ref), biased toward zero; the bound takes twice the estimate."""
    k_blocks = -(-K // BK)
    steps = -(-k_blocks // split) * BK // 16                   # k=16 steps of the longest split
    return 2.0 * steps * 2.0 ** -23 * ref.pow(2).mean().sqrt().item()


def record_split_k(monkeypatch):
    from llavamod import kernels as K
    seen, gemm = [], K.gemm

    def wrapped(*a, **kw):
        seen.append(kw.get("split_k", 1))
        return gemm(*a, **kw)
    monkeypatch.setattr(K, "gemm", wrapped)
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("M,H,split", [(128, 1024, True), (128, 2048, True), (300, 1024, True), (300, 2048, True), (2048, 1024, True),
                                       (2048, 2048, False)])   # 16 x 8 = 128 output tiles: enough to fill the GPU, no split
def test_lm_head_dgrad_split_k_matches_fp64(M, H, split, monkeypatch):
    from llavamod import kernels as K
    from tests.test_gemm_gpu import check
    g = torch.Generator(device="cuda").manual_seed(M + H)
    dy = torch.randn(M, V_FULL, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(V_FULL, H, device="cuda", generator=g).to(torch.bfloat16)
    seen = record_split_k(monkeypatch)
    dx = K.mm_nn(dy, w)
    assert len(seen) == 1 and ((seen[0] > 1) == split), seen
    ref = dgrad_ref_fp64(dy, w)
    check(dx, ref, V_FULL, extra=accumulation_extra(ref, seen[0]))


@pytest.mark.gpu
def test_lm_head_dgrad_split_k_dynamic_rows(monkeypatch):
    """The compact loss head's dgrad: 885 active rows of a 1024-row buffer, the extent in device memory.  Rows past the extent up to the
    tile boundary are zero (gather_rows pads them); the tile past it holds garbage that must not reach the output."""
    from llavamod import kernels as K
    from tests.test_gemm_gpu import check
    M, n, H = 1024, 885, 1024
    g = torch.Generator(device="cuda").manual_seed(n)
    dy = torch.randn(M, V_FULL, device="cuda", generator=g).to(torch.bfloat16)
    dy[n:896] = 0
    w = torch.randn(V_FULL, H, device="cuda", generator=g).to(torch.bfloat16)
    seen = record_split_k(monkeypatch)
    dx = K.mm_nn(dy, w, m_dev=torch.tensor([n], dtype=torch.int32, device="cuda"))
    assert len(seen) == 1 and seen[0] > 1, seen
    ref = dgrad_ref_fp64(dy[:n], w)
    check(dx[:n], ref, V_FULL, extra=accumulation_extra(ref, seen[0]))
    assert bool((dx[n:] == 0).all())
