"""kernels.DistillHeadFn (K.distill_head: the lm_head GEMM, the fused mimic-KL + shifted-CE kernel and the lm_head backward; the loss of
every mimic step) element by element against float64, compact (rows from K.active_rows) and dense, at the full Qwen vocabulary and at the
row-extent edges of the compact path.

Every case
  - runs three micro-batches with different hidden states, teacher logits and upstream scalars g into an lm_head gradient view carved out
    of an arena of sentinels (helpers.Arena), each under helpers.poisoned_uninitialised_memory: the logits rows past the GEMM's last
    stored tile, the gathered rows past the padding and every buffer nobody wrote hold NaN;
  - checks every stage from the kernels' own previous stage (helpers.distill_head_reference_fp64), so each bound covers one stage:
      student logits    the Function's GEMM run again gives d logits and losses with the Function's bits; its rows below count against
                        float64 h[perm] W^T (_gemm_tol, K = H)
      loss, d logits    kl_reference_fp64 on those logits placed back on their rows: align and ce within check_out4's bound, the counts
                        exact, total = w_kd align + w_ce ce to one fp32 rounding, check_dlogits on the active rows; d logits exactly 0 in
                        columns vocab and above and in rows [count, round_up(count, 128))
      d hidden          g (d logits W) from the kernel's d logits: _gemm_tol (K = V_s), plus the split-K term of test_loss_head_gpu when
                        mm_nn splits the reduction, plus one rounding for the product with g; exactly 0 on every row that is not active and
                        in the compact dgrad's rows past count
      lm_head gradient  old + d logits^T (g h) over the active rows, from the value the micro-batch before left (_gemm_tol, K = count,
                        + 2^-23 |ref|); nothing outside the view changes
  - runs twice and requires the same bytes.  The exception is d hidden where mm_nn splits the reduction (the lm_head dgrad with few output
    tiles): its split-K partial sums are added with fp32 atomics in any order, so two runs may differ in the last bit;
  - prints its worst err / bound.
test_upstream_scale checks that g reaches both gradients without a bias; test_tied_embedding the two accumulations into the view that
config 2's tied lm_head shares with the token embedding, in the order autograd runs them."""
import math

import pytest
import torch

from tests.helpers import (BF16_U, DEV, IGNORE_INDEX, Arena, check_dlogits, check_exact_bound, distill_head_reference_fp64,
                           embed_grad_reference_fp64, kl_row_masks, no_nan, poisoned_uninitialised_memory, randn, twice)
from tests.test_loss_head_gpu import accumulation_extra, record_split_k

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
V_QWEN = 151936
V_SMALL = 4136
MICRO_BATCHES = 3
G_MB = (1.0, 0.37, 1.0 / 3.0)                     # the upstream scalar of each micro-batch
PATCHES = 576


def K():
    from llavamod import kernels
    return kernels


def f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def round_up(n, m):
    return -(-n // m) * m


# ---------------------------------------------------------------------------------------------------------------------
# labels
# ---------------------------------------------------------------------------------------------------------------------
def bench_labels(T, V, seed):
    """The bench's layout at T = 2048 (576 image rows + 40 % of 1473 text ids ignored): 884 supervised rows and one CE-only row."""
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (1, T), generator=g)
    lab[0, :1164] = IGNORE_INDEX
    return lab


def run_labels(B, T, V, seed):
    """A prompt, ignored runs inside every sequence and a padded tail on the last one: KD-only, CE-only and inactive rows between active
    ones, and labels 0 and V - 1."""
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (B, T), generator=g)
    lab[:, :T // 4] = IGNORE_INDEX
    for b in range(B):
        for _ in range(6):
            a = int(torch.randint(T // 4, T, (1,), generator=g))
            lab[b, a:a + int(torch.randint(1, 40, (1,), generator=g))] = IGNORE_INDEX
    lab[-1, T - T // 8:] = IGNORE_INDEX
    lab[0, T // 2], lab[0, T // 2 + 1] = 0, V - 1
    return lab


def count_labels(B, T, V, count, seed):
    """Labels with exactly `count` active rows (distill_all False): runs of labels at a sequence start (k labels, k active rows) and inside a
    sequence (k labels, k + 1 active rows: the row before the run is CE-only), the rows between them inactive."""
    for s in range(seed, seed + 1000):
        g = torch.Generator().manual_seed(s)
        lab = torch.full((B, T), IGNORE_INDEX, dtype=torch.long)
        left = count
        for b in range(B):
            free = 0                                                   # first row of the sequence not yet decided
            while left > 0 and free < T:
                k = int(torch.randint(1, 80, (1,), generator=g))
                if free == 0 and int(torch.randint(0, 2, (1,), generator=g)):
                    k = min(k, left, T)
                    lab[b, :k] = torch.randint(0, V, (k,), generator=g)
                    left -= k
                else:
                    s0 = max(free, 1) + int(torch.randint(0, 4, (1,), generator=g))   # the CE-only row s0, labels from s0 + 1
                    k = min(k, left - 1, T - s0 - 1)
                    if k < 1:
                        break
                    lab[b, s0 + 1:s0 + 1 + k] = torch.randint(0, V, (k,), generator=g)
                    left -= k + 1
                    free = s0 + 1 + k + 1
                    continue
                free = k + 1
        m_kd, m_ce, _ = kl_row_masks(lab.reshape(-1), T)
        if left == 0 and int((m_kd | m_ce).sum()) == count:
            return lab
    raise AssertionError(f"no label layout with {count} active rows")


# ---------------------------------------------------------------------------------------------------------------------
# one case: three micro-batches, every stage
# ---------------------------------------------------------------------------------------------------------------------
def record_dgrad(monkeypatch):
    """Every kernels.mm_nn call the Function makes: (its output, the split_k of the GEMM it ran)."""
    seen = record_split_k(monkeypatch)
    calls, mm_nn = [], K().mm_nn

    def wrapped(*a, **kw):
        n0 = len(seen)
        out = mm_nn(*a, **kw)
        calls.append((out.clone(), max(seen[n0:])))
        return out
    monkeypatch.setattr(K(), "mm_nn", wrapped)
    return calls


def teacher_logits(n_rows, n_valid, vocab, ld, seed):
    """[n_rows, ld] bf16: seeded logits in rows < n_valid and columns < vocab, NaN elsewhere (nothing there may be read)."""
    t = torch.full((n_rows, ld), float("nan"), dtype=bf16, device=DEV)
    t[:n_valid, :vocab] = randn(n_valid, vocab, seed=seed, scale=3.0)
    return t


def run_head(k, hidden, W, lab, vocab, w_kd, w_ce, distill_all, view, compact, t_fn, g):
    """The Function as the trainer runs it, under poisoned memory; returns what the checks need."""
    B, T, H = hidden.shape
    with poisoned_uninitialised_memory():
        rows = k.active_rows(lab.reshape(-1), T, distill_all) if compact else None
        count = int(rows[1]) if compact else B * T
        t = t_fn(count)
        total, align, ce = k.distill_head(hidden, W, t, lab, vocab, w_kd, w_ce, distill_all, head_grad=view, rows=rows)
        assert type(total.grad_fn).__name__.startswith("DistillHeadFn")
        dl = total.grad_fn.saved_tensors[0]                            # d logits, written over the logits in the forward
        total.backward(torch.tensor(g, dtype=torch.float32, device=DEV))
    torch.cuda.synchronize()
    return dict(rows=rows, count=count, t=t, total=total.detach(), align=align, ce=ce, dl=dl)


def check_stages(k, r, hidden, W, lab, vocab, w_kd, w_ce, distill_all, g, old, view, split, report, tag):
    """Every stage of one micro-batch against float64 (see the module docstring)."""
    B, T, H = hidden.shape
    N, Vs = B * T, W.shape[0]
    rows, count, dl = r["rows"], r["count"], r["dl"]
    h2 = hidden.detach().reshape(N, H)
    flat = lab.reshape(-1)
    # the Function's GEMM and loss kernel again: the same d logits and losses, bit for bit
    if rows is not None:
        logits = k.gemm(k.gather_rows(h2, *rows), W, m_dev=rows[1])
        stored = round_up(count, 128)
    else:
        logits = k.gemm(h2, W)
        stored = N
    d2 = logits.clone()
    out4, _ = k.kl_fused(d2, r["t"], flat, T, vocab, w_kd, w_ce, distill_all, dlogits=d2, rows=rows)
    if Vs > vocab:
        d2[:, vocab:].zero_()
    assert torch.equal(d2[:stored].view(torch.int16), dl[:stored].view(torch.int16)), f"{tag}: d logits differ from the Function's run"
    assert torch.equal(out4[:2].view(torch.int32), torch.stack([r["align"], r["ce"]]).view(torch.int32)), f"{tag}: losses differ"
    store = torch.float32 if Vs * N > 1 << 26 else torch.float64
    ref = distill_head_reference_fp64(h2, W, r["t"], flat, T, vocab, w_kd, w_ce, distill_all, g, rows=rows, logits=logits, dlogits=dl,
                                      old=old, store=store)
    act = ref["act"]
    own = slice(0, count) if rows is not None else act                 # the kernel rows that hold the active rows
    check_exact_bound(f"logits {tag}", logits[own], ref["logits"], ref["logits_tol"], report)
    kl = ref["kl"]
    assert out4[2].item() == kl["n_kd"] and out4[3].item() == kl["n_ce"], (tag, out4.tolist(), kl["n_kd"], kl["n_ce"])
    for name, got in (("align", r["align"]), ("ce", r["ce"])):        # check_out4's bound; 0/0 gives NaN on both sides
        want = torch.tensor(kl[name], dtype=torch.float64)
        check_exact_bound(f"{name} {tag}", got, want, 2e-5 * want.abs() + 1e-6, report)
    a64, c64 = r["align"].double(), r["ce"].double()
    want = w_kd * a64 + (w_ce * c64 if w_ce != 0.0 else 0.0)
    check_exact_bound(f"total {tag}", r["total"], want, 2.0 ** -23 * (abs(w_kd) * a64.abs() + abs(w_ce) * c64.abs()), report)
    d_full = torch.zeros(N, vocab, dtype=bf16, device=DEV)
    d_full[act] = dl[own, :vocab]
    check_dlogits(d_full, kl, msg=f"d logits {tag}")
    del d_full
    if Vs > vocab:
        assert int(dl[:stored, vocab:].ne(0).sum()) == 0, f"{tag}: d logits columns vocab and above are not zero"
    if rows is not None:
        assert int(dl[count:stored].view(torch.int16).ne(0).sum()) == 0, f"{tag}: d logits rows [count, round_up(count, 128)) are not +0"
    else:
        inactive = torch.ones(N, dtype=torch.bool, device=DEV)
        inactive[act] = False
        assert int(dl[inactive].ne(0).sum()) == 0, f"{tag}: d logits of an inactive row are not zero"
    tol = ref["dh_tol"]
    if split > 1:
        tol = tol + (1 + BF16_U) * abs(g) * accumulation_extra(ref["dh"][act] / g, split, K=Vs)
    check_exact_bound(f"d hidden {tag}", hidden.grad.reshape(N, H), ref["dh"], tol, report)
    check_exact_bound(f"lm_head grad {tag}", view, ref["dW"], ref["dW_tol"], report)
    if count == 0:
        assert torch.equal(view.view(torch.int16), old.view(torch.int16)), f"{tag}: no active row, but the lm_head gradient changed"
    del ref


def distill_case(monkeypatch, tag, B, T, H, Vs, vocab, labels_fn, compact, w_ce, distill_all, split, ld_t=None, w_kd=1.0, seed=0):
    """Three micro-batches of one configuration, run twice."""
    k = K()
    calls = record_dgrad(monkeypatch)
    N = B * T
    W = randn(Vs, H, seed=seed, scale=3.0 / math.sqrt(H))
    ld_t = ld_t or vocab

    def run(report):
        arena = Arena([(Vs, H)], seed=seed + 1, scale=1e-6)
        (view,) = arena.views
        outs = []
        for mb in range(MICRO_BATCHES):
            g = f32(G_MB[mb])
            s = seed + 10 * mb
            hidden = randn(B, T, H, seed=s + 2).requires_grad_(True)
            lab = labels_fn(mb).to(DEV)
            n_t = round_up(N, 256) if compact else N
            old = arena.snapshot()[0]
            r = run_head(k, hidden, W, lab, vocab, w_kd, w_ce, distill_all, view, compact,
                         lambda count: teacher_logits(n_t, count, vocab, ld_t, s + 3), g)
            t = f"{tag} mb={mb} g={g:.4g}"
            arena.check_sentinels(t)
            dh = hidden.grad.reshape(N, H)
            no_nan(t, dh=dh, view=view)
            cap, used = calls[-1]
            assert (used > 1) == split, f"{t}: mm_nn split_k {used}, the case expects {'a split' if split else 'no split'}"
            m_kd, m_ce, _ = kl_row_masks(lab.reshape(-1), T, distill_all)
            assert int(dh[~(m_kd | m_ce)].ne(0).sum()) == 0, f"{t}: d hidden of a row that is not active is not zero"
            if compact:
                assert int(cap[r["count"]:].ne(0).sum()) == 0, f"{t}: the compact dgrad wrote rows past count"
            if report is not None:
                check_stages(k, r, hidden, W, lab, vocab, w_kd, w_ce, distill_all, g, old, view, used, report, t)
            outs += [r["total"].clone(), r["align"].clone(), r["ce"].clone()] + ([] if split else [dh.clone()])
        return outs + [arena.buf.clone()]

    twice(tag, run, label="DISTILL")


# ---------------------------------------------------------------------------------------------------------------------
# the Function at the vocabulary and shapes of the bench and its models
# ---------------------------------------------------------------------------------------------------------------------
# (id, B, T, H, compact, labels, split): config 2 (885 of 2048 rows; 16 x 4 = 64 output tiles of the dgrad: split), the 1.8B student
# (4096 rows x H 2048: 256 tiles, no split) compact and dense, Qwen2-0.5B's H 896 dense (6 x 4 tiles: split)
FULL_CASES = [("cfg2_compact", 1, 2048, 1024, True, "bench", True),
              ("1p8b_compact", 1, 4096, 2048, True, "runs", False),
              ("1p8b_dense", 1, 4096, 2048, False, "runs", False),
              ("h896_dense", 2, 333, 896, False, "runs", True)]


def test_full_cases_cover_both_dgrad_paths():
    assert {c[-1] for c in FULL_CASES} == {True, False}


@pytest.mark.parametrize("case", FULL_CASES, ids=[c[0] for c in FULL_CASES])
def test_full_vocab(case, monkeypatch):
    tag, B, T, H, compact, kind, split = case

    def labels(mb):
        if kind == "bench":
            lab = bench_labels(T, V_QWEN, seed=mb)
            m_kd, m_ce, _ = kl_row_masks(lab.reshape(-1), T)
            assert int((m_kd | m_ce).sum()) == 885
            return lab
        return run_labels(B, T, V_QWEN, seed=100 + mb)

    distill_case(monkeypatch, tag, B, T, H, V_QWEN, V_QWEN, labels, compact, 1.0, False, split, seed=H + T)


# ---------------------------------------------------------------------------------------------------------------------
# row-extent edges of the compact path, at a small vocabulary (N = 4136 < 16384: no split)
# ---------------------------------------------------------------------------------------------------------------------
H_SMALL = 512
# (B, T, count or None for distill_all, w_ce): buffer rows 333 and 778 (not multiples of 256)
EDGES = [(3, 111, c, c % 2) for c in (0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257)] + \
        [(3, 111, 333, 1), (3, 111, None, 1), (3, 111, None, 0), (2, 389, None, 0), (2, 389, 389, 0)]


@pytest.mark.parametrize("edge", EDGES, ids=[f"N{b * t}_{'all' if c is None else c}_ce{w}" for b, t, c, w in EDGES])
def test_extent_edges(edge, monkeypatch):
    B, T, count, w_ce = edge
    distill_all = count is None

    def labels(mb):
        if distill_all:
            return run_labels(B, T, V_SMALL, seed=200 + mb)
        if count == B * T:
            return torch.randint(0, V_SMALL, (B, T), generator=torch.Generator().manual_seed(mb))
        return count_labels(B, T, V_SMALL, count, seed=1000 * mb)

    distill_case(monkeypatch, f"N={B * T} count={'all' if count is None else count} distill_all={distill_all} w_ce={w_ce}", B, T, H_SMALL,
                 V_SMALL, V_SMALL, labels, True, float(w_ce), distill_all, False, seed=B * T + (count or 0))


# ---------------------------------------------------------------------------------------------------------------------
# a student vocabulary wider than the KD slice
# ---------------------------------------------------------------------------------------------------------------------
VS_WIDE, LD_T = 4224, 4352


@pytest.mark.parametrize("compact", [True, False], ids=["compact", "dense"])
def test_vocab_slice(compact, monkeypatch):
    """Student V_s 4224 over the KD vocabulary 4136, teacher logits with row stride 4352, w_ce 0: columns vocab and above add nothing to
    d hidden or the lm_head gradient (its rows vocab and above stay as they were, bit for bit)."""
    B, T = 3, 111
    distill_case(monkeypatch, f"V_s={VS_WIDE} vocab={V_SMALL} {'compact' if compact else 'dense'}", B, T, H_SMALL, VS_WIDE, V_SMALL,
                 lambda mb: run_labels(B, T, V_SMALL, seed=300 + mb), compact, 0.0, False, False, ld_t=LD_T, w_kd=0.75, seed=7)


def test_vocab_slice_refuses_ce():
    from llavamod import _C
    k = K()
    B, T = 3, 111
    W = randn(VS_WIDE, H_SMALL, seed=1)
    lab = run_labels(B, T, V_SMALL, seed=1).to(DEV)
    with pytest.raises(_C.LmodError, match="fused CE needs"):
        k.distill_head(randn(B, T, H_SMALL, seed=2), W, teacher_logits(B * T, B * T, V_SMALL, LD_T, 3), lab, V_SMALL, 1.0, 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# the upstream scalar g
# ---------------------------------------------------------------------------------------------------------------------
BIAS_LIMIT = 2.0 ** -12


@pytest.mark.parametrize("shape", ["cfg2_compact", "small_dense"])
def test_upstream_scale(shape, monkeypatch):
    """One micro-batch at g = 1, 0.5, 1/3 and 0.37 into a zero lm_head gradient view.  At g = 1 both gradients are the unscaled GEMMs' bits
    (d hidden: the mm_nn result scattered; the view: mm_tn_acc of the saved d logits and hidden rows); at g = 0.5 d hidden is exactly half
    of the same run's unscaled dgrad.  At g = 1/3 and 0.37, against g times the unscaled result (the dgrad of the same run, the view of the
    g = 1 run), the mean signed relative error over the elements must stay below 2^-12 for both gradients: rounding g itself to bf16
    scales every element by bf16(g) / g, about 2^-9 away from 1, which a per-element bound of 2^-8 does not see."""
    k = K()
    calls = record_dgrad(monkeypatch)
    if shape == "cfg2_compact":
        B, T, H, V, compact = 1, 2048, 1024, V_QWEN, True
        lab = bench_labels(T, V, seed=5).to(DEV)
    else:
        B, T, H, V, compact = 3, 111, H_SMALL, V_SMALL, False
        lab = run_labels(B, T, V, seed=5).to(DEV)
    N = B * T
    W = randn(V, H, seed=11, scale=3.0 / math.sqrt(H))
    h0 = randn(B, T, H, seed=12)
    n_t = round_up(N, 256) if compact else N
    res = {}
    for g in (1.0, 0.5, 1.0 / 3.0, 0.37):
        arena = Arena([(V, H)], seed=13)
        (view,) = arena.views
        view.zero_()
        hidden = h0.clone().requires_grad_(True)
        r = run_head(k, hidden, W, lab, V, 1.0, 1.0, False, view, compact, lambda count: teacher_logits(n_t, count, V, V, 14), f32(g))
        arena.check_sentinels(f"g={g}")
        cap = calls[-1][0]
        if compact:
            unscaled = torch.zeros(N, H, dtype=bf16, device=DEV)
            unscaled[r["rows"][0][:r["count"]].long()] = cap[:r["count"]]
        else:
            unscaled = cap
        res[g] = dict(dh=hidden.grad.reshape(N, H).clone(), view=view.clone(), unscaled=unscaled, r=r)
    one, half = res[1.0], res[0.5]
    assert torch.equal(one["dh"].view(torch.int16), one["unscaled"].view(torch.int16)), "g = 1: d hidden is not the unscaled dgrad"
    h2 = h0.reshape(N, H)
    r1 = one["r"]
    zero = torch.zeros_like(one["view"])
    if compact:
        k.mm_tn_acc(r1["dl"], k.gather_rows(h2, *r1["rows"]), zero, k_dev=r1["rows"][1])
    else:
        k.mm_tn_acc(r1["dl"], h2, zero)
    assert torch.equal(one["view"].view(torch.int16), zero.view(torch.int16)), "g = 1: the lm_head gradient is not the unscaled wgrad"
    assert torch.equal(half["dh"].double(), 0.5 * half["unscaled"].double()), "g = 0.5: d hidden is not half the unscaled dgrad"
    if not compact:                                                    # no split-K: the dgrad has the same bits in every run
        assert torch.equal(half["dh"].double(), 0.5 * one["dh"].double()), "g = 0.5: d hidden is not half of d hidden at g = 1"
    for g in (1.0 / 3.0, 0.37):
        gv = f32(g)
        for name, got, ref in (("d hidden", res[g]["dh"], gv * res[g]["unscaled"].double()),
                               ("lm_head grad", res[g]["view"], gv * one["view"].double())):
            floor = ref.pow(2).mean().sqrt() / 8
            sel = ref.abs() > floor
            rel = (got.double()[sel] - ref[sel]) / ref[sel]
            mean = float(rel.mean())
            print(f"\nDISTILL upstream scale {shape} g={gv:.6g} {name}: mean signed relative error {mean:.3g} over {int(sel.sum())} elements "
                  f"(limit {BIAS_LIMIT:.3g})")
            assert int(sel.sum()) > 10000
            assert abs(mean) < BIAS_LIMIT, f"g={gv}: {name} is scaled with a bias, mean relative error {mean:.3g}"


# ---------------------------------------------------------------------------------------------------------------------
# config 2's tied embedding: the lm_head gradient view is SpliceFn's embedding-gradient view
# ---------------------------------------------------------------------------------------------------------------------
def test_tied_embedding(monkeypatch):
    """The token embedding and the lm_head are one weight [151936, 1024] with one gradient view.  The spliced embeddings go straight into
    the loss head, so autograd runs DistillHeadFn.backward (head wgrad into the view) and then SpliceFn.backward (embedding gradient of the
    head's d hidden into the same view).  The view is checked after each: the head wgrad against the old value, then
    embed_grad_reference_fp64 against the value the head wgrad left."""
    from llavamod.model.llava_arch import IMAGE_TOKEN_INDEX, embed_grad_order, splice_plan
    k = K()
    calls = record_dgrad(monkeypatch)
    H, V, Tt = 1024, V_QWEN, 1473
    gen = torch.Generator().manual_seed(21)
    ids = torch.randint(0, V, (1, Tt), generator=gen)
    ids[0, :40] = torch.randint(0, 16, (40,), generator=gen)           # a template prefix: repeated tokens
    ids[0, 35] = IMAGE_TOKEN_INDEX
    src, _, _, _, img = splice_plan(ids.numpy(), None, None, PATCHES)
    T = src.shape[1]
    assert T == 2048
    src_d, img_d = torch.from_numpy(src).to(DEV), torch.from_numpy(img).to(DEV)
    order = torch.from_numpy(embed_grad_order(src)).to(DEV)
    sigma = (3.0 / math.sqrt(H)) ** 0.5                                # embedding rows as hidden rows: logits of std 3
    emb = randn(V, H, seed=22, scale=sigma)
    feats = randn(1, PATCHES, H, seed=23, scale=sigma).requires_grad_(True)
    lab = bench_labels(T, V, seed=24).to(DEV)
    g = f32(0.37)
    arena = Arena([(V, H)], seed=25, scale=1e-6)
    (view,) = arena.views
    old = view.clone()
    mid = {}
    with poisoned_uninitialised_memory():
        x = k.splice_embed(feats, emb, src_d, img_d, PATCHES, embed_grad=view, order=order)
        rows = k.active_rows(lab.reshape(-1), T)
        count = int(rows[1])
        t = teacher_logits(round_up(T, 256), count, V, V, 26)
        total, align, ce = k.distill_head(x, emb, t, lab, V, 1.0, 1.0, False, head_grad=view, rows=rows)
        dl = total.grad_fn.saved_tensors[0]
        splice = total.grad_fn.next_functions[0][0]
        assert type(splice).__name__.startswith("SpliceFn"), type(splice).__name__
        splice.register_prehook(lambda gr: mid.update(view=view.clone(), d=gr[0].clone()))
        total.backward(torch.tensor(g, dtype=torch.float32, device=DEV))
    torch.cuda.synchronize()
    arena.check_sentinels("tied embedding")
    assert calls[-1][1] > 1                                            # config 2's split-K dgrad
    report = {}
    x2 = x.detach().reshape(T, H)
    ref = distill_head_reference_fp64(x2, emb, t, lab.reshape(-1), T, V, 1.0, 1.0, False, g, rows=rows, dlogits=dl, old=old,
                                      store=torch.float32)
    act = ref["act"]
    tol = ref["dh_tol"] + (1 + BF16_U) * g * accumulation_extra(ref["dh"][act] / g, calls[-1][1], K=V)
    check_exact_bound("d hidden into SpliceFn", mid["d"].reshape(T, H), ref["dh"], tol, report)
    check_exact_bound("view after the head wgrad", mid["view"], ref["dW"], ref["dW_tol"], report)
    del ref
    er = embed_grad_reference_fp64(mid["d"], src_d, mid["view"])
    check_exact_bound("view after the embedding gradient", view[er["toks"]], er["want"], er["tol"], report)
    untouched = torch.ones(V, dtype=torch.bool, device=DEV)
    untouched[er["toks"]] = False
    assert torch.equal(view[untouched].view(torch.int16), mid["view"][untouched].view(torch.int16))
    assert int(er["counts"].max()) >= 2
    worst = max(report, key=report.get)
    print(f"\nDISTILL tied embedding: worst err/bound {report[worst]:.3g} ({worst}; {len(report)} checks)")
