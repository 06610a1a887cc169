"""CPU pins of the float64 references of csrc/logp.cu (tests/helpers.py): logp_reference_fp64 agrees with float64 autograd of
R.dpo_get_logp (sum and average), softmax_rows_reference_fp64 with R.get_logp / R.get_p, align_dense_reference_fp64 with
R.compute_align_loss, on rows with -inf logits too; and the bounds catch the defects a subtly wrong kernel would have -- each planted
defect below must fail its check while the unperturbed fp32 computation passes."""
import pytest
import torch

from oracle import restated as R
from tests.helpers import (IGNORE_INDEX, align_dense_reference_fp64, check_exact_bound, logp_reference_fp64,
                           softmax_rows_reference_fp64)

bf16, f64 = torch.bfloat16, torch.float64
NINF = float("-inf")
B, T, V = 4, 12, 100          # V % 8 = 4: a scalar tail after twelve 16-byte vectors


def fails(fn):
    with pytest.raises(AssertionError):
        fn()


def setup(seed=0):
    """[B*T, V] bf16 logits (randn * 3) with -inf entries, flat labels, g_seq.  Sequence 3 is wholly ignored; sequence 2 holds a row whose
    label column is -inf (its seq is -inf).  No masked row has a -inf at column 0 (see logp_reference_fp64)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * T, V, generator=g) * 3
    labels = torch.randint(0, V, (B * T,), generator=g)
    labels[[0, 1, 5, 6, 13, 20]] = IGNORE_INDEX
    labels[3 * T:] = IGNORE_INDEX
    labels[[2, 3, 4, 7, 8, 9, 10, 11]] = torch.tensor([0, V - 1, 95, 96, 7, 8, 50, 51])    # labels at the vector and tail edges
    labels[T] = 17                                            # first label of sequence 1 (what an unmasked last position of 0 reads)
    x[2, 5] = NINF                                            # one -inf
    x[3, 8:16] = NINF                                         # an aligned 16-byte vector of -inf
    x[8, 0:8] = NINF
    x[14] = NINF                                              # all -inf but the label and one other column
    x[14, int(labels[15])] = 2.0
    x[14, (int(labels[15]) + 33) % V] = -1.0
    x[2 * T + 4, int(labels[2 * T + 5])] = NINF              # the label itself at -inf
    g_seq = torch.tensor([1.75, -0.625, 0.0, -3.0], dtype=f64)
    return x.to(bf16), labels, g_seq


def test_logp_reference_matches_dpo_get_logp_and_its_autograd():
    x, labels, g_seq = setup()
    ref = logp_reference_fp64(x, labels, T, V, g_seq)
    lab2 = labels.view(B, T)
    x64 = x.to(f64).view(B, T, V).requires_grad_(True)
    seq = R.dpo_get_logp(x64, lab2)
    avg = R.dpo_get_logp(x64.detach(), lab2, average_log_prob=True)
    assert torch.isneginf(seq[2]) and torch.isneginf(ref["seq"][2]) and torch.isnan(avg[3]) and torch.isnan(ref["avg"][3])
    for got, want in ((ref["seq"], seq.detach()), (ref["avg"], avg)):
        same = (got == want) | (torch.isnan(got) & torch.isnan(want))
        assert bool((same | ((got - want).abs() <= 1e-12 * want.abs())).all()), (got, want)
    (seq * g_seq).sum().backward()
    assert torch.allclose(ref["g"], x64.grad.view(B * T, V), rtol=1e-12, atol=1e-15)
    # per row: lse and tok of the next label, 0 on masked rows and at the last position of every sequence
    act = ref["active"]
    assert not bool(act[T - 1::T].any()) and int(act.sum()) == int(ref["n"].sum())
    xa = x.to(f64)[act]
    lse = torch.logsumexp(xa, -1)
    assert torch.allclose(ref["lse"][act], lse, rtol=1e-14) and bool((ref["lse"][~act] == 0).all())
    assert bool((ref["tok"][~act] == 0).all()) and bool((ref["g"][~act] == 0).all())
    # the gradient bound's scale is |g| (q + onehot): at the label column it is |g| (1 + q)
    r = int(torch.nonzero(act)[5])
    b, c = r // T, int(ref["nxt"][r])
    q = float(torch.softmax(x[r].to(f64), -1)[c])
    assert abs(float(ref["gscale"][r, c]) - abs(float(g_seq[b])) * (1 + q)) <= 1e-15


def test_softmax_rows_reference_matches_get_logp_and_get_p():
    x, _, _ = setup(1)
    ld = torch.full((x.shape[0], V + 12), float("nan"), dtype=bf16)
    ld[:, :V] = x
    lp, lp_tol = softmax_rows_reference_fp64(ld, V, True)
    p, p_tol = softmax_rows_reference_fp64(ld, V, False)
    # the oracle computes in fp32 (dtype=torch.float32): within the bounds, -inf exactly where the reference has it
    want_lp = R.get_logp(x[None], kd_vocab=V)[0]
    want_p = R.get_p(x[None], kd_vocab=V)[0]
    assert bool(torch.isneginf(lp).eq(torch.isneginf(want_lp)).all()) and int(torch.isneginf(lp).sum()) > 0
    assert torch.allclose(lp, torch.log_softmax(x.to(f64), -1), rtol=1e-13, atol=1e-13)
    check_exact_bound("get_logp", want_lp, lp, lp_tol)
    check_exact_bound("get_p", want_p, p, p_tol)
    # a lse over V - 1 columns is out of bound
    x32 = x.float()
    short = x32 - torch.logsumexp(x32[:, :V - 1], -1, keepdim=True)
    fails(lambda: check_exact_bound("log_softmax, tail column dropped", short, lp, lp_tol))
    fails(lambda: check_exact_bound("softmax, tail column dropped", short.exp(), p, p_tol))


@pytest.mark.parametrize("distill_all", [False, True])
def test_align_dense_reference_matches_compute_align_loss(distill_all):
    x, labels, _ = setup(2)
    logp = torch.log_softmax(x.float(), -1)
    probs = torch.softmax((x.float() * 0.5 + 1).to(bf16).float(), -1)
    assert int(torch.isinf(logp).sum()) > 0
    ref = align_dense_reference_fp64(logp, probs, labels, distill_all)
    want = R.compute_align_loss(logp.to(f64)[None], probs.to(f64)[None], labels[None], distill_all)
    assert abs(float(ref["loss"]) - float(want)) <= 1e-14 * abs(float(want))
    # all rows masked: 0/0, as the reference
    none = align_dense_reference_fp64(logp, probs, torch.full_like(labels, IGNORE_INDEX))
    assert torch.isnan(none["loss"]) and torch.isnan(R.compute_align_loss(logp.to(f64)[None], probs.to(f64)[None],
                                                                          torch.full_like(labels, IGNORE_INDEX)[None]))
    # the fp32 sums pass; a -inf term kept as 0 * ... (NaN), a row counted that the mask drops, do not
    fin = torch.isfinite(logp)
    row32 = torch.where(fin, probs * torch.where(fin, logp, torch.zeros_like(logp)), torch.zeros_like(logp)).sum(-1)
    check_exact_bound("row_x fp32", row32, ref["row_x"], ref["row_x_tol"])
    m = torch.ones_like(row32) if distill_all else (labels != IGNORE_INDEX).float()
    check_exact_bound("loss fp32", -(row32 * m).sum() / m.sum(), ref["loss"], ref["loss_tol"])
    fails(lambda: check_exact_bound("row_x, -inf kept", (probs * logp).sum(-1), ref["row_x"], ref["row_x_tol"]))
    if not distill_all:
        fails(lambda: check_exact_bound("loss, every row counted", -row32.mean(), ref["loss"], ref["loss_tol"]))


def emulate(x, labels, g_seq, defect=None):
    """The kernels' arithmetic as fp32 torch ops (lse, tok = x[next label] - lse, the masked sum, d = bf16(-g q + g onehot), zeros on
    masked rows) with one planted defect."""
    N = x.shape[0]
    xf = x[:, :V].float()
    nxt = torch.full_like(labels, IGNORE_INDEX)
    nxt[:-1] = labels[1:]
    if defect == "unshifted label":
        nxt = labels.clone()
    if defect != "last position not masked":
        nxt[torch.arange(N) % T == T - 1] = IGNORE_INDEX
    act = nxt != IGNORE_INDEX
    cols = {"tail column dropped": xf[:, :V - 1], "vector-edge column dropped": torch.cat([xf[:, :7], xf[:, 8:]], 1)}.get(defect, xf)
    lse = torch.logsumexp(cols, -1)
    r_act = torch.nonzero(act)[:, 0]
    if defect == "lse off by 1e-4 on one row":
        lse[r_act[3]] += 1e-4
    lab = torch.where(act, nxt, torch.zeros_like(nxt))
    tok = torch.where(act, xf.gather(1, lab[:, None])[:, 0] - lse, torch.zeros_like(lse))
    keep = act.clone()
    if defect == "seq drops one token":
        keep[r_act[2]] = False
    seq = (torch.where(keep, tok, torch.zeros_like(tok))).view(B, T).sum(-1)
    g = g_seq.float().roll(1) if defect == "g_seq of the neighbouring sequence" else g_seq.float()
    gr = g.repeat_interleave(T)[:, None]
    q = torch.exp(xf - lse[:, None])
    oh = torch.zeros_like(q) if defect == "no one-hot term" else torch.zeros_like(q).scatter_(1, lab[:, None], 1.0)
    d = gr * (oh - q)
    dmask = act.clone()
    if defect == "masked row with a gradient":
        dmask[int(torch.nonzero(~act)[0])] = True
    d = torch.where(dmask[:, None], d, torch.zeros_like(d))
    return dict(lse=torch.where(act, lse, torch.zeros_like(lse)), tok=tok, seq=seq, d=d.to(bf16))


def check_all(out, ref):
    check_exact_bound("lse", out["lse"], ref["lse"], ref["lse_tol"])
    check_exact_bound("tok", out["tok"], ref["tok"], ref["tok_tol"])
    check_exact_bound("seq", out["seq"], ref["seq"], ref["seq_tol"])
    check_exact_bound("d", out["d"], ref["g"], ref["g_tol"])


DEFECTS = ["unshifted label", "last position not masked", "tail column dropped", "vector-edge column dropped", "no one-hot term",
           "masked row with a gradient", "g_seq of the neighbouring sequence", "lse off by 1e-4 on one row", "seq drops one token"]


@pytest.mark.parametrize("defect", DEFECTS)
def test_logp_bounds_catch_planted_defects(defect):
    x, labels, _ = setup(3)
    x = torch.where(torch.isinf(x.float()), torch.zeros_like(x), x)     # finite rows: every sequence sum is a finite number here
    g_seq = torch.tensor([1.75, -0.625, 0.3, -3.0], dtype=f64)
    ref = logp_reference_fp64(x, labels, T, V, g_seq)
    check_all(emulate(x, labels, g_seq), ref)
    fails(lambda: check_all(emulate(x, labels, g_seq, defect), ref))


def test_check_exact_bound_matches_infinities_and_the_nan_average_only_exactly():
    want = torch.tensor([NINF, float("nan"), 1.0], dtype=f64)
    tol = torch.tensor([float("inf"), 1.0, 0.5], dtype=f64)
    assert check_exact_bound("ok", torch.tensor([NINF, float("nan"), 1.25]), want, tol) == 0.5
    fails(lambda: check_exact_bound("finite for -inf", torch.tensor([-1e30, float("nan"), 1.0]), want, tol))
    fails(lambda: check_exact_bound("number for NaN", torch.tensor([NINF, 0.0, 1.0]), want, tol))
    fails(lambda: check_exact_bound("NaN for a number", torch.tensor([NINF, float("nan"), float("nan")]), want, tol))
