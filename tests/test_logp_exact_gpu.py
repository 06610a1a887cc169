"""The log-prob gather and softmax-row kernels (csrc/logp.cu) element by element against the float64 references of tests/helpers.py, at
the vocabulary, stride, label and mask edges where they go wrong, and as the trainers call them.

lmod_logp_gather_fwd / _bwd give the DPO step's sequence log-probs and their gradient (kernels.LogpHeadFn, d logits written in place
over the saved logits), the frozen reference's log-probs and the SFT loss (ShiftedCEFn); lmod_softmax_rows and lmod_align_loss_dense are
AlignTrainer.get_logp / get_p / compute_align_loss.  Every case checks each output against its bound (logp_reference_fp64,
softmax_rows_reference_fp64, align_dense_reference_fp64; the derivations are next to them), that a second launch gives the same bytes,
and that nothing outside [0, V) of a row is read (the input's pad columns hold NaN) or written (the output's pad columns hold a sentinel).
Rows with -inf logits must give the same finite answer as torch.  Each case prints its worst err / bound."""
import json
import math
import os

import pytest
import torch

from tests.helpers import (IGNORE_INDEX, _gemm_tol, align_dense_reference_fp64, check_exact_bound, logp_reference_fp64,
                           softmax_rows_reference_fp64)

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
NAN, NINF = float("nan"), float("-inf")
SENT = 12345.0                                     # bf16 12352; fp32 exact
V_QWEN, V_WIDE = 151936, 152064
VOCABS = [1, 7, 8, 9, 2047, 2048, 2049, 8191, 8192, 8193, 8200, V_QWEN, V_WIDE]
REPORT = {}


def _k():
    from llavamod import kernels as K
    return K


def _pad8(n):
    return (n + 7) // 8 * 8


def same_bits(a, b):
    iv = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


def padded(x, ld, fill=NAN, dtype=BF16):
    """[N, ld] buffer holding x in its first V columns and `fill` in the pad columns."""
    buf = torch.full((x.shape[0], ld), fill, dtype=dtype, device="cuda")
    buf[:, :x.shape[1]] = x.to(dtype)
    return buf


def gather_fwd(x, ld, labels, B, T, V, average=False):
    K = _k()
    tok = torch.empty(B * T, dtype=F32, device="cuda")
    lse = torch.empty(B * T, dtype=F32, device="cuda")
    seq = torch.empty(B, dtype=F32, device="cuda")
    K.call("lmod_logp_gather_fwd", K.ptr(x), ld, K.ptr(labels), B, T, V, K.ptr(tok), K.ptr(lse), K.ptr(seq), 1 if average else 0)
    torch.cuda.synchronize()
    return seq, tok, lse


def gather_bwd(x, ld, labels, B, T, V, lse, g32, d, ld_d):
    K = _k()
    K.call("lmod_logp_gather_bwd", K.ptr(x), ld, K.ptr(labels), B, T, V, K.ptr(lse), K.ptr(g32), 0, K.ptr(d), ld_d)
    torch.cuda.synchronize()


def label_edges(V):
    """0, V - 1, the last vectorised column and the first tail column, and the thread-stride edge 2047 / 2048 (those inside [0, V))."""
    nvec = V // 8
    return sorted({c for c in (0, V - 1, 8 * nvec - 1, 8 * nvec, 2047, 2048) if 0 <= c < V})


def mask_runs(labels, B, T):
    """Ignored runs in every sequence: its first two labels and, when T > 10, positions 5-6; the last of B >= 4 sequences is wholly
    ignored."""
    lab = labels.view(B, T)
    lab[:, :2] = IGNORE_INDEX
    if T > 10:
        lab[:, 5:7] = IGNORE_INDEX
    if B >= 4:
        lab[-1] = IGNORE_INDEX
    return labels


KINDS = ["typical", "constant", "peaked", "large", "ninf_one", "ninf_vec0", "ninf_veck", "ninf_most"]


def plant_row(x, r, V, kind, c, gen):
    """Make row r of x [N, V] (fp32) the given kind around label column c; returns the label (some kinds move it off their -inf run)."""
    dev = x.device
    if kind == "constant":
        x[r] = 1.5                                                     # lse = 1.5 + ln V
    elif kind == "peaked":
        x[r] = torch.randn(V, device=dev, generator=gen)
        x[r, c] = float(x[r].max()) + 30                              # q ~ 1: the label column is g (1 - q)
    elif kind == "large":
        x[r] = torch.rand(V, device=dev, generator=gen) * 200 - 100
    elif kind == "ninf_one" and V >= 2:                               # one -inf in the first 256 columns
        j = (7 * r + 3) % min(256, V)
        j = (j + 1) % min(256, V) if j == c else j
        if j != c:
            x[r, j] = NINF
    elif kind == "ninf_vec0" and V > 8:                               # eight aligned -inf at [0, 8): thread 0's first vector
        x[r, :8] = NINF
        c = c if c >= 8 else V - 1
    elif kind == "ninf_veck" and V >= 16:                             # eight aligned -inf at [8k, 8k + 8), k < 256
        k = min(1 + (37 * r) % 255, V // 8 - 1)
        x[r, 8 * k:8 * k + 8] = NINF
        c = c if not (8 * k <= c < 8 * k + 8) else (V - 1 if V - 1 >= 8 * k + 8 else 0)
    elif kind == "ninf_most" and V >= 2:                              # all -inf but the label and one other column
        o = (c + V // 2 + 1) % V
        o = (o + 1) % V if o == c else o
        keep = x[r, [c, o]].clone()
        x[r] = NINF
        x[r, [c, o]] = keep
    return c


def build_case(B, T, V, seed, kinds=True, label_ninf_seq=None):
    """Logits [B*T, V] fp32 (randn * 3, and the kinds above on the active rows in turn) and flat labels with ignored runs; every active
    row's next label cycles through label_edges(V), the row's argmax and its argmin.  label_ninf_seq: in that sequence one active row has
    its label column at -inf (tok and seq are -inf there)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    N = B * T
    x = torch.randn(N, V, device="cuda", generator=gen) * 3
    labels = mask_runs(torch.randint(0, V, (N,), device="cuda", generator=gen), B, T)
    lab_cpu = labels.cpu()
    edges = label_edges(V) + ["argmax", "argmin"]
    i = 0
    planted_ninf_label = False
    for r in range(N):
        if r % T == T - 1 or int(lab_cpu[r + 1]) == IGNORE_INDEX:
            continue
        kind = KINDS[i % len(KINDS)] if kinds else "typical"
        choice = edges[(i // 2) % len(edges)]
        c = choice if isinstance(choice, int) else 0
        c = plant_row(x, r, V, kind, c, gen)
        if choice == "argmax" and kind in ("typical", "large", "ninf_one"):
            c = int(x[r].argmax())
        elif choice == "argmin" and kind in ("typical", "large", "ninf_one"):
            c = int(torch.where(torch.isinf(x[r]), torch.full_like(x[r], float("inf")), x[r]).argmin())
        if label_ninf_seq is not None and r // T == label_ninf_seq and not planted_ninf_label and V >= 2 and kind == "typical":
            x[r, c] = NINF                                            # the label itself at -inf: tok = -inf, gradient g at c
            planted_ninf_label = True
        labels[r + 1] = c
        i += 1
    return x, labels


def run_gather(name, x, labels, B, T, V, g_seq, g_dtype=F64, extra=16):
    """Both gather kernels on x [B*T, V] against logp_reference_fp64: forward (sum and average forms), backward out of place (ld_d > V,
    sentinel pad) and in place over the logits (as LogpHeadFn.backward runs it), each launched twice.  Returns the reference."""
    N = B * T
    ld = _pad8(V) + extra
    xb = padded(x, ld)
    seq, tok, lse = gather_fwd(xb, ld, labels, B, T, V)
    seq2, tok2, lse2 = gather_fwd(xb, ld, labels, B, T, V)
    assert same_bits(seq, seq2) and same_bits(tok, tok2) and same_bits(lse, lse2), f"{name}: forward bytes differ between launches"
    avg, tok_a, lse_a = gather_fwd(xb, ld, labels, B, T, V, average=True)
    assert same_bits(tok_a, tok) and same_bits(lse_a, lse), f"{name}: the average form changed tok / lse"
    ref = logp_reference_fp64(xb, labels, T, V, g_seq, g_dtype=g_dtype)
    w = {}
    w["lse"] = check_exact_bound(f"{name} lse", lse, ref["lse"], ref["lse_tol"], REPORT)
    w["tok"] = check_exact_bound(f"{name} tok", tok, ref["tok"], ref["tok_tol"], REPORT)
    w["seq"] = check_exact_bound(f"{name} seq", seq, ref["seq"], ref["seq_tol"], REPORT)
    w["avg"] = check_exact_bound(f"{name} avg", avg, ref["avg"], ref["avg_tol"], REPORT)
    act = ref["active"]
    assert bool((tok[~act] == 0).all()) and bool((lse[~act] == 0).all()), f"{name}: masked row with a nonzero tok / lse"
    # backward, out of place, d with a wider row stride than the logits
    g32 = g_seq.to("cuda", F32).contiguous()
    assert torch.equal(g32.double(), g_seq.to("cuda", F64)), "g_seq must be exact in fp32"
    ld_d = ld + 8
    d = padded(torch.zeros(N, 0, device="cuda"), ld_d, SENT)
    gather_bwd(xb, ld, labels, B, T, V, lse, g32, d, ld_d)
    d2 = padded(torch.zeros(N, 0, device="cuda"), ld_d, SENT)
    gather_bwd(xb, ld, labels, B, T, V, lse, g32, d2, ld_d)
    assert same_bits(d, d2), f"{name}: d logits bytes differ between launches"
    assert bool((d[:, V:] == torch.tensor(SENT, dtype=BF16, device="cuda")).all()), f"{name}: a pad column of d was written"
    w["d"] = check_exact_bound(f"{name} d", d[:, :V], ref["g"], ref["g_tol"], REPORT)
    assert int(d[~act, :V].contiguous().view(torch.int16).ne(0).sum()) == 0, f"{name}: masked row / last position of d is not +0"
    # in place over the logits (ld_d = ld): the same bytes, the pad columns untouched
    xc = xb.clone()
    gather_bwd(xc, ld, labels, B, T, V, lse, g32, xc, ld)
    assert same_bits(xc[:, :V], d[:, :V]), f"{name}: in-place d differs from out-of-place d"
    assert same_bits(xc[:, V:], xb[:, V:]), f"{name}: in-place backward wrote a pad column"
    print(f"\nLOGPEXACT {name}: worst err/bound " + " ".join(f"{k} {v:.3g}" for k, v in w.items()))
    return ref


@pytest.mark.parametrize("V", VOCABS)
def test_logp_gather_vocab_edges(V):
    """Four sequences of 16: g_seq of mixed sign and size, 0 on an active sequence; the last wholly ignored (seq = 0, average NaN); every
    row kind and label edge; a -inf label in sequence 2."""
    B, T = 4, 16
    x, labels = build_case(B, T, V, seed=V, label_ninf_seq=2)
    g_seq = torch.tensor([1.75, 0.0, -0.296875, -3.0], dtype=F64)
    ref = run_gather(f"V={V}", x, labels, B, T, V, g_seq)
    assert float(ref["n"][3]) == 0 and float(ref["seq"][3]) == 0 and math.isnan(float(ref["avg"][3]))
    if V >= 2:
        assert math.isinf(float(ref["seq"][2])), "the -inf label row was not planted"


@pytest.mark.parametrize("T", [1, 2])
def test_logp_gather_short_sequences(T):
    """T = 1: no position has a next label (every row masked, seq 0, average NaN); T = 2: one active row per sequence."""
    B, V = 5, 8200
    x, labels = build_case(B, T, V, seed=T, kinds=False)
    labels = torch.randint(0, V, (B * T,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    labels[T * 2:T * 2 + T] = IGNORE_INDEX
    g_seq = torch.tensor([1.5, -0.5, 2.0, -1.25, 0.75], dtype=F64)
    ref = run_gather(f"T={T}", x, labels, B, T, V, g_seq)
    assert int(ref["active"].sum()) == (0 if T == 1 else B - 1)


def test_logp_gather_at_real_length():
    """B = 2, T = 2048 at the Qwen vocabulary: 4096 rows, 1.24 GB of logits; the sequence-sum chain at its real length."""
    B, T, V = 2, 2048, V_QWEN
    gen = torch.Generator(device="cuda").manual_seed(2048)
    x = torch.randn(B * T, V, device="cuda", generator=gen) * 3
    labels = torch.randint(0, V, (B * T,), device="cuda", generator=gen)
    lab = labels.view(B, T)
    lab[:, :100] = IGNORE_INDEX                                       # a prompt
    lab[0, 700:760] = IGNORE_INDEX
    lab[1, 1500:] = IGNORE_INDEX                                      # padding
    edges = torch.tensor(label_edges(V), device="cuda")
    labels[200::97] = edges.repeat(-(-labels[200::97].numel() // edges.numel()))[:labels[200::97].numel()]
    g_seq = torch.tensor([0.8125, -1.375], dtype=F64)
    run_gather("B=2 T=2048", x.to(BF16), labels, B, T, V, g_seq, g_dtype=F32)


def test_logp_head_at_the_qwen_head_shape():
    """kernels.logp_head as the DPO step runs it (H = 896, V = 151936): the sequence log-probs, d hidden and the accumulation into a
    nonzero lm_head gradient, against float64 GEMMs of the kernel's own d logits (the GEMMs are covered by test_gemm_exact_gpu.py; this
    checks the in-place d, the strides and accumulate-not-overwrite)."""
    K = _k()
    H, V, B, T = 896, V_QWEN, 2, 333
    N = B * T
    gen = torch.Generator(device="cuda").manual_seed(896)
    hidden = torch.randn(B, T, H, device="cuda", generator=gen).to(BF16)
    W = (torch.randn(V, H, device="cuda", generator=gen) * (3 / math.sqrt(H))).to(BF16)
    labels = mask_runs(torch.randint(0, V, (N,), device="cuda", generator=gen), B, T)
    e = torch.tensor(label_edges(V) + [V // 2], device="cuda")
    labels[40:40 + e.numel()] = e
    old = (torch.randn(V, H, device="cuda", generator=gen) * 0.01).to(BF16)
    head_grad = old.clone()
    g_seq = torch.tensor([1.25, -0.75], dtype=F64)
    h = hidden.clone().requires_grad_(True)
    seq = K.logp_head(h, W, labels.view(B, T), head_grad)
    seq.backward(g_seq.to("cuda", F32))
    torch.cuda.synchronize()
    # the kernel's own logits (the GEMM LogpHeadFn.forward runs) and d logits
    logits = K.mm_nt(hidden.reshape(N, H), W)
    seq2, tok, lse = gather_fwd(logits, V, labels, B, T, V)
    assert same_bits(seq2, seq.detach()), "logp_head: seq differs from the gather on the same logits"
    ref = logp_reference_fp64(logits, labels, T, V, g_seq)
    w = {"seq": check_exact_bound("logp_head seq", seq, ref["seq"], ref["seq_tol"], REPORT),
         "tok": check_exact_bound("logp_head tok", tok, ref["tok"], ref["tok_tol"], REPORT)}
    d = torch.empty(N, V, dtype=BF16, device="cuda")
    gather_bwd(logits, V, labels, B, T, V, lse, g_seq.to("cuda", F32), d, V)
    w["d"] = check_exact_bound("logp_head d", d, ref["g"], ref["g_tol"], REPORT)
    del ref
    d64, W64, h64 = d.double(), W.double(), hidden.reshape(N, H).double()
    dh = d64 @ W64
    maj = d64.abs() @ W64.abs()
    w["dh"] = check_exact_bound("logp_head dh", h.grad.reshape(N, H), dh, _gemm_tol(dh, maj, V) + 16 * 2.0 ** -23 * maj, REPORT)
    del dh, maj
    hg = old.double() + d64.t() @ h64
    maj = old.double().abs() + d64.abs().t() @ h64.abs()
    w["head_grad"] = check_exact_bound("logp_head head_grad", head_grad, hg, _gemm_tol(hg, maj, N) + 2.0 ** -23 * hg.abs(), REPORT)
    assert float((hg - old.double()).abs().max()) > 0.1, "the accumulated gradient must be distinguishable from the old value"
    print("\nLOGPEXACT logp_head: worst err/bound " + " ".join(f"{k} {v:.3g}" for k, v in w.items()))


def test_shifted_ce_loss_and_gradient():
    """ShiftedCEFn (forward(labels=...) loss): loss = -sum(seq) / cnt and d logits with g = -1 / cnt per sequence."""
    from llavamod.model.language_model.llava_qwen_common import ShiftedCEFn
    B, T, V = 2, 300, V_QWEN
    x, labels = build_case(B, T, V, seed=300, kinds=False)
    xb = x.to(BF16).view(B, T, V)
    lab = labels.view(B, T)
    xl = xb.clone().requires_grad_(True)
    loss = ShiftedCEFn.apply(xl, lab)
    loss.backward()
    xl2 = xb.clone().requires_grad_(True)
    loss2 = ShiftedCEFn.apply(xl2, lab)
    loss2.backward()
    torch.cuda.synchronize()
    assert same_bits(loss.detach(), loss2.detach()) and same_bits(xl.grad, xl2.grad), "ShiftedCEFn: bytes differ between launches"
    cnt = int((lab[:, 1:] != IGNORE_INDEX).sum())
    ref = logp_reference_fp64(xb.view(B * T, V), labels, T, V, torch.full((B,), -1.0 / cnt, dtype=F64))
    want = -ref["seq"].sum() / cnt
    tol = (ref["seq_tol"].sum() + B * 2.0 ** -24 * ref["seq"].abs().sum()) / cnt + 2.0 ** -24 * want.abs()
    w = {"loss": check_exact_bound("ShiftedCE loss", loss.detach(), want, tol, REPORT),
         "d": check_exact_bound("ShiftedCE d", xl.grad.view(B * T, V), ref["g"], ref["g_tol"], REPORT)}
    print("\nLOGPEXACT ShiftedCE: worst err/bound " + " ".join(f"{k} {v:.3g}" for k, v in w.items()))


def softmax_inputs(N, V, seed):
    """Rows for the compat forms: randn * 3, with one -inf in the first 256 columns (and a finite value 256 columns on, in the same
    thread), an aligned run of eight -inf, a large-magnitude row and a constant row."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, V, device="cuda", generator=gen) * 3
    for r in range(N):
        kind = r % 6
        if kind == 1:
            x[r, (11 * r) % min(256, V)] = NINF
        elif kind == 2:
            k = (5 * r) % min(256, V // 8)
            x[r, 8 * k:8 * k + 8] = NINF
        elif kind == 3:
            x[r] = torch.rand(V, device="cuda", generator=gen) * 200 - 100
        elif kind == 4:
            x[r] = 1.5
        elif kind == 5:
            x[r, :V:3] = NINF
    return x


@pytest.mark.parametrize("V,ld", [(300, 304), (V_QWEN, V_WIDE)])
@pytest.mark.parametrize("log_mode", [True, False])
def test_softmax_rows(V, ld, log_mode):
    """lmod_softmax_rows (get_logp / get_p) with the row stride of the wider teacher (152064) over the Qwen vocabulary, -inf entries."""
    K = _k()
    N = 30
    xb = padded(softmax_inputs(N, V, seed=V + log_mode), ld)
    ld_out = V + 8
    outs = []
    for _ in range(2):
        out = padded(torch.zeros(N, 0, device="cuda"), ld_out, SENT, F32)
        K.call("lmod_softmax_rows", K.ptr(xb), ld, N, V, 1 if log_mode else 0, K.ptr(out), ld_out)
        torch.cuda.synchronize()
        outs.append(out)
    out = outs[0]
    assert same_bits(outs[0], outs[1]), "softmax_rows: bytes differ between launches"
    assert bool((out[:, V:] == SENT).all()), "softmax_rows: a pad column of the output was written"
    assert same_bits(K.softmax_rows(xb, V, log_mode), out[:, :V].contiguous()), "kernels.softmax_rows differs from the raw call"
    want, tol = softmax_rows_reference_fp64(xb, V, log_mode)
    name = f"softmax_rows V={V} {'log' if log_mode else 'prob'}"
    worst = check_exact_bound(name, out[:, :V], want, tol, REPORT)
    assert not bool(torch.isnan(out[:, :V]).any())
    print(f"\nLOGPEXACT {name}: worst err/bound {worst:.3g}")


@pytest.mark.parametrize("mode", ["labels", "distill_all", "all_masked"])
def test_align_loss_dense(mode):
    """lmod_align_loss_dense (compute_align_loss) on the kernels' own log-probs (with -inf entries, dropped from the sum) and probs; the
    all-masked batch gives NaN (0/0), as the reference."""
    K = _k()
    N, V = 40, V_QWEN
    s = softmax_inputs(N, V, seed=7)
    t = torch.randn(N, V, device="cuda", generator=torch.Generator(device="cuda").manual_seed(8)) * 3 + 0.5 * torch.nan_to_num(s, neginf=0)
    logp = K.softmax_rows(s.to(BF16), V, True)
    probs = K.softmax_rows(t.to(BF16), V, False)
    assert int(torch.isinf(logp).sum()) > 0 and not bool(torch.isnan(logp).any())
    labels = torch.randint(0, V, (N,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    labels[[0, 1, 5, 6, 7, 20, 33]] = IGNORE_INDEX
    if mode == "all_masked":
        labels[:] = IGNORE_INDEX
    distill_all = mode == "distill_all"
    res = []
    for _ in range(2):
        row_x = torch.full((N,), NAN, dtype=F32, device="cuda")
        out = torch.full((1,), NAN, dtype=F32, device="cuda")
        K.call("lmod_align_loss_dense", K.ptr(logp), K.ptr(probs), V, K.ptr(labels), N, V, 1 if distill_all else 0, K.ptr(row_x),
               K.ptr(out))
        torch.cuda.synchronize()
        res.append((row_x, out))
    (row_x, out), (row_x2, out2) = res
    assert same_bits(row_x, row_x2) and same_bits(out, out2), "align_loss_dense: bytes differ between launches"
    assert same_bits(K.align_loss_dense(logp, probs, labels, distill_all).reshape(1), out)
    ref = align_dense_reference_fp64(logp, probs, labels, distill_all)
    w = {"row_x": check_exact_bound(f"align_loss_dense {mode} row_x", row_x, ref["row_x"], ref["row_x_tol"], REPORT),
         "loss": check_exact_bound(f"align_loss_dense {mode} loss", out[0], ref["loss"], ref["loss_tol"], REPORT)}
    if mode == "all_masked":
        assert math.isnan(float(out[0]))
    print(f"\nLOGPEXACT align_loss_dense {mode}: worst err/bound " + " ".join(f"{k} {v:.3g}" for k, v in w.items()))


def teardown_module(module):
    out = os.environ.get("LLAVAMOD_TEST_REPORT")
    if out and REPORT:
        with open(out, "a") as f:
            f.write(json.dumps({"logp_err_over_bound": REPORT}) + "\n")
    print("logp err/bound:", json.dumps(REPORT))
