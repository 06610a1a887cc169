"""Shared fixtures for the GPU parity tests, smoke() and bench.py: tiny config-1 models, seeded batches, and the
oracle-side evaluation of the same step."""
import contextlib
import math
import types

import torch

from oracle import restated as R


def tiny_pair(device="cuda", student_layers=2, teacher_layers=2, vocab=512, seed=0):
    from llavamod.model import synthetic as S
    arch_s = dict(S.ARCH["tiny"], num_hidden_layers=student_layers, vocab_size=vocab)
    arch_t = dict(S.ARCH["tiny"], num_hidden_layers=teacher_layers, vocab_size=vocab, intermediate_size=320)
    teacher = S.make_teacher(arch_t, "tiny", device=device, seed=seed)
    student = S.make_student(arch_s, "tiny", device=device, seed=seed + 1, margs=S.moe_args(), share_tower_with=teacher)
    return student, teacher


def tiny_batch(student, B=2, Tt=40, seed=0, pad=(0, 0), n_img_tokens=1):
    """config-1 shape: 32x32 image -> 16 patches, text length chosen so the spliced length is 40-1+16 = 55 (odd on purpose)."""
    g = torch.Generator().manual_seed(seed)
    V = student.config.vocab_size
    ids = torch.randint(0, V, (B, Tt), generator=g)
    ids[:, 5] = -200
    mask = torch.ones(B, Tt, dtype=torch.bool)
    for b, p in enumerate(pad[:B]):
        if p:
            mask[b, Tt - p:] = False
    labels = ids.clone()
    labels[:, : int(0.4 * Tt)] = -100
    labels[~mask] = -100
    images = [torch.randn(3, 32, 32, generator=g).to(torch.bfloat16) for _ in range(B)]
    Tn = Tt - 1 + 16
    n_moe = sum(1 for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    E = 4
    noise = [R.gumbel_noise((B * Tn, E), g) for _ in range(n_moe)]
    return dict(input_ids=ids, labels=labels, attention_mask=mask, images=images), noise


def cfgs_of(model):
    c = model.config
    t = model.get_image_tower().config
    cc = R.ClipCfg(hidden=t.hidden_size, inter=t.intermediate_size, layers=t.num_hidden_layers, heads=t.num_attention_heads,
                   image=t.image_size, patch=t.patch_size, eps=t.layer_norm_eps, select_layer=c.mm_vision_select_layer)
    moe_layers = [i for i, l in enumerate(model.model.layers) if hasattr(l.mlp, "deepspeed_moe")]
    kw = {}
    if moe_layers:
        m = model.model.layers[moe_layers[0]].mlp
        kw = dict(moe_layers=moe_layers, num_experts=m.num_experts, capacity_factor=m.capacity_factor, min_capacity=m.min_capacity,
                  aux_coef=model.router_aux_loss_coef)
    lc = R.LMCfg(hidden=c.hidden_size, inter=c.intermediate_size, layers=c.num_hidden_layers, heads=c.num_attention_heads,
                 kv_heads=c.num_key_value_heads, vocab=c.vocab_size, rope_theta=c.rope_theta, eps=c.rms_norm_eps,
                 tie=bool(getattr(c, "tie_word_embeddings", False)), kd_vocab=min(R.KD_VOCAB, c.vocab_size), **kw)
    return lc, cc


def oracle_state(model, dtype=torch.float32):
    return {k: v.detach().to("cpu").to(dtype if v.dtype != torch.float32 or dtype == torch.float32 else v.dtype) for k, v in model.state_dict().items()}


def oracle_forward(model, batch, noise=None, sd=None, dtype=torch.float32):
    lc, cc = cfgs_of(model)
    sd = sd if sd is not None else oracle_state(model, dtype)
    imgs = [im.to(dtype) for im in batch["images"]]
    return R.llava_forward(sd, lc, cc, batch["input_ids"], batch["attention_mask"], batch["labels"], imgs, noise), lc


def oracle_mimic_loss(student, teacher, batch, noise, loss_type="kd_lm", moe_loss_enable=True, sd_s=None, sd_t=None):
    with torch.no_grad():
        t_out, _ = oracle_forward(teacher, batch, sd=sd_t)
    s_out, lc = oracle_forward(student, batch, noise, sd=sd_s)
    return R.mimic_compute_loss(s_out, t_out["logits"], loss_type, moe_loss_enable, False, lc.kd_vocab)


IGNORE_INDEX = -100


def kl_row_masks(labels, T, distill_all=False):
    """(m_kd, m_ce) per row of the flat [N] labels: the KD mask is the row's own label (align_trainer.py:514-517, not shifted), the CE mask
    is the NEXT position's label (shifted CE), and the last position of every sequence has no next label."""
    labels = labels.reshape(-1)
    N = labels.numel()
    nxt = torch.full_like(labels, IGNORE_INDEX)
    nxt[:-1] = labels[1:]
    nxt[torch.arange(N, device=labels.device) % T == T - 1] = IGNORE_INDEX
    m_kd = torch.ones_like(labels, dtype=torch.bool) if distill_all else labels != IGNORE_INDEX
    return m_kd, nxt != IGNORE_INDEX, nxt


def kl_reference_fp64(s, t, labels, T, V, w_kd, w_ce, distill_all=False, g_dtype=torch.float64, block_bytes=1 << 30):
    """Plain float64 restatement of the fused loss head (csrc/kl.cu): mimic-KL of R.compute_align_loss plus the shifted CE, per row and
    reduced, and the gradient the kernel writes into dlogits.

    s, t: [N, >= V] logits (the first V columns are used), labels: [N] flat, T: sequence length.  Works on the tensors' device in blocks of
    rows so that the float64 temporaries stay under about `block_bytes`.  Returns a dict:
      row    [N, 4] float64: x = sum p_T log q_S over the terms where log q_S is finite, nll = lse_S - s[next label] (0 without a next
             label), lse_S, lse_T; all four 0 on rows with neither mask (the kernel skips them)
      align  -sum(x m_kd) / sum(m_kd)   (0/0 -> NaN, align_trainer.py:526)
      ce     sum(nll m_ce) / sum(m_ce)
      n_kd, n_ce
      g      [N, V] g_dtype: ckd m_kd (q - p) + cce m_ce (q - onehot(next label)), ckd = w_kd / n_kd, cce = w_ce / n_ce
      gscale [N, V] g_dtype: ca q + cb p with ca = ckd m_kd + cce m_ce, cb = ckd m_kd -- the size of the two terms the kernel combines,
             which its error bound scales with.
    g is d(w_kd align + w_ce ce)/ds wherever the student logits are finite.  On a row with -inf student logits autograd of the masked
    product gives ckd (q sum_kept p - p [kept]); like the kernel, g keeps the form (q - p) there (the logits of a real lm_head are finite)."""
    s, t = s[:, :V], t[:, :V]
    labels = labels.reshape(-1).to(s.device)
    N = labels.numel()
    m_kd, m_ce, nxt = kl_row_masks(labels, T, distill_all)
    active = m_kd | m_ce
    n_kd, n_ce = float(m_kd.sum()), float(m_ce.sum())
    ckd = w_kd / n_kd if n_kd else 0.0
    cce = w_ce / n_ce if n_ce else 0.0
    row = torch.zeros(N, 4, dtype=torch.float64, device=s.device)
    g = torch.zeros(N, V, dtype=g_dtype, device=s.device)
    gscale = torch.zeros(N, V, dtype=g_dtype, device=s.device)
    step = max(1, block_bytes // (8 * 8 * V))                    # about eight [rows, V] float64 temporaries per block
    for r0 in range(0, N, step):
        r1 = min(N, r0 + step)
        s64, t64 = s[r0:r1].double(), t[r0:r1].double()
        lse_s, lse_t = torch.logsumexp(s64, -1), torch.logsumexp(t64, -1)
        logq = s64 - lse_s[:, None]
        q, p = logq.exp(), (t64 - lse_t[:, None]).exp()
        x = torch.where(torch.isinf(logq), torch.zeros_like(logq), p * logq).sum(-1)
        mc = m_ce[r0:r1]
        lab = torch.where(mc, nxt[r0:r1], torch.zeros_like(nxt[r0:r1]))
        nll = torch.where(mc, lse_s - s64.gather(1, lab[:, None])[:, 0], torch.zeros_like(lse_s))
        act = active[r0:r1]
        row[r0:r1] = torch.where(act[:, None], torch.stack([x, nll, lse_s, lse_t], 1), torch.zeros(1, 4, dtype=torch.float64, device=s.device))
        a = ckd * m_kd[r0:r1].double() + cce * mc.double()
        b = ckd * m_kd[r0:r1].double()
        gb = a[:, None] * q - b[:, None] * p
        gb.scatter_add_(1, lab[:, None], -cce * mc.double()[:, None])
        g[r0:r1] = gb.to(g_dtype)
        gscale[r0:r1] = (a[:, None] * q + b[:, None] * p).to(g_dtype)
        del s64, t64, logq, q, p, gb
    mk, mc = m_kd.double(), m_ce.double()
    align = -(row[:, 0] * mk).sum() / mk.sum()
    ce = (row[:, 1] * mc).sum() / mc.sum()
    return dict(row=row, align=float(align), ce=float(ce), n_kd=n_kd, n_ce=n_ce, g=g, gscale=gscale)


# Element-wise bound of the kernel's dlogits against kl_reference_fp64:  |g_k - g| <= 2^-8 |g| + KL_GRAD_EPS (ca q + cb p) + 2^-126.
#   2^-8 |g|   the bf16 store of g: 8 significant bits, so half an ulp is up to 2^-8 relative.
#   KL_GRAD_EPS bounds the relative error of each fp32 q = 2^(s*log2e - lse_S*log2e) and p (same form), which the cancellation in ca*q - cb*p
#              turns into an absolute error of up to eps*(ca q + cb p).  For |lse| < 128 and |s - lse| < 64 (every case tested):
#                lse_S itself: max + lg2(Z)*ln2 rounded to fp32 (half ulp at 64..128 = 3.8e-6) + the fp32 sum Z (~1e-6)   ~4.8e-6
#                -lse_S*log2e rounded (|.| < 256: half ulp 7.6e-6 in log2 units, x ln2)                                         5.3e-6
#                the fma s*log2e + (-lse_S*log2e) rounded (|.| < 128: 3.8e-6 x ln2)                                             2.6e-6
#                ex2.approx (2^-22.5)                                                                                           1.7e-7
#              sum 1.3e-5.  The fp32 roundings of -cb*p and of the fma ca*q + (-cb*p) add at most 2^-23 (ca q + cb p), i.e. 1.2e-7 to eps;
#              all of it rounded up to 2e-5.
#   2^-126     ex2.approx.ftz flushes results below the smallest normal fp32 to zero.
KL_GRAD_EPS = 2e-5
# Per-row bounds of row_out = (x, nll, lse_S, lse_T): lse (and nll = lse_S - s[label]) within 1e-5 + 2e-6 |lse| (a few fp32 ulps of lse
# plus the fp32 sum-exp); x = sum p log q within 2e-5 |x| + 1e-5.
KL_LSE_RTOL, KL_LSE_ATOL = 2e-6, 1e-5
KL_X_RTOL, KL_X_ATOL = 2e-5, 1e-5


def check_dlogits(d, ref, msg="dlogits", eps=KL_GRAD_EPS, block=64):
    """d: the kernel's [N, >= V] bf16 gradient; ref: kl_reference_fp64's result.  Compared in blocks of rows (the full-vocabulary case is
    hundreds of MB per float temporary)."""
    g_all, sc_all = ref["g"], ref["gscale"]
    N, V = g_all.shape
    nbad, first = 0, None
    for r0 in range(0, N, block):
        r1 = min(N, r0 + block)
        g = g_all[r0:r1].to(d.device, torch.float64)
        err = (d[r0:r1, :V].double() - g).abs()
        tol = 2.0 ** -8 * g.abs() + eps * sc_all[r0:r1].to(d.device, torch.float64) + 2.0 ** -126
        bad = ~(err <= tol)                                       # NaN counts as bad
        if bad.any():
            nbad += int(bad.sum())
            if first is None:
                i = torch.nonzero(bad)[0]
                r, c = int(i[0]), int(i[1])
                first = (r0 + r, c, float(d[r0 + r, c]), float(g[r, c]), float(tol[r, c]))
    assert nbad == 0, f"{msg}: {nbad} / {N * V} elements out of bound; first (row, col, got, want, tol) = {first}"


def check_row_out(row_out, ref, msg="row_out"):
    got, want = row_out.double().cpu(), ref["row"].cpu()
    for j, name, rtol, atol, scale in ((0, "x", KL_X_RTOL, KL_X_ATOL, 0), (1, "nll", KL_LSE_RTOL, KL_LSE_ATOL, 2),
                                       (2, "lse_S", KL_LSE_RTOL, KL_LSE_ATOL, 2), (3, "lse_T", KL_LSE_RTOL, KL_LSE_ATOL, 3)):
        err = (got[:, j] - want[:, j]).abs()
        tol = atol + rtol * want[:, scale].abs()
        bad = ~(err <= tol)
        assert not bad.any(), (f"{msg} {name}: {int(bad.sum())} / {len(bad)} rows out of bound; first row {int(torch.nonzero(bad)[0])}: "
                               f"got {got[bad][0].tolist()} want {want[bad][0].tolist()}")


def check_out4(out4, ref, msg="out4"):
    o = out4.double().cpu()
    assert o[2].item() == ref["n_kd"] and o[3].item() == ref["n_ce"], (msg, o.tolist(), ref["n_kd"], ref["n_ce"])
    for j, key in ((0, "align"), (1, "ce")):
        assert abs(o[j].item() - ref[key]) <= 2e-5 * abs(ref[key]) + 1e-6, (msg, key, o[j].item(), ref[key])


# ---------------------------------------------------------------------------------------------------
# log-prob gather and the dense compat forms (csrc/logp.cu): float64 references and element-wise bounds
# ---------------------------------------------------------------------------------------------------
# Every kernel of logp.cu gives a row to one CTA of 256 threads.  The lse is an online (m, z) per thread over the thread's columns
# (16-byte vectors i, i + 256, ... then the tail; softmax_rows strides single columns by 256), then block_max / block_sum and
# lse = M + lg2(Z) ln2.  Bounds in the regime |x| < 128 for every finite logit (so |lse| < 128 + ln V; every case tested), with
# A = max(|lse|, max |finite x|) of the row:
#   lse:  KL_LSE_ATOL + KL_LSE_RTOL A + (ceil(V/256) + 20) 2^-24
#           KL_LSE_*: -m log2e rounded once per thread (2^-24 |m| nats, |m| <= A), the fma x log2e - m log2e rounded (2^-24 |x - m| log2e
#           on a term of weight e^-|x - m|, at most 2^-24 in all), fp32 log2e (2^-26 |x - m|), ex2.approx per term and per rescale of z
#           (2^-22 each; a thread's running max rises about ln(n) times on rows in random order), lg2.approx and the roundings of
#           M + lg2(Z) ln2 -- far below 1e-5 + 2e-6 A.
#           The fp32 sum Z: a thread adds at most 8 ceil(V/2048) + 1 <= ceil(V/256) + 9 positive terms in order, block_sum 10 more levels
#           (5 shuffles, 5 over the warps' partials): relative (ceil(V/256) + 20) 2^-24, the same in nats.
#   tok = x[label] - lse:  the lse bound + 2^-24 |tok|.
#   seq (logp_seq_sum_kernel):  the sum of the active rows' tok bounds + (ceil((T-1)/256) + 10) 2^-24 sum|tok| (a thread adds
#           ceil((T-1)/256) rows in order, then block_sum); the average form divides by the exact count: that / n + 2^-24 |avg|.
#   d logits = bf16(-g q + g onehot), q = ex2(fma(x, log2e, -lse_k log2e)) from the forward's fp32 lse_k:
#           2^-8 |d| + eps |g| (q + onehot) + 2^-126 (1 + |g|), eps = LOGP_GRAD_EPS per element:
#             the lse bound (lse_k - lse) + 2^-24 |lse| (-lse_k log2e rounded) + 2^-23 |x - lse| (the fma rounded, fp32 log2e)
#             + 2^-21 (ex2.approx 2^-22, the product -g q and the add of g, and the fp32 g its caller formed, 2^-24 each);
#           as in KL_GRAD_EPS the cancellation of g onehot - g q on the label column turns the relative error of q into an absolute one.
#           2^-126 (1 + |g|): ex2.approx.ftz flushes q below 2^-126 to zero.
#   softmax_rows:  log mode  x - lse_k:  the lse bound + 2^-24 |x - lse|;
#                  prob mode ex2((x - lse_k) log2e):  p (the lse bound + 3 2^-24 |x - lse| + 2^-22) + 2^-126  (the difference, fp32
#                  log2e and the product rounded, ex2.approx).
#   align_loss_dense, from the kernel's own fp32 logp and probs (only the reductions are under test):
#           row_x = sum p l over the finite l:  (ceil(V/256) + 12) 2^-24 sum|p l|  (a product and an add per term, block_sum);
#           loss = -sum(row_x m) / sum(m):  (sum of the masked row_x bounds + (ceil(n/1024) + 10) 2^-24 sum|row_x m|) / sum(m)
#           + 2^-24 |loss|  (1024 threads, block_sum; the count is exact).
# Values that are not finite in the reference (tok = -inf at a -inf label, the 0/0 average) must match exactly: see check_exact_bound.
LOGP_ABS_FLOOR = 2.0 ** -126


def logp_lse_tol(lse, amax, V):
    return KL_LSE_ATOL + KL_LSE_RTOL * torch.maximum(lse.abs(), amax) + (math.ceil(V / 256) + 20) * FP32_U


def _finite_absmax(x):
    return torch.where(torch.isfinite(x), x.abs(), torch.zeros_like(x)).amax(-1)


def _seq_chain(T):
    return math.ceil(max(T - 1, 0) / 256) + 10


def logp_reference_fp64(logits, labels, T, V, g_seq=None, g_dtype=torch.float64, block_bytes=1 << 30):
    """Float64 restatement of lmod_logp_gather_fwd / _bwd (R.dpo_get_logp and its gradient) on [N, >= V] bf16 logits (the first V columns)
    and the flat [N] labels of B = N / T sequences.  Row r = b T + t predicts labels[r + 1]; the last position of a sequence has no next
    label.  Works on the tensors' device in blocks of rows so that the float64 temporaries stay near `block_bytes`.  Returns a dict:
      nxt, active [N]     the next label (-100 when none) and whether it is set
      lse, tok [N]        float64, 0 on masked rows (as the kernel writes them); tok = x[next label] - lse
      lse_tol, tok_tol    the bounds above
      seq, seq_tol [B]    the masked sum of tok; avg, avg_tol the average form (0/0 gives NaN, as R.dpo_get_logp); n [B] the counts
    With g_seq [B] (the upstream gradient of seq):
      g [N, V]            g_b (onehot(next label) - q) on active rows, 0 on masked rows (g_dtype)
      gscale [N, V]       |g_b| (q + onehot), the size of the two terms the kernel combines
      g_tol [N, V]        the element-wise bound of the bf16 d logits
    One input differs from R.dpo_get_logp on purpose: a -inf at column 0 of a masked row.  R.dpo_get_logp gathers column 0 there (the
    label is replaced by 0) and multiplies -inf by 0, which is NaN in its sum; the kernel skips masked rows and writes 0, as this does."""
    x_all = logits[:, :V]
    dev = x_all.device
    labels = labels.reshape(-1).to(dev)
    N = labels.numel()
    B = N // T
    _, active, nxt = kl_row_masks(labels, T)
    lab = torch.where(active, nxt, torch.zeros_like(nxt))
    f64 = torch.float64
    lse = torch.zeros(N, dtype=f64, device=dev)
    tok = torch.zeros_like(lse)
    amax = torch.zeros_like(lse)
    grads = g_seq is not None
    if grads:
        gb_row = g_seq.to(dev, f64).repeat_interleave(T) * active.to(f64)
        g = torch.zeros(N, V, dtype=g_dtype, device=dev)
        gscale = torch.zeros_like(g)
        g_tol = torch.zeros_like(g)
    step = max(1, block_bytes // (8 * 8 * V))
    for r0 in range(0, N, step):
        r1 = min(N, r0 + step)
        x = x_all[r0:r1].to(f64)
        l_b = torch.logsumexp(x, -1)
        a_b = _finite_absmax(x)
        t_b = x.gather(1, lab[r0:r1, None])[:, 0] - l_b
        act = active[r0:r1]
        lse[r0:r1] = torch.where(act, l_b, torch.zeros_like(l_b))
        tok[r0:r1] = torch.where(act, t_b, torch.zeros_like(t_b))
        amax[r0:r1] = torch.where(act, a_b, torch.zeros_like(a_b))
        if grads:
            gr = gb_row[r0:r1, None]
            q = (x - l_b[:, None]).exp()
            oh = torch.zeros_like(q).scatter_(1, lab[r0:r1, None], 1.0)
            gg = gr * (oh - q)
            sc = gr.abs() * (q + oh)
            dx = torch.where(torch.isfinite(x), (x - l_b[:, None]).abs(), torch.zeros_like(x))
            eps = logp_lse_tol(l_b, a_b, V)[:, None] + FP32_U * l_b.abs()[:, None] + 2 * FP32_U * dx + 2.0 ** -21
            gt = BF16_U * gg.abs() + eps * sc + LOGP_ABS_FLOOR * (1 + gr.abs())
            g[r0:r1] = torch.where(act[:, None], gg, torch.zeros_like(gg)).to(g_dtype)
            gscale[r0:r1] = torch.where(act[:, None], sc, torch.zeros_like(sc)).to(g_dtype)
            g_tol[r0:r1] = torch.where(act[:, None], gt, torch.zeros_like(gt)).to(g_dtype)
            del q, oh, gg, sc, dx, eps, gt
        del x
    lse_tol = torch.where(active, logp_lse_tol(lse, amax, V), torch.zeros_like(lse))
    tok_tol = torch.where(active, lse_tol + FP32_U * tok.abs(), torch.zeros_like(lse))
    m = active.to(f64).view(B, T)
    tk = tok.view(B, T)
    seq = (tk * m).sum(-1)
    n = m.sum(-1)
    seq_tol = (tok_tol.view(B, T) * m).sum(-1) + _seq_chain(T) * FP32_U * (tk.abs() * m).sum(-1)
    avg = seq / n
    avg_tol = seq_tol / n + FP32_U * avg.abs()
    out = dict(nxt=nxt, active=active, lse=lse, tok=tok, lse_tol=lse_tol, tok_tol=tok_tol, seq=seq, seq_tol=seq_tol, avg=avg,
               avg_tol=avg_tol, n=n)
    if grads:
        out.update(g=g, gscale=gscale, g_tol=g_tol)
    return out


def softmax_rows_reference_fp64(logits, V, log_mode):
    """lmod_softmax_rows on [N, >= V] bf16 logits (the first V columns): log_softmax (log_mode) or softmax of each row in float64, with the
    bound above.  Returns (out [N, V], tol [N, V]) float64 on the logits' device; -inf logits give -inf (log mode) or 0."""
    x = logits[:, :V].to(torch.float64)
    lse = torch.logsumexp(x, -1, keepdim=True)
    lt = logp_lse_tol(lse, _finite_absmax(x)[:, None], V)
    y = x - lse
    dx = torch.where(torch.isfinite(y), y.abs(), torch.zeros_like(y))
    if log_mode:
        return y, lt + FP32_U * dx
    p = y.exp()
    return p, p * (lt + 3 * FP32_U * dx + 2.0 ** -22) + LOGP_ABS_FLOOR


def align_dense_reference_fp64(logp, probs, labels, distill_all=False):
    """lmod_align_loss_dense (R.compute_align_loss) in float64 on the kernel's own fp32 inputs logp, probs [N, V] and the flat [N] labels
    (not shifted; distill_all counts every row).  row_x = sum p l over the finite l; loss = -sum(row_x m) / sum(m), NaN when no row
    counts.  Returns dict(row_x, row_x_tol [N], loss, loss_tol) with the bounds above."""
    l, p = logp.to(torch.float64), probs.to(torch.float64)
    n, V = l.shape
    fin = torch.isfinite(l)
    pl = torch.where(fin, p * torch.where(fin, l, torch.zeros_like(l)), torch.zeros_like(l))
    row_x = pl.sum(-1)
    row_tol = (math.ceil(V / 256) + 12) * FP32_U * pl.abs().sum(-1)
    labels = labels.reshape(-1).to(l.device)
    m = torch.ones_like(row_x) if distill_all else (labels != IGNORE_INDEX).to(torch.float64)
    c = m.sum()
    loss = -(row_x * m).sum() / c
    loss_tol = ((row_tol * m).sum() + (math.ceil(n / 1024) + 10) * FP32_U * (row_x.abs() * m).sum()) / c + FP32_U * loss.abs()
    return dict(row_x=row_x, row_x_tol=row_tol, loss=loss, loss_tol=loss_tol)


def check_exact_bound(name, got, want, tol, report=None, block=256):
    """Element-wise |got - want| <= tol for the logp.cu outputs ([N] or [N, V]; compared in blocks of rows).  An element equal to the
    reference passes (-inf = -inf, and a NaN where the reference has NaN: the 0/0 average); where the reference is not finite nothing else
    does.  On failure names the first element out of bound and the worst err / bound.  Returns the worst err / bound; `report`, a dict,
    keeps the largest under `name`."""
    got = got.detach().reshape(-1) if got.dim() == 0 else got.detach()
    want, tol = torch.as_tensor(want).to(got.device).reshape(got.shape), torch.as_tensor(tol).to(got.device).reshape(got.shape)
    nbad, first, worst = 0, None, 0.0
    for r0 in range(0, max(1, got.shape[0]), block):
        g, w = got[r0:r0 + block].to(torch.float64), want[r0:r0 + block].to(torch.float64)
        t = tol[r0:r0 + block].to(torch.float64)
        same = (g == w) | (torch.isnan(g) & torch.isnan(w))
        t = torch.where(torch.isfinite(w), t, torch.zeros_like(t))
        err = torch.where(same, torch.zeros_like(g), (g - w).abs().nan_to_num(float("inf")))
        ok = same | (err <= t)
        ratio = torch.where(same, torch.zeros_like(err), (err / t).nan_to_num(float("inf"), float("inf"), float("inf")))
        if ratio.numel():
            worst = max(worst, float(ratio.max()))
        if not bool(ok.all()):
            nbad += int((~ok).sum())
            if first is None:
                i = tuple(int(v) for v in torch.nonzero(~ok)[0])
                first = ((r0 + i[0],) + i[1:], g[i].item(), w[i].item(), t[i].item())
    if report is not None:
        report[name] = max(worst, report.get(name, 0.0))
    assert nbad == 0, (f"{name}: {nbad} / {got.numel()} elements out of bound, max err/bound {worst:.3g}; first (index, got, want, bound) "
                       f"= {first}")
    return worst


# ---------------------------------------------------------------------------------------------------
# flash attention (csrc/attn.cu, csrc/attn_bwd.cu): float64 reference and element-wise bounds
# ---------------------------------------------------------------------------------------------------
def attn_visible(B, T, causal, keep=None, device="cpu"):
    """[B, T, T] bool: may query row i see key j.  The semantics of R.sdpa_mask: the causal mask plus key padding (keep [B, T] bool,
    contiguous real tokens), and a row with no visible key (in front of a left-padded sequence, or a sample that is all padding) sees every
    key.  Key padding goes with causal=True only, as in the kernels."""
    assert causal or keep is None, "key padding is only defined together with the causal mask"
    vis = torch.ones(T, T, dtype=torch.bool, device=device)
    if causal:
        vis = vis.tril()
    vis = vis[None].expand(B, T, T)
    if keep is not None:
        vis = vis & keep.to(device=device, dtype=torch.bool)[:, None, :]
    return vis | ~vis.any(-1, keepdim=True)


# Element-wise bounds of the kernels against attn_reference_fp64, from the kernels' own arithmetic.  u = 2^-8 is the unit roundoff of bf16,
# 2^-24 that of fp32.  Per query row i (natural-log units, s_ij = q_i.k_j the raw dot product, c = scale):
#   A_i     = max_j sum_d |q_id k_jd| over the visible keys, Smax_i = max_j |s_ij|.
#   delta_i bounds the relative error of every fp32 P_ij = ex2(fma(s_ij, c log2e, -m)) the kernels form:
#             c (hd/16 + 1) 2^-23 A_i   the fp32 score from wgmma, which truncates its accumulator at each k = 16 step (hd/16 steps, +1 for
#                                       the alignment inside a step);
#             2^-22 c Smax_i            the fp32 constant c log2e (2^-23 relative) and the rounding of the fma residual (|.| <= 2 c Smax log2e);
#             2^-22                     ex2.approx.
#   gamma_i = (n_i/4 + 2 nblk_i + 4) 2^-24, the fp32 sum l (each of the 4 threads of a row adds n/4 terms in order, one fma per key block,
#             then two shuffles) and the rescales of o and l by alpha once per key block; n_i visible keys, nblk_i <= n_i/BKV + 2 blocks.
#   o:   |o_k - o| <= 2^-8 |o| + (2^-8 + (n_i/16 + 2) 2^-23 + 2 delta_i + gamma_i) (P|V|)_i
#             2^-8 |o| is the bf16 store.  P is rounded to bf16 before P V (2^-8) while l sums the unrounded P; the fp32 accumulator of P V
#             truncates at each of the (n_i/16 + 2) k = 16 steps that hold a visible key; o/l carries delta_i from the numerator and from the
#             denominator, and gamma_i from l.  P|V| = sum_j p_ij |v_j| majorises every one of these sums.
#   lse: |lse_k - lse| <= delta_i + gamma_i + 2^-22 (2 + log2 n_i + |lse_i|)
#             the shift m cancels between m and the P it scales; lg2.approx (2^-22 absolute per unit of log2 l) and the fp32 roundings of
#             m + lg2(l) and of the product by ln2.
# Backward (P recomputed as ex2(fma(s, c log2e, -lse_k log2e)) from the forward's fp32 lse_k):
#   deltab_i = the score and ex2 terms of delta_i + 2^-22 |lse_i| (lse_k log2e rounded, the fma residual) + |lse_k,i - lse_i|.
#   dP_ij = dO_i.V_j in fp32 wgmma: error (hd/16 + 1) 2^-23 (|dO_i|.|V_j|).  D_i from attn_dsum_kernel is rowsum(dO_i o_k,i) of the
#   forward's bf16 output: its difference from the exact rowsum(dO_i O_i) is dD_i = rowsum(dO_i (o_k,i - O_i)), computed exactly here, plus
#   the fp32 sum (hd/32 fmas per lane, then five shuffles): (hd/32 + 6) 2^-24 sum |dO_i o_k,i|.
#   dS = P (dP - D) c goes to bf16 before both of its products, so every dS_ij is off by at most c E_ij with
#     E_ij = P_ij ((2^-8 + deltab_i + 2^-22) |dP_ij - D_i| + (1 + 2^-7) (err(dP_ij) + |dD_i| + err(D_i))),   F_ij = P_ij |dP_ij - D_i|.
#   The bf16 rounding of dS acts on the kernel's dS, which already carries the dP and D errors: in a peaked row dP - D nearly cancels
#   and those errors can be most of dS, so they are counted (1 + 2^-8)(1 + deltab) <= 1 + 2^-7 times.
#   dV: |dV_k - dV| <= 2^-8 |dV| + (2^-8 + (n_kv + 1) 2^-23) (P^T |dO|) + (P^T (deltab |dO|))
#   dK: |dK_k - dK| <= 2^-8 |dK| + c (E^T |Q|) + c (n_kv + 1) 2^-23 (F^T |Q|)
#             n_kv = group (T/16 + 1) bounds the k = 16 steps of the register accumulators of dK and dV over every query of every head of the
#             GQA group (the heads' terms are summed here in float64 too).
#   dQ: |dQ_k - dQ| <= 2^-8 |dQ| + c (E |K|) + c (9 2^-23 + n_kb 2^-24) (F |K|)
#             each 128-key block adds its partial dS K (8 wgmma k-steps) with an fp32 red.add; n_kb = T/128 + 1 adds in any order.
#   Every bound also gets ATTN_ABS_FLOOR: ex2.approx.ftz flushes P below 2^-126 to zero, which moves no sum by more than T 2^-126 max|v|.
ATTN_ABS_FLOOR = 2.0 ** -100


def attn_reference_fp64(qkv, B, T, nh, nkv, hd, causal, scale, keep=None, dout=None, out_kernel=None, lse_kernel=None,
                        block_bytes=3 << 29):
    """Plain float64 attention on the fused bf16 QKV buffer [B*T, (nh + 2 nkv) hd] (q heads | k heads | v heads, GQA by index: query head h
    reads kv head h // (nh / nkv)), under the mask of attn_visible.  Runs on qkv's device in blocks of heads, so that the float64 [T, T]
    temporaries of one block stay near `block_bytes`.

    Returns a dict: o [B*T, nh*hd] and lse [B, nh, T] (float64, the kernel's layouts) with their bounds o_tol and lse_tol, and the majorants
    behind them (PV = P|V|, delta, nvis per row).  With dout [B*T, nh*hd], also dqkv [B*T, (nh + 2 nkv) hd] from the analytic gradients
    (P, dP = dO V^T, D = rowsum(dO O), dS = P (dP - D)) and its bound dqkv_tol.  out_kernel / lse_kernel, the forward kernel's outputs that
    the backward kernel consumes, make the dD and lse terms of the gradient bounds exact; without them the forward bounds stand in."""
    dev = qkv.device
    f64 = torch.float64
    x = qkv.detach().to(f64).view(B, T, nh + 2 * nkv, hd)
    q, k, v = (x[:, :, a:b].permute(0, 2, 1, 3) for a, b in ((0, nh), (nh, nh + nkv), (nh + nkv, nh + 2 * nkv)))
    vis = attn_visible(B, T, causal, keep, dev)
    nvis = vis.sum(-1).to(f64)                                       # [B, T]
    group = nh // nkv
    bkv = 128 if hd <= 64 else 64
    u, e23, e22, e24 = 2.0 ** -8, 2.0 ** -23, 2.0 ** -22, 2.0 ** -24
    o = torch.zeros(B, nh, T, hd, dtype=f64, device=dev)
    o_tol, PVall = torch.zeros_like(o), torch.zeros_like(o)
    lse = torch.zeros(B, nh, T, dtype=f64, device=dev)
    lse_tol, delta_all = torch.zeros_like(lse), torch.zeros_like(lse)
    grads = dout is not None
    if grads:
        do = dout.detach().to(dev, f64).view(B, T, nh, hd).permute(0, 2, 1, 3)
        ok = None if out_kernel is None else out_kernel.detach().to(dev, f64).view(B, T, nh, hd).permute(0, 2, 1, 3)
        lk = None if lse_kernel is None else lse_kernel.detach().to(dev, f64)
        dq, dq_tol = torch.zeros_like(o), torch.zeros_like(o)
        dk = torch.zeros(B, nkv, T, hd, dtype=f64, device=dev)
        dv, dk_tol, dv_tol = torch.zeros_like(dk), torch.zeros_like(dk), torch.zeros_like(dk)
        n_kv = group * (T / 16 + 1)
        n_kb = T / 128 + 1
    hb = max(1, min(nh, block_bytes // (12 * 8 * T * T)))
    ninf = float("-inf")
    for b in range(B):
        visb, nv = vis[b], nvis[b][:, None]                          # [T, T], [T, 1]
        for h0 in range(0, nh, hb):
            h1 = min(nh, h0 + hb)
            kvi = torch.arange(h0, h1, device=dev) // group
            qb, kb, vb = q[b, h0:h1], k[b][kvi], v[b][kvi]           # [h, T, hd]
            s = (qb @ kb.transpose(-1, -2)).masked_fill(~visb, ninf)
            lse_b = torch.logsumexp(s * scale, -1)                   # [h, T]
            P = torch.exp(s * scale - lse_b[..., None])
            ob = P @ vb
            A = (qb.abs() @ kb.abs().transpose(-1, -2)).masked_fill(~visb, 0).amax(-1)
            Smax = s.abs().masked_fill(~visb, 0).amax(-1)
            d_score = scale * ((hd / 16 + 1) * e23 * A + e22 * Smax)
            delta = d_score + e22
            gamma = (nv[:, 0] / 4 + 2 * (nv[:, 0] / bkv + 2) + 4) * e24
            PV = P @ vb.abs()
            o[b, h0:h1], lse[b, h0:h1], PVall[b, h0:h1], delta_all[b, h0:h1] = ob, lse_b, PV, delta
            o_tol[b, h0:h1] = u * ob.abs() + (u + (nv / 16 + 2) * e23 + 2 * delta[..., None] + gamma[..., None]) * PV + ATTN_ABS_FLOOR
            lse_t = delta + gamma + e22 * (2 + torch.log2(nv[:, 0]) + lse_b.abs()) + ATTN_ABS_FLOOR
            lse_tol[b, h0:h1] = lse_t
            if not grads:
                continue
            dob = do[b, h0:h1]
            okb = ob if ok is None else ok[b, h0:h1]
            lerr = lse_t if lk is None else (lk[b, h0:h1] - lse_b).abs()
            deltab = d_score + e22 * (1 + lse_b.abs()) + lerr        # [h, T]
            dP = dob @ vb.transpose(-1, -2)
            D = (dob * ob).sum(-1)
            if ok is None:
                dD = (dob.abs() * o_tol[b, h0:h1]).sum(-1)
            else:
                dD = (dob * (okb - ob)).sum(-1).abs()
            eD = (hd / 32 + 6) * e24 * (dob.abs() * okb.abs()).sum(-1)
            edP = (hd / 16 + 1) * e23 * (dob.abs() @ vb.abs().transpose(-1, -2))
            R = dP - D[..., None]
            dS = P * R
            F = P * R.abs()
            E = (u + deltab[..., None] + e22) * F + (1 + 2.0 ** -7) * P * (edP + (dD + eD)[..., None])
            del s, dP, R, edP
            qa, ka = qb.abs(), kb.abs()
            dq[b, h0:h1] = scale * (dS @ kb)
            dq_tol[b, h0:h1] = scale * (E @ ka + (9 * e23 + n_kb * e24) * (F @ ka))
            Pt = P.transpose(-1, -2)
            dk[b].index_add_(0, kvi, scale * (dS.transpose(-1, -2) @ qb))
            dv[b].index_add_(0, kvi, Pt @ dob)
            dk_tol[b].index_add_(0, kvi, scale * (E.transpose(-1, -2) @ qa + (n_kv + 1) * e23 * (F.transpose(-1, -2) @ qa)))
            dv_tol[b].index_add_(0, kvi, (u + (n_kv + 1) * e23) * (Pt @ dob.abs()) + Pt @ (deltab[..., None] * dob.abs()))
            del P, Pt, dS, F, E
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(B * T, -1)       # noqa: E731  [B, H, T, hd] -> [B*T, H*hd]
    res = dict(o=rows(o), lse=lse, o_tol=rows(o_tol), lse_tol=lse_tol, PV=rows(PVall), delta=delta_all, nvis=nvis)
    if grads:
        res["dqkv"] = torch.cat([rows(dq), rows(dk), rows(dv)], 1)
        res["dqkv_tol"] = torch.cat([rows(dq_tol + u * dq.abs()), rows(dk_tol + u * dk.abs()), rows(dv_tol + u * dv.abs())], 1) + ATTN_ABS_FLOOR
    return res


def check_attn(name, got, want, tol, T, hd=None, report=None):
    """Element-wise |got - want| <= tol.  got / want / tol in the kernel's layouts: [B*T, H*hd] (row b*T + t, column h*hd + d; pass hd) or
    lse [B, H, T].  On failure names the worst element by (sample, head, row, column), the count out of bound and max(err / bound).
    Returns max(err / bound); `report`, a dict, collects it under `name`."""
    got = got.detach().to(want.device, torch.float64)
    err = (got - want).abs()
    ratio = (err / tol).nan_to_num(float("inf"))                    # a NaN in got counts as out of bound
    bad = ~(err <= tol)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if report is not None:
        report[name] = max(worst, report.get(name, 0.0))
    nbad = int(bad.sum())
    if nbad:
        i = int(ratio.reshape(-1).argmax())
        if got.dim() == 3:
            H = got.shape[1]
            where = dict(sample=i // (H * T), head=(i // T) % H, row=i % T, column=None)
        else:
            r, c = divmod(i, got.shape[1])
            where = dict(sample=r // T, head=c // hd, row=r % T, column=c % hd)
        g, w, t = got.reshape(-1)[i].item(), want.reshape(-1)[i].item(), tol.reshape(-1)[i].item()
        raise AssertionError(f"{name}: {nbad} / {got.numel()} elements out of bound, max err/bound {worst:.3g}; worst at {where}: "
                             f"got {g!r} want {w!r} bound {t:.3g}")
    return worst


def check_attn_grads(name, dqkv, ref, T, nh, nkv, hd, report=None):
    """dq, dk and dv of a fused gradient buffer against attn_reference_fp64(..., dout=...)."""
    out = {}
    for part, sl in (("dq", slice(0, nh * hd)), ("dk", slice(nh * hd, (nh + nkv) * hd)), ("dv", slice((nh + nkv) * hd, None))):
        out[part] = check_attn(f"{name} {part}", dqkv[:, sl], ref["dqkv"][:, sl], ref["dqkv_tol"][:, sl], T, hd, report)
    return out


def make_trainer(student, teacher, loss_type="kd_lm", accum=1, lr=2e-5, max_steps=100, kind="align", moe_loss_enable=True):
    from llavamod.config.args import TrainingArguments
    from llavamod.train.align_trainer import AlignTrainer
    from llavamod.train.dpo_trainer import DPOTrainer
    args = TrainingArguments(output_dir="/tmp/lmod_out", per_device_train_batch_size=1, gradient_accumulation_steps=accum,
                             learning_rate=lr, weight_decay=0.0, warmup_ratio=0.03, lr_scheduler_type="cosine", max_steps=max_steps,
                             logging_steps=0, save_strategy="no", bf16=True)
    args.moe_enable = True
    cls = AlignTrainer if kind == "align" else DPOTrainer
    tr = cls(model=student, ref_model=teacher, args=args, loss_type=loss_type, moe_loss_enable=moe_loss_enable)
    tr._total_steps = max_steps
    return tr


# ---------------------------------------------------------------------------------------------------
# sparse MoE block (csrc/moe.cu, grouped modes of csrc/gemm.cu, kernels.MoEFn): float64 reference and element-wise bounds
# ---------------------------------------------------------------------------------------------------
# Every stage is recomputed in float64 from the tensors the kernels produced at the stage before it, so each bound covers the arithmetic
# of one stage and errors do not compound.  u = 2^-8 is the unit roundoff of bf16, 2^-24 that of fp32.
#   GEMM stages (h1, y, dact, dxp; the wgrads dW_gu, dW_dn with the old buffer value in ref):
#       |got - ref| <= 2^-8 |ref| + (1 + 2^-8) (ceil(K/16) + 1) 2^-23 (|A| |B|)  [+ 2^-23 |ref| for the fp32 add of the old value]
#     the wgmma fp32 accumulator truncates toward zero at each k = 16 step (relative 2^-23 per step, +1 for the alignment inside a step),
#     so (|A||B|) majorises the error element by element; the bf16 store adds half an ulp (2^-8 relative) of the rounded value.  K is the
#     reduction length: H or I (or 2I) for the row GEMMs, the group's 128-aligned row count for the wgrads.
#   fp32 FMA chains: n 2^-24 sum|a||b|, n the chain the kernel runs:
#     logits   H/32 FMAs per lane + 5 butterfly adds             dw      (combine_bwd) the same over dout . y
#     dwg      ceil(S/32) FMAs per split + 32 split sums + the add to the old value
#     dx       dxp[r1] + dxp[r2] + E FMAs of dlogits . wg (E + 2 roundings), then the bf16 store (2^-8 |ref|)
#   gates: softmax of the kernel's fp32 logits with expf (<= 2 ulp), the rounded shift l - max, an E-term sum and a division:
#       |got - ref| <= 2^-22 (E + 4 + max_e |l - max|) g
#   act / dh1: SwiGLU of the kernel's bf16 h1.  bf16(silu(g)) and the bf16 store are 2^-8 each; the sigmoid (__expf: relative error
#     about 2^-22 (2 + |g|)) and the fp32 products are covered by 2^-16.  dh1 also carries the error of dact (bf16 of a GEMM
#     accumulator): 2^-8 |dact| + the GEMM term above, times |d dh1 / d dact|.
#   dlogits: gate_bwd's fp32 arithmetic.  dg_e (l_aux term + renormalisation term) is off by at most 16 2^-24 D_e (D_e the sum of the
#     terms' magnitudes), the dot sum_j g_j dg_j by sum_j g_j (16 2^-24 D_j + E 2^-24 |dg_j|), the final g (dg - dot) by 2 2^-24 of itself.
#   l_aux: E sum_e mean(g_e) count_e / S over the tiles' fp32 sums (tpb + ntiles + E + 8 roundings of positive terms).
# Bit-exact stages (compared by bits against a torch fp32 emulation): the scatter copy (xp rows = x rows); w = g / max(g1 + g2, eps) of
# the kernel's gates; dy = bf16(bf16(w) dout); out = bf16(res + bf16(fp32(bf16(w1) y1 + bf16(w2) y2))) (both products are exact in fp32,
# so the sum is one rounding, as the kernel's fma); zero padding rows of xp, h1, act and y below offsets[E].
FLT_EPS = 2.0 ** -23


def moe_route_tpb(S):
    """Tokens per CTA of the router (route_tpb in csrc/moe.cu): a multiple of 16 that keeps the grid at <= 1024 CTAs."""
    tpb = 16
    while -(-S // tpb) > 1024:
        tpb += 16
    return tpb


def _gemm_tol(ref, maj, K):
    return 2.0 ** -8 * ref.abs() + (1 + 2.0 ** -8) * (math.ceil(K / 16) + 1) * 2.0 ** -23 * maj


def moe_reference_fp64(x, res, wg, w_gu, w_dn, noise, cf, min_cap, dout=None, g_laux=0.0, old=None, k=None, eps=FLT_EPS, w_bf16=True,
                       store=torch.float64):
    """Float64 restatement of the sparse-MoE block (DeepSpeed top-2 gating, SwiGLU experts, combine) stage by stage.

    x, res [S, H] bf16; wg [E, H] fp32; w_gu [E, 2I, H], w_dn [E, H, I] bf16; noise [S, E] fp32.  With dout [S, H] (and g_laux, the
    upstream gradient of l_aux) the backward stages too; old: the gradient buffers' values before the call ({'wg', 'w_gu', 'w_dn'}).
    k: the kernels' tensors per stage (kernels.moe_forward_stages / moe_backward_stages, plus the grads under 'g_wg', 'g_w_gu', 'g_w_dn');
    every stage takes its inputs from k.  Without k the reference chains its own float64 stages.  eps is the clamp of the renormalisation
    (fp32's in the kernels), w_bf16 rounds the combine weights to bf16 (the einsum's type_as in the model).  Works on x's device.

    Returns {stage: (want, tol)} -- tol None for bit-exact stages -- plus the routing record under 'rec' (top2gating of the fp32 logits:
    idx [S, 2], row [S, 2] in the 128-aligned compact layout, offsets [E+1], used [E], counts [E], capacity) and, for each GEMM stage, its
    rows (the routed rows below offsets[E]); want/tol of the large stages are kept as `store`."""
    dev = x.device
    f64 = torch.float64
    S, H = x.shape
    E, I2, _ = w_gu.shape
    I = I2 // 2
    kk = k if k is not None else {}
    out = {}
    own = {}

    def src(name):
        return (kk[name] if name in kk and kk[name] is not None else own[name])

    x64, wg64 = x.to(f64), wg.to(dev, f64)
    # ---- gate: logits (fp32 GEMV), softmax, routing record
    logits = x64 @ wg64.t()
    own["logits"] = logits
    lane_fmas = 8 * -(-H // 256)                                 # per lane: ceil(H / 8 / 32) vectors of 8 (gate GEMV, combine_bwd)
    out["logits"] = (logits, (lane_fmas + 6) * 2.0 ** -24 * (x64.abs() @ wg64.abs().t()))
    lk = src("logits").to(f64)
    gates = torch.softmax(lk, 1)
    own["gates"] = gates
    out["gates"] = (gates, 2.0 ** -22 * (E + 4 + (lk - lk.amax(1, keepdim=True)).abs().amax(1, keepdim=True)) * gates)
    o = R.top2gating(lk.float().cpu(), noise.float().cpu(), cf, min_cap)
    C = o["capacity"]
    idx = torch.stack([o["idx1"], o["idx2"]], 1).to(dev)
    keep = torch.stack([o["keep1"], o["keep2"]], 1).to(dev)
    counts = o["exp_counts"].to(dev)
    cnt = torch.minimum(torch.bincount(idx[:, 0], minlength=E) + torch.bincount(idx[:, 1], minlength=E), torch.tensor(C, device=dev))
    offsets = torch.zeros(E + 1, dtype=torch.long, device=dev)
    offsets[1:] = ((cnt + 127) // 128 * 128).cumsum(0)
    slot = torch.stack([o["slot1"], o["slot2"]], 1).to(dev)
    row = torch.where(keep, offsets[idx] + slot, torch.full_like(slot, -1))
    rec = dict(idx=idx, row=row, keep=keep, offsets=offsets, used=cnt, counts=counts, capacity=C)
    out["rec"] = rec
    gk = src("gates")
    # ---- renormalised weights (bit exact in fp32 from the kernel's gates) and l_aux
    g32 = gk.float() if "gates" in kk else gk
    gsel = torch.where(keep, g32.gather(1, idx), torch.zeros_like(g32[:, :2]))
    den = (gsel[:, 0] + gsel[:, 1]).clamp(min=eps)
    w = gsel / den[:, None]
    own["w"] = w
    out["w"] = (w, None)
    ce = counts.to(f64) / S
    laux = E * (gk.to(f64).mean(0) * ce).sum()
    tpb = moe_route_tpb(S)
    out["l_aux"] = (laux, (tpb + -(-S // tpb) + E + 8) * 2.0 ** -24 * laux.abs())
    wk = src("w")
    wr = wk.to(torch.bfloat16).to(f64) if w_bf16 else wk.to(f64)
    # ---- scatter: xp rows are the token rows; padding rows are zero
    n_rows = int(offsets[-1])
    tok = torch.full((n_rows,), -1, dtype=torch.long, device=dev)
    for c in range(2):
        tok[row[:, c][keep[:, c]]] = torch.arange(S, device=dev)[keep[:, c]]
    rec["tok"] = tok
    xp = torch.zeros(n_rows, H, dtype=x.dtype, device=dev)
    xp[tok >= 0] = x[tok[tok >= 0]]
    own["xp"] = xp
    out["xp"] = (xp, None)
    groups = [(int(offsets[e]), int(offsets[e]) + int(cnt[e]), int(offsets[e + 1])) for e in range(E)]   # (first, end of routed, end)
    rec["groups"] = groups

    def per_expert(name, a_name, wfun, K, n_out):
        want = torch.zeros(n_rows, n_out, dtype=store, device=dev)
        tol = torch.zeros_like(want)
        a = src(a_name)
        for e, (r0, r1, _) in enumerate(groups):
            if r1 > r0:
                A = a[r0:r1].to(f64)
                B = wfun(e)
                want[r0:r1] = (A @ B).to(store)
                tol[r0:r1] = _gemm_tol(want[r0:r1].to(f64), A.abs() @ B.abs(), K).to(store)
        own[name] = want
        out[name] = (want, tol)
        return want

    # ---- expert forward
    per_expert("h1", "xp", lambda e: w_gu[e].to(dev, f64).t(), H, I2)
    h1k = src("h1")[:n_rows].to(f64)
    gg, uu = h1k[:, :I], h1k[:, I:]
    sg = torch.sigmoid(gg)
    act = gg * sg * uu
    own["act"] = act.to(store)
    out["act"] = (own["act"], ((2.0 ** -7 + 2.0 ** -16) * act.abs()).to(store))
    del h1k, gg, uu, sg
    per_expert("y", "act", lambda e: w_dn[e].to(dev, f64).t(), I, H)
    # ---- combine (bit exact in fp32 from the kernel's y and w)
    yk = src("y")
    yt = torch.float32 if "y" in kk else f64
    ysel = [torch.where(keep[:, c:c + 1], yk[row[:, c].clamp(min=0)].to(yt), torch.zeros(S, H, dtype=yt, device=dev)) for c in range(2)]
    if "y" in kk:
        wb = wk.to(torch.bfloat16).float()
        comb = (wb[:, :1] * ysel[0] + wb[:, 1:] * ysel[1]).to(torch.bfloat16)
        outv = (res.float() + comb.float()).to(torch.bfloat16)
    else:
        outv = res.to(f64) + wr[:, :1] * ysel[0].to(f64) + wr[:, 1:] * ysel[1].to(f64)
    own["out"] = outv
    out["out"] = (outv, None)
    del ysel
    if dout is None:
        return out
    # ---- backward: combine -> dy (bit exact), dw (fp32 chains)
    d64 = dout.to(f64)
    dy = torch.zeros(n_rows, H, dtype=torch.bfloat16 if "w" in kk else f64, device=dev)
    for c in range(2):
        m = keep[:, c]
        if "w" in kk:
            dy[row[m, c]] = (wk[m, c:c + 1].to(torch.bfloat16).float() * dout[m].float()).to(torch.bfloat16)
        else:
            dy[row[m, c]] = wr[m, c:c + 1] * d64[m]
    own["dy"] = dy
    out["dy"] = (dy, None)
    dw = torch.zeros(S, 2, dtype=f64, device=dev)
    dwt = torch.zeros_like(dw)
    for c in range(2):
        m = keep[:, c]
        yr = yk[row[m, c]].to(f64)
        dw[m, c] = (d64[m] * yr).sum(1)
        dwt[m, c] = (lane_fmas + 6) * 2.0 ** -24 * (d64[m].abs() * yr.abs()).sum(1)
    own["dw"] = dw
    out["dw"] = (dw, dwt)
    # ---- expert backward: dact = dy W_dn, dh1 = SwiGLU backward (from the kernel's h1), wgrads, dxp
    per_expert("dact", "dy", lambda e: w_dn[e].to(dev, f64), H, I)
    dact, dact_tol = own["dact"].to(f64), out["dact"][1].to(f64)
    h1k = src("h1")[:n_rows].to(f64)
    gg, uu = h1k[:, :I], h1k[:, I:]
    sg = torch.sigmoid(gg)
    cg, cu = uu * sg * (1 + gg * (1 - sg)), gg * sg
    dh1 = torch.cat([dact * cg, dact * cu], 1)
    derr = dact_tol + 2.0 ** -16 * dact.abs()
    dh1_tol = 2.0 ** -8 * dh1.abs() + (1 + 2.0 ** -8) * torch.cat([derr * cg.abs(), derr * cu.abs()], 1)
    own["dh1"] = dh1.to(store)
    out["dh1"] = (own["dh1"], dh1_tol.to(store))
    del h1k, gg, uu, sg, cg, cu, dact, dact_tol, derr, dh1, dh1_tol
    per_expert("dxp", "dh1", lambda e: w_gu[e].to(dev, f64), I2, H)
    olds = old or {}
    for gname, a_name, b_name, M, N in (("w_dn", "dy", "act", H, I), ("w_gu", "dh1", "xp", I2, H)):
        want = torch.zeros(E, M, N, dtype=store, device=dev)
        tol = torch.zeros_like(want)
        A, B = src(a_name), src(b_name)
        for e, (r0, r1, r2) in enumerate(groups):
            o_e = olds[gname][e].to(dev, f64) if gname in olds else torch.zeros(M, N, dtype=f64, device=dev)
            if r1 > r0:
                a, b = A[r0:r1].to(f64), B[r0:r1].to(f64)
                ref = a.t() @ b + o_e
                tol[e] = (_gemm_tol(ref, a.abs().t() @ b.abs(), r2 - r0) + 2.0 ** -23 * ref.abs()).to(store)
                want[e] = ref.to(store)
            else:
                want[e] = o_e.to(store)                      # an expert without rows leaves its gradient untouched, bit for bit
        out["g_" + gname] = (want, tol)
    # ---- gate backward: dlogits through the renormalisation (clamped or not) and the softmax, plus the l_aux term
    gk64 = gk.to(f64)
    dwk = src("dw").to(f64)
    a = torch.where(keep[:, 0], gk64.gather(1, idx[:, :1])[:, 0], torch.zeros(S, dtype=f64, device=dev))
    b = torch.where(keep[:, 1], gk64.gather(1, idx[:, 1:])[:, 0], torch.zeros(S, dtype=f64, device=dev))
    ssum = a + b
    lterm = (g_laux * E * counts.to(f64) / S / S)[None].expand(S, E)
    clamp = ssum <= eps                                          # torch.clamp(min=eps): zero derivative of the sum below eps
    inv2 = 1.0 / (ssum * ssum).clamp(min=1e-300)
    da = torch.where(clamp, dwk[:, 0] / eps, (dwk[:, 0] - dwk[:, 1]) * b * inv2)
    db = torch.where(clamp, dwk[:, 1] / eps, (dwk[:, 1] - dwk[:, 0]) * a * inv2)
    da, db = da * keep[:, 0], db * keep[:, 1]
    rterm = torch.zeros(S, E, dtype=f64, device=dev)
    rterm.scatter_add_(1, idx[:, :1], da[:, None])
    rterm.scatter_add_(1, idx[:, 1:], db[:, None])
    dg = lterm + rterm
    D = lterm.abs() + rterm.abs()
    dot = (gk64 * dg).sum(1, keepdim=True)
    dl = gk64 * (dg - dot)
    u = 2.0 ** -24
    dl_tol = gk64 * (16 * u * D + (gk64 * (16 * u * D + E * u * dg.abs())).sum(1, keepdim=True)) + 2 * u * dl.abs() + 2.0 ** -140
    own["dlogits"] = dl
    out["dlogits"] = (dl, dl_tol)
    # ---- dx = dxp[r1] + dxp[r2] + dlogits wg ;  dwg += dlogits^T x
    dxpk, dlk = src("dxp"), src("dlogits").to(f64)
    gate_term = dlk @ wg64
    maj = dlk.abs() @ wg64.abs()
    dx = gate_term.clone()
    for c in range(2):
        m = keep[:, c]
        v = dxpk[row[m, c]].to(f64)
        dx[m] += v
        maj[m] += v.abs()
    own["dx"] = dx
    out["dx"] = (dx, 2.0 ** -8 * dx.abs() + (1 + 2.0 ** -8) * (E + 2) * u * maj)
    out["dx_gate"] = gate_term
    o_wg = olds["wg"].to(dev, f64) if "wg" in olds else torch.zeros(E, H, dtype=f64, device=dev)
    dwg = o_wg + dlk.t() @ x64
    out["g_wg"] = (dwg, (-(-S // 32) + 34) * u * (dlk.abs().t() @ x64.abs() + o_wg.abs()))
    return out


def check_moe(name, got, want, tol=None, report=None, rows=None):
    """One stage of moe_reference_fp64: bit for bit when tol is None, else element-wise |got - want| <= tol.  rows (optional) restricts the
    comparison to a bool mask or index of the first dimension (the routed rows of an expert-row tensor).  On failure names the worst
    element by (token or expert row, column), the count out of bound and max(err / bound).  Returns max(err / bound) (0 for exact stages);
    `report`, a dict, collects it under `name`."""
    if rows is not None:
        got, want = got[rows], want[rows]
        tol = None if tol is None else tol[rows]
    if tol is None:
        g, w = got.detach().to(want.device), want
        assert g.dtype == w.dtype and g.shape == w.shape, (name, g.dtype, w.dtype, g.shape, w.shape)
        bad = g.view(torch.int16 if g.element_size() == 2 else torch.int32) != w.view(torch.int16 if w.element_size() == 2 else torch.int32) \
            if g.is_floating_point() else g != w
        nbad = int(bad.sum())
        if nbad:
            i = tuple(int(t) for t in torch.nonzero(bad)[0])
            raise AssertionError(f"{name}: {nbad} / {g.numel()} elements differ in bits; first at {i}: got {g[i].item()!r} want {w[i].item()!r}")
        if report is not None:
            report.setdefault(name, 0.0)
        return 0.0
    got = got.detach().to(want.device, torch.float64)
    want, tol = want.to(torch.float64), tol.to(torch.float64)
    err = (got - want).abs()
    ratio = (err / tol).nan_to_num(float("inf"), float("inf"), 0.0)   # a NaN in got counts as out of bound; 0/0 is in bound
    ratio = torch.where(err == 0, torch.zeros_like(ratio), ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if report is not None:
        report[name] = max(worst, report.get(name, 0.0))
    nbad = int((~(err <= tol)).sum())
    if nbad:
        i = int(ratio.reshape(-1).argmax())
        where = tuple(int(t) for t in torch.unravel_index(torch.tensor(i), ratio.shape))
        g, w, t = got.reshape(-1)[i].item(), want.reshape(-1)[i].item(), tol.reshape(-1)[i].item()
        raise AssertionError(f"{name}: {nbad} / {got.numel()} elements out of bound, max err/bound {worst:.3g}; worst at (row, col) {where}: "
                             f"got {g!r} want {w!r} bound {t:.3g}")
    return worst


# ---------------------------------------------------------------------------------------------------
# norm / rotary / activation / splice / embedding-gradient / optimizer kernels (csrc/elementwise.cu, csrc/optim.cu): float64 references
# ---------------------------------------------------------------------------------------------------
# Each reference states the formula of the kernel (include/lmod.h), keeps the bf16 roundings the reference model materialises and computes
# the rest in float64.  Stages are checked from the kernel's own previous stage (y from the kernel's rstd), so a rounding that flips because
# of an fp32 input does not need a loose bound.  u = 2^-8 is the unit roundoff of bf16, 2^-24 that of fp32; a bound "u |ref| + (1 + u) E"
# is the bf16 store of a value the kernel computed in fp32 with error at most E.  A chain of n fp32 additions of terms t (in any order)
# is off by at most n 2^-24 sum|t|.  Every kernel of these files reduces a row with one CTA of 128 threads: H / 128 terms per thread, then
# block_sum (5 shuffle levels, a shared-memory hop, 5 more levels), so a row reduction is a chain of at most H / 128 + 11 additions.
BF16_U = 2.0 ** -8
FP32_U = 2.0 ** -24
ELEM_ABS_FLOOR = 2.0 ** -100          # fp32 flushes / __expf overflow (silu(g) = -0 below g = -88.7) move nothing by more than ~2^-120


def bf16_of(t):
    """Round to bf16 the way the kernels do (fp32 value, round to nearest even) and return float64."""
    return t.float().to(torch.bfloat16).to(torch.float64)


def _row_chain(H):
    return H / 128 + 11


def rmsnorm_reference_fp64(x, w, eps, res=None, rstd_k=None):
    """lmod_rmsnorm_fwd:  s = bf16(x + res) (or x),  rstd = 1 / sqrt(mean(s^2) + eps),  y = bf16(w * bf16(s * rstd)).
    Returns s (bf16, bit exact), rstd (float64) with rstd_tol, and y (bf16) computed from rstd_k, the kernel's fp32 rstd (the fp32
    product s * rstd_k rounded to bf16, times w -- exact in fp32 -- rounded again: bit exact), or from float32(rstd) without it.
      rstd_tol: the sum of squares is a chain of H / 128 + 11 fmas (relative (H/128 + 11) 2^-24, all terms positive), the division by H and
      the + eps one rounding each, rsqrtf at most 2 ulp (2^-22): relative 0.5 (H/128 + 13) 2^-24 + 2^-22."""
    s = x if res is None else (x.float() + res.float()).to(torch.bfloat16)
    H = s.shape[-1]
    s64 = s.double()
    rstd = torch.rsqrt((s64 * s64).mean(-1) + eps)
    rstd_tol = (0.5 * (_row_chain(H) + 2) * FP32_U + 2.0 ** -22) * rstd
    r32 = (rstd_k if rstd_k is not None else rstd).float()
    y = (w.float() * (s.float() * r32[..., None]).to(torch.bfloat16).float()).to(torch.bfloat16)
    return dict(s=s, rstd=rstd, rstd_tol=rstd_tol, y=y)


def rmsnorm_bwd_reference_fp64(dy, s, w, rstd_k, dres=None):
    """lmod_rmsnorm_bwd from the kernel's rstd:  g = dy w,  xhat = s rstd,  dx = rstd (g - xhat mean(g xhat)) (+ dres).
    The kernel keeps g in fp32; the reference model's autograd rounds it to bf16 first (the weight multiply is a bf16 op).
      tol:     the fp32 arithmetic.  g and xhat are one product each (2^-24 relative); dot = sum(g xhat) / H is a chain of H/128 + 11 fmas over
               terms |g xhat| plus the division; xhat dot and the difference, the product by rstd and the + dres are 4 more roundings:
                 E = 2^-24 (4 rstd |g| + rstd^2 |s| (6 |dot| + (H/128 + 13) sum|g xhat| / H) + |ref|)
      tol_g:   what the reference model's bf16(dy w) adds on top: |delta g| <= u |g| moves dx by rstd (u |g| + |xhat| mean(u |g xhat|))."""
    H = s.shape[-1]
    r = rstd_k.double()[..., None]
    g = dy.double() * w.double()
    xh = s.double() * r
    dot = (g * xh).mean(-1, keepdim=True)
    adot = (g * xh).abs().mean(-1, keepdim=True)
    dx = r * (g - xh * dot)
    if dres is not None:
        dx = dx + dres.double()
    E = FP32_U * (4 * r * g.abs() + r * r * s.double().abs() * (6 * dot.abs() + (_row_chain(H) + 2) * adot) + dx.abs())
    tol = BF16_U * dx.abs() + (1 + BF16_U) * E + ELEM_ABS_FLOOR
    tol_g = r * BF16_U * (g.abs() + xh.abs() * adot)
    return dict(dx=dx, tol=tol, tol_g=tol_g)


def accumulate_tol(old, S, e):
    """Bound of grad = bf16(fp32(old + bf16(S'))) against the exact old + S, where the kernel's fp32 sum S' is within e of S:
    |bf16(S') - S| <= u |S| + (1 + u) e;  the fp32 add and the bf16 rounding of old + bf16(S') add (u + 2^-24) |old + bf16(S')|."""
    return (BF16_U + FP32_U) * (old + S).abs() + (1 + 2 * BF16_U) * (BF16_U * S.abs() + (1 + BF16_U) * e) + ELEM_ABS_FLOOR


def bias_grad_reference_fp64(dy, old):
    """The bias gradient of kernels.LinearFn / QKVRopeFn:  bgrad = bf16(old + bf16(S')),  S' = dy.sum(0), torch's fp32 column sum of the
    bf16 rows dy [M, N] rounded to bf16 once, then `bgrad.add_` (one fp32 add of two bf16 values, rounded to bf16).
      torch's reduction kernel picks its own order (a chain per thread, then a tree over threads and blocks).  In any order each term goes
      through at most M - 1 fp32 additions, so |S' - S| <= gamma_{M-1} sum_r |dy_r|, gamma_n = n 2^-24 / (1 - n 2^-24) <= M 2^-24 for
      M <= 4096 (M (M - 1) <= 2^24).  accumulate_tol adds the two bf16 roundings.
    Returns want = old + S and tol, float64 [N]."""
    d = dy.double()
    M = d.shape[0]
    assert M <= 4096, "the first-order chain bound below holds for M <= 4096"
    S = d.sum(0)
    o = old.double()
    return dict(want=o + S, tol=accumulate_tol(o, S, M * FP32_U * d.abs().sum(0)))


def qkv_rope_reference_fp64(x, w, bias, cos, sin, pos, nh, nkv, hd, K_red):
    """lmod_gemm_qkv_rope (and GEMM + lmod_rope, which it equals bit for bit) on x [M, K] bf16, w [N, K], bias [N] or None:
    P = x W^T + b in float64; the q and k heads rotated, Y1 = P1 c - P2 s, Y2 = P2 c + P1 s (c, s the bf16 table rows of pos, P1 / P2 the
    two halves of a head); the v heads Y = P.  The GEMM's bf16 p is within E = _gemm_tol(P, |x||W|^T + |b|, K_red) of P; the rotation is
    y1 = bf16(bf16(p1 c) + bf16(-p2 s)) (y2 alike):
      |p1 c - P1 c| <= |c| E1; rounding p1 c adds u |p1 c| <= u (|P1 c| + |c| E1), the same for p2 s, so before the last rounding the error
      is E' = (1 + u)(|c| E1 + |s| E2) + u (|P1 c| + |P2 s|); the last rounding adds u (|Y1| + E'):
        tol = u |Y| + (1 + u) E'.
    Returns (want, tol), float64 [M, N]."""
    x64, w64 = x.double(), w.double()
    P = x64 @ w64.t()
    maj = x64.abs() @ w64.abs().t()
    if bias is not None:
        P, maj = P + bias.double(), maj + bias.double().abs()
    return rope_of_product_fp64(P, _gemm_tol(P, maj, K_red), cos, sin, pos, nh, nkv, hd)


def rope_of_product_fp64(P, E, cos, sin, pos, nh, nkv, hd):
    """The rotation of qkv_rope_reference_fp64 on a given float64 product P [M, N] whose bf16 kernel value is within E of it (the bf16 GEMM
    there, the e4m3 GEMM of lmod_gemm_e4m3_qkv_rope in tests/decoder_oracle.py).  Returns (want, tol), float64 [M, N]."""
    M = P.shape[0]
    nr = nh + nkv
    h = hd // 2
    p = P[:, :nr * hd].view(M, nr, hd)
    e = E[:, :nr * hd].view(M, nr, hd)
    c, s = cos[pos].double()[:, None, :h], sin[pos].double()[:, None, :h]
    p1, p2, e1, e2 = p[..., :h], p[..., h:], e[..., :h], e[..., h:]
    Y = torch.cat([p1 * c - p2 * s, p2 * c + p1 * s], -1)
    Ep = torch.cat([(1 + BF16_U) * (c.abs() * e1 + s.abs() * e2) + BF16_U * ((p1 * c).abs() + (p2 * s).abs()),
                    (1 + BF16_U) * (c.abs() * e2 + s.abs() * e1) + BF16_U * ((p2 * c).abs() + (p1 * s).abs())], -1)
    tol = BF16_U * Y.abs() + (1 + BF16_U) * Ep + ELEM_ABS_FLOOR
    want, tl = P.clone(), E.clone()
    want[:, :nr * hd] = Y.reshape(M, -1)
    tl[:, :nr * hd] = tol.reshape(M, -1)
    return want, tl


def rmsnorm_wgrad_reference_fp64(dy, s, rstd_k, old):
    """lmod_rmsnorm_wgrad:  wgrad = bf16(old + bf16(sum_r t_r)),  t_r = bf16(dy_r * bf16(s_r * rstd_r)) (autograd of `w * h.to(bf16)`).
    The terms are bit exact in fp32 from the kernel's rstd; the kernel sums them in fp32: a warp walks 32 of a 256-row chunk, 8 warps are
    folded, and the chunks meet in red.add in any order -- a chain of at most min(rows, 32) + 8 + ceil(rows / 256) additions."""
    rows = s.shape[0]
    xh = (s.float() * rstd_k.float()[:, None]).to(torch.bfloat16).float()
    t = (dy.float() * xh).to(torch.bfloat16).double()
    S = t.sum(0)
    n = min(rows, 32) + 8 + -(-rows // 256)
    e = n * FP32_U * t.abs().sum(0)
    o = old.double()
    return dict(want=o + S, tol=accumulate_tol(o, S, e))


def layernorm_reference_fp64(x, w, b, eps):
    """lmod_layernorm_fwd:  y = bf16((x - mean) rstd w + b),  rstd = 1 / sqrt(mean((x - mean)^2) + eps)  (CLIP LayerNorm).
      The fp32 mean is off by e_mu <= (H/128 + 12) 2^-24 mean|x| (the chain and the division); that shifts every x - mean by e_mu and the
      variance by e_mu^2 (sum(x - mean) = 0), the variance chain is relative (H/128 + 12) 2^-24, rsqrtf 2^-22, + eps one rounding:
        rho_r = 0.5 ((H/128 + 12) 2^-24 + e_mu^2 / var) + 2^-22 + 2^-24
      y = fma((x - mean) rstd, w, b) rounds x - mean, its product by rstd and the fma:  E = rstd |w| (|x - mean| (rho_r + 3 2^-24) + e_mu)
      + 2^-24 |y|."""
    H = x.shape[-1]
    x64 = x.double()
    mu = x64.mean(-1, keepdim=True)
    d = x64 - mu
    var = (d * d).mean(-1, keepdim=True)
    r = torch.rsqrt(var + eps)
    y = d * r * w.double() + b.double()
    e_mu = (_row_chain(H) + 1) * FP32_U * x64.abs().mean(-1, keepdim=True)
    rho = 0.5 * ((_row_chain(H) + 1) * FP32_U + e_mu * e_mu / (var + eps)) + 2.0 ** -22 + FP32_U
    E = r * w.double().abs() * (d.abs() * (rho + 3 * FP32_U) + e_mu) + FP32_U * y.abs()
    return dict(y=y, tol=BF16_U * y.abs() + (1 + BF16_U) * E + ELEM_ABS_FLOOR)


def rope_bwd_reference_fp64(dq, cos, sin, pos, hd):
    """Backward of lmod_rope (the transpose rotation) on a [rows, n_heads * hd] block of heads:  d1' = d1 c + d2 s,  d2' = d2 c - d1 s
    with c, s the bf16 table rows of pos.  The kernel computes each in fp32 (two products and an add, or an fma) and stores bf16 once:
      tol = u |ref| + (1 + u) 2 2^-24 (|d1 c| + |d2 s|).
    tol_ag bounds the distance to autograd of R.apply_rope in bf16, which rounds d c, d s and their sum to bf16: one ulp (2^-7 relative)
    of |d1 c| + |d2 s|."""
    rows = dq.shape[0]
    x = dq.double().view(rows, -1, hd)
    c = cos[pos].double()[:, None, : hd // 2]
    s_ = sin[pos].double()[:, None, : hd // 2]
    d1, d2 = x[..., : hd // 2], x[..., hd // 2:]
    o = torch.cat([d1 * c + d2 * s_, d2 * c - d1 * s_], -1)
    mag = (d1 * c).abs() + (d2 * s_).abs()
    mag = torch.cat([mag, (d2 * c).abs() + (d1 * s_).abs()], -1)
    tol = BF16_U * o.abs() + (1 + BF16_U) * 2 * FP32_U * mag + ELEM_ABS_FLOOR
    return dict(d=o.reshape(rows, -1), tol=tol.reshape(rows, -1), tol_ag=(2.0 ** -7 * mag + ELEM_ABS_FLOOR).reshape(rows, -1))


def _sig_rel(z):
    """Relative error bound of the kernels' fp32 sigmoid 1 / (1 + __expf(-z)): __expf is ex2.approx of the fp32 product z log2e (2 ulp +
    |z| 2^-24 in the exponent), then an add and an IEEE division:  (|z| + 8) 2^-22."""
    return (z.abs() + 8) * 2.0 ** -22


def silu_mul_reference_fp64(gu, I):
    """lmod_silu_mul_fwd / _bwd on [rows, >= 2I] gate | up (row stride = gu's):  out = bf16(bf16(silu(g)) u);
    dg = d u sg (1 + g (1 - sg)),  du = d g sg,  sg = sigmoid(g).
      fwd tol: |u| (u |silu| + (1 + u) |silu| rho),  rho = _sig_rel(g) (silu = g sg, one more product)
      bwd tol: the fp32 sg carries sg rho; 1 - sg, g (1 - sg) and the products add 2^-24 terms:  E = |d u| sg (1 + |g|) (|g| + 8) 2^-21,
               E = |d g| sg (|g| + 8) 2^-21 for du."""
    g, u = gu[:, :I].double(), gu[:, I:2 * I].double()
    sg = torch.sigmoid(g)
    si = g * sg
    rho = _sig_rel(g) + FP32_U
    out = si * u
    out_tol = BF16_U * out.abs() + (1 + BF16_U) * u.abs() * si.abs() * (BF16_U + (1 + BF16_U) * rho) + ELEM_ABS_FLOOR

    def bwd(d):
        d = d.double()
        dg = d * u * sg * (1 + g * (1 - sg))
        du = d * g * sg
        Eg = (d * u).abs() * sg * (1 + g.abs()) * (g.abs() + 8) * 2.0 ** -21
        Eu = (d * g).abs() * sg * (g.abs() + 8) * 2.0 ** -21
        return dict(dg=dg, du=du, dg_tol=BF16_U * dg.abs() + (1 + BF16_U) * Eg + ELEM_ABS_FLOOR,
                    du_tol=BF16_U * du.abs() + (1 + BF16_U) * Eu + ELEM_ABS_FLOOR)
    return dict(out=out, out_tol=out_tol, bwd=bwd)


ACT_GELU_REF, ACT_QUICK_GELU_REF, ACT_NONE_REF = 0, 1, 2


def bias_act_reference_fp64(x, bias, act):
    """lmod_bias_act_fwd:  y = bf16(act(bf16(x + bias))) (the bias add is one bf16 op, bit exact in fp32; the CLIP fc1 bias path).
      GELU (erf):    0.5 z (1 + erf(z / sqrt2)); erff is within 2 ulp (2^-23 absolute near |erf| = 1, where 1 + erf cancels), the argument
                     product shifts erf by at most 2^-24: E = 0.5 |z| 2^-22 + 2^-23 |y|
      quick-GELU:    z sigmoid(1.702 z):  E = |y| (_sig_rel(1.702 z) + 2^-23)
      identity:      exact."""
    z = x.float()
    if bias is not None:
        z = (z + bias.float()).to(torch.bfloat16).float()
    z = z.double()
    if act == ACT_GELU_REF:
        y = 0.5 * z * (1 + torch.erf(z / math.sqrt(2)))
        E = 0.5 * z.abs() * 2.0 ** -22 + 2.0 ** -23 * y.abs()
    elif act == ACT_QUICK_GELU_REF:
        y = z * torch.sigmoid(1.702 * z)
        E = y.abs() * (_sig_rel(1.702 * z) + 2.0 ** -23)
    else:
        y, E = z, torch.zeros_like(z)
    return dict(y=y, tol=BF16_U * y.abs() + (1 + BF16_U) * E + ELEM_ABS_FLOOR)


def gelu_bwd_reference_fp64(dy, x):
    """lmod_gelu_bwd:  dx = dy (cdf(x) + x pdf(x)).  cdf via erff (2^-22 absolute with the argument product), pdf via __expf(-x^2 / 2)
    (relative _sig_rel(x^2 / 2)), three more roundings:  E = |dy| (2^-22 + |x| pdf (_sig_rel(x^2/2) + 2^-24) + 3 2^-24 (cdf + |x| pdf))."""
    x64, d = x.double(), dy.double()
    cdf = 0.5 * (1 + torch.erf(x64 / math.sqrt(2)))
    pdf = torch.exp(-0.5 * x64 * x64) / math.sqrt(2 * math.pi)
    ref = d * (cdf + x64 * pdf)
    xp = x64.abs() * pdf
    E = d.abs() * (2.0 ** -22 + xp * (_sig_rel(0.5 * x64 * x64) + FP32_U) + 3 * FP32_U * (cdf + xp))
    return dict(dx=ref, tol=BF16_U * ref.abs() + (1 + BF16_U) * E + ELEM_ABS_FLOOR)


def embed_grad_reference_fp64(dout, src, old):
    """lmod_embed_grad (nn.Embedding backward behind the splice, then the bf16 accumulation into .grad):  for every token t with rows
    R_t = {r : src[r] = t},  grad[t] = bf16(old[t] + bf16(sum_{r in R_t} dout[r]));  rows with src < 0 (image patches, padding) add nothing.
    The kernel sums a token's n_t rows in one fp32 chain: e = n_t 2^-24 sum|dout| (accumulate_tol).
    Returns the touched token ids (sorted), want = old + S and tol for their rows [U, H], and the counts n_t."""
    flat = src.reshape(-1)
    keep = flat >= 0
    rows = torch.nonzero(keep)[:, 0]
    toks, inv, cnt = torch.unique(flat[keep], return_inverse=True, return_counts=True)
    H = dout.shape[-1]
    d = dout.reshape(-1, H)[rows].double()
    S = torch.zeros(toks.numel(), H, dtype=torch.float64, device=dout.device).index_add_(0, inv, d)
    A = torch.zeros_like(S).index_add_(0, inv, d.abs())
    o = old[toks].double()
    return dict(toks=toks, counts=cnt, want=o + S, tol=accumulate_tol(o, S, cnt.double()[:, None] * FP32_U * A))


def splice_reference(embed_w, feats, src, img, n_patches):
    """lmod_splice_embed: row r is embed_w[src] (src >= 0), feats[img, -1 - src] (src < 0, img >= 0) or zero -- a copy, bit exact."""
    flat, im = src.reshape(-1), img.reshape(-1)
    H = embed_w.shape[1]
    out = torch.zeros(flat.numel(), H, dtype=embed_w.dtype, device=embed_w.device)
    t = flat >= 0
    out[t] = embed_w[flat[t]]
    f = (flat < 0) & (im >= 0)
    out[f] = feats.reshape(-1, H)[im[f] * n_patches + (-1 - flat[f])]
    return out


def splice_bwd_reference(dout, src, img, n_img, n_patches):
    """lmod_splice_embed_bwd: dfeats[img, -1 - src] = dout[r] for the image rows (each feature row is spliced once), zero elsewhere."""
    flat, im = src.reshape(-1), img.reshape(-1)
    H = dout.shape[-1]
    d = torch.zeros(n_img * n_patches, H, dtype=dout.dtype, device=dout.device)
    f = (flat < 0) & (im >= 0)
    d[im[f] * n_patches + (-1 - flat[f])] = dout.reshape(-1, H)[f]
    return d.view(n_img, n_patches, H)


def sumsq_reference_fp64(g, chunk=1 << 27):
    """sum(g^2) in float64, in chunks (a 10^9-element buffer)."""
    flat = g.reshape(-1)
    tot = 0.0
    for i in range(0, flat.numel(), chunk):
        c = flat[i:i + chunk].double()
        tot += float((c * c).sum())
    return tot


def sumsq_chain(n, blocks):
    """Length of lmod_sumsq's fp32 chain: each of the 256 threads of `blocks` CTAs adds ceil(n / (blocks 256)) squares (one fma each; the
    bf16 path rounds up to whole vectors of 8 and a tail), block_sum (11), the last CTA adds ceil(blocks / 256) partials per thread,
    block_sum again (11) and the add into out."""
    return -(-n // (blocks * 256)) + 8 + -(-blocks // 256) + 23


def sumsq_blocks(n, n_sms):
    """The grid of lmod_sumsq: one CTA per 2048 elements, capped at 8 CTAs per SM (and at 4096)."""
    return max(1, min((n // 8 + 255) // 256, n_sms * 8, 4096))


def adamw_reference_fp64(master, m, v, grad, step, lr, beta1, beta2, eps, wd, gnorm_sq=None, max_norm=0.0, grad_scale=1.0,
                         bias_correction=True, fp32_hyper=True):
    """lmod_adamw (torch.optim.AdamW with clip_grad_norm_ folded into a scalar) in float64 on the fp32 inputs, with the hyperparameters as
    the fp32 values the kernel receives:
      coef = grad_scale min(1, max_norm / (sqrt(gnorm_sq) grad_scale + 1e-6))  (no clipping when gnorm_sq is None or max_norm = 0)
      g = grad coef;  p' = p (1 - lr wd);  m' = b1 m + (1 - b1) g;  v' = b2 v + (1 - b2) g^2
      p'' = p' - (lr / bc1) m' / (sqrt(v') / sqrt(bc2) + eps),  bc_i = 1 - b_i^step.
    Bounds (the kernel's fp32 arithmetic; IEEE sqrtf and division):
      coef: sqrtf, two products, an add, a division, fminf: relative rho_c = 6 2^-24;  g = grad coef: rho_g = rho_c + 2^-24
      m: E_m = 3 2^-24 (|b1 m| + |(1 - b1) g|) + (1 - b1) |g| rho_g
      v: E_v = 4 2^-24 (b2 v + (1 - b2) g^2) + 2 rho_g (1 - b2) g^2
      denom: relative rho_d = E_v / (2 v') + 5 2^-24 (sqrtf, bc2_sqrt rounded to fp32, the division, the + eps)
      p: E_p = 3 2^-24 |p'| + (lr / bc1) / denom (E_m + |m'| (rho_d + 4 2^-24)) + 2^-24 |p''|   (1 - lr wd, lr / bc1 with bc1 in fp32,
         m / denom, the product, the difference).
    bias_correction=False drops bc1 and bc2 (a planted defect for the tests of the bound).  fp32_hyper=False takes the hyperparameters as
    the Python floats torch.optim.AdamW uses (1 - beta2 formed in double): the kernel's 1 - fp32(0.999) differs from fp32(0.001) by
    1.3e-5 relative, a deviation of the second-moment increment that the oracle pin must not mistake for arithmetic error."""
    f = (lambda a: float(torch.tensor(a, dtype=torch.float32))) if fp32_hyper else float    # noqa: E731  the value the kernel receives
    lr, b1, b2, eps, wd, mn, gs = f(lr), f(beta1), f(beta2), f(eps), f(wd), f(max_norm), f(grad_scale)
    coef = gs
    if gnorm_sq is not None and mn > 0:
        total = math.sqrt(float(gnorm_sq)) * gs
        coef = gs * min(1.0, mn / (total + f(1e-6)))
    u = FP32_U
    rho_g = 7 * u
    g = grad.double() * coef
    p0, m0, v0 = master.double(), m.double(), v.double()
    bc1 = 1 - b1 ** step if bias_correction else 1.0
    bc2 = 1 - b2 ** step if bias_correction else 1.0
    p1 = p0 * (1 - lr * wd)
    m1 = b1 * m0 + (1 - b1) * g
    v1 = b2 * v0 + (1 - b2) * g * g
    den = torch.sqrt(v1) / math.sqrt(bc2) + eps
    p2 = p1 - (lr / bc1) * m1 / den
    E_m = 3 * u * ((b1 * m0).abs() + ((1 - b1) * g).abs()) + (1 - b1) * g.abs() * rho_g
    E_v = 4 * u * (b2 * v0 + (1 - b2) * g * g) + 2 * rho_g * (1 - b2) * g * g
    rho_d = torch.where(v1 > 0, E_v / (2 * v1), torch.zeros_like(v1)) + 5 * u
    E_p = 3 * u * p1.abs() + (lr / bc1) / den * (E_m + m1.abs() * (rho_d + 4 * u)) + u * p2.abs()
    return dict(master=p2, m=m1, v=v1, master_tol=E_p + ELEM_ABS_FLOOR, m_tol=E_m + ELEM_ABS_FLOOR, v_tol=E_v + ELEM_ABS_FLOOR, coef=coef)


def check_bound(name, got, want, tol=None, report=None):
    """Element-wise |got - want| <= tol (bit for bit when tol is None) with a message naming the worst element; see check_moe."""
    return check_moe(name, got, want, tol, report)


def moe_plan_pairs(S, E, n1, n2, seed=0):
    """[S, 2] (first, second) expert of every token with n1[e] first and n2[e] second choices, first != second, in a seeded order."""
    g = torch.Generator().manual_seed(seed)
    assert sum(n1) == S and sum(n2) == S
    e1 = torch.cat([torch.full((n,), e, dtype=torch.long) for e, n in enumerate(n1)])[torch.randperm(S, generator=g)]
    left = list(n2)
    e2 = torch.empty(S, dtype=torch.long)
    done = []
    for s in torch.randperm(S, generator=g).tolist():          # the expert with the most second choices left, other than the first
        c = max((e for e in range(E) if e != int(e1[s]) and left[e] > 0), key=lambda e: left[e], default=None)
        if c is None:                                          # only the token's own first choice is left: trade with a placed token
            c = int(e1[s])
            t = next((t for t in done if int(e2[t]) != c and int(e1[t]) != c), None)
            assert t is not None, "moe_plan_pairs: counts cannot be met with first != second"
            e2[s], e2[t] = e2[t].clone(), c
        else:
            e2[s] = c
        left[c] -= 1
        done.append(s)
    return torch.stack([e1, e2], 1)


def moe_planted_inputs(pairs, E, H, specials=(), seed=0, x_scale=1.0):
    """Inputs whose routing is exactly `pairs` [S, 2] (first, second expert per token).  Column e < E of x carries the token's first
    choice: x[s, e1] in [0.75, 1.25], wg[e, e] = 4, so logit e1 leads the random part (x[:, 16:] . wg[:, 16:], std about 0.3) by a clear
    margin; the noise adds 10 to the second choice.  specials: (token, logits, noise) rows planted exactly: x[s] is one-hot in a column
    of its own (16 - E > index), wg's column holds the logits (fp32, so the kernel's GEMV gives them bit for bit), noise[s] = noise.
    Returns x [S, H] bf16, wg [E, H] fp32, noise [S, E] fp32 (CPU)."""
    S = pairs.shape[0]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(S, H, generator=g) * x_scale
    x[:, :16] = 0
    x[torch.arange(S), pairs[:, 0]] = 0.75 + 0.5 * torch.rand(S, generator=g)
    wg = torch.randn(E, H, generator=g) * (0.3 / math.sqrt(H - 16) / x_scale)
    wg[:, :16] = 0
    wg[torch.arange(E), torch.arange(E)] = 4.0
    noise = torch.zeros(S, E)
    noise[torch.arange(S), pairs[:, 1]] = 10.0
    for i, (s, logits, nz) in enumerate(specials):
        col = E + i
        assert col < 16
        x[s] = 0
        x[s, col] = 1
        wg[:, col] = torch.as_tensor(logits, dtype=torch.float32)
        noise[s] = torch.as_tensor(nz, dtype=torch.float32)
    return x.to(torch.bfloat16), wg.contiguous(), noise


def moe_special_rows(E, S, clamp_to=None):
    """The planted routing edges (token, logits, noise, expected (first, second), what) on tokens S-1, S-2 (late: their first choice,
    expert 0, has overflowed; pairs must give them first choice 0) and tokens 0, 1, 2 (early):
      equal logits -> first choice 0, second choice a tie of logits + noise between experts 1 and 2 -> 1;
      1-ulp near tie at |logit| ~ 0.1 (gates tie, logits do not) -> first choice 0;
      a tie in logits + noise for the second choice with distinct logits;
      late: first choice dropped, second (clamp_to, default E-1) kept with a gate below FLT_EPSILON (clamped renormalisation);
      late: both choices dropped (second choice 1, which must be full by then)."""
    ct = E - 1 if clamp_to is None else clamp_to
    f = torch.tensor
    nt = float(torch.nextafter(f(0.1, dtype=torch.float32), f(1.0, dtype=torch.float32)))
    pad = lambda v, fill: (list(v) + [fill] * E)[:E]             # noqa: E731
    rows = [
        (0, [0.5] * E, pad([0.0, 3.0, 3.0], 0.0), (0, 1), "equal logits"),
        (1, pad([0.1, nt], -1.0) if E == 2 else pad([0.1, nt, -1.0, -2.0], -2.5), pad([0.0, 0.0, 10.0], 0.0) if E > 2 else [0.0, 0.0],
         (0, 2) if E > 2 else (0, 1), "1-ulp near tie"),
        (2, pad([1.0, 0.5, 0.25], -1.0), pad([0.0, 1.0, 1.25], 0.0) if E > 2 else [0.0, 1.0], (0, 1), "tie in logits + noise"),
        (S - 2, [8.0] + [-8.2 if e == ct else -9.0 for e in range(1, E)], [10.0 if e == ct else 0.0 for e in range(E)], (0, ct),
         "dropped first, clamped second"),
        (S - 1, pad([3.0, 1.0], -1.0), pad([0.0, 10.0], 0.0), (0, 1), "both dropped"),
    ]
    return rows


def moe_force_pairs(pairs, rows):
    """Give the special tokens their (first, second) pair by swapping with a token that has it (the counts stay as planned)."""
    pairs = pairs.clone()
    fixed = set()
    for s, _, _, want, _ in rows:
        want = torch.tensor(want)
        if not torch.equal(pairs[s], want):
            cand = [t for t in torch.nonzero((pairs == want).all(1))[:, 0].tolist() if t not in fixed and t != s]
            assert cand, ("moe_force_pairs: no token has the pair", tuple(want.tolist()))
            t = cand[0]
            pairs[[s, t]] = pairs[[t, s]]
        fixed.add(s)
    return pairs


def moe_run_stages(x, res, wg, w_gu, w_dn, noise, cf, mc, dout, g_laux, old):
    """kernels.moe_forward_stages + moe_backward_stages with weight gradients accumulated into copies of `old`; one dict of every
    intermediate, the gradients under 'g_wg', 'g_w_gu', 'g_w_dn'."""
    from llavamod import kernels as K
    grads = {k: v.clone() for k, v in old.items()}
    st = K.moe_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, mc)
    bw = K.moe_backward_stages(st, x, wg, w_gu, w_dn, dout, torch.tensor(g_laux, device="cuda"), grads)
    k = {**st, **bw, **{"g_" + n: v for n, v in grads.items()}}
    return k


def check_moe_stages(k, ref, E, old, report=None, backward=True):
    """Every stage of moe_run_stages against moe_reference_fp64(..., k=k): the routing record bit for bit, then each stage's bound.
    backward=False: the forward stages only (k from kernels.moe_forward_stages, ref without dout)."""
    rec = ref["rec"]
    n_rows = int(rec["offsets"][-1])
    assert torch.equal(k["idx"].long(), rec["idx"]), "routing record (first / second expert)"
    assert torch.equal(k["row"].long(), rec["row"]), "routing record (rows: slots and drops)"
    assert torch.equal(k["offsets"].long(), rec["offsets"])
    assert k["capacity"] == rec["capacity"] and int(k["meta"][1]) == rec["capacity"]
    assert torch.equal(k["meta"][4:4 + E].long(), rec["counts"])
    routed = rec["tok"] >= 0
    pad = ~routed
    for name in ("logits", "gates") + (("dw", "dlogits", "dx") if backward else ()):
        check_moe(name, k[name], *ref[name], report=report)
    check_moe("w", k["w"], ref["w"][0], None, report)
    la_want, la_tol = ref["l_aux"]
    assert abs(float(k["meta"][0]) - float(la_want)) <= float(la_tol), ("l_aux", float(k["meta"][0]), float(la_want))
    check_moe("xp", k["xp"][:n_rows], ref["xp"][0], None, report)
    for name in ("h1", "act", "y") + (("dh1", "dxp", "dact") if backward else ()):
        check_moe(name, k[name][:n_rows], *ref[name], report=report, rows=routed)
        if name in ("h1", "act", "y"):                           # padding rows below offsets[E] are exact zeros
            assert int(k[name][:n_rows][pad].ne(0).sum()) == 0, f"{name}: non-zero padding row"
    check_moe("out", k["out"], ref["out"][0], None, report)
    if not backward:
        return
    check_moe("dy", k["dy"][:n_rows], ref["dy"][0], None, report)
    assert int(k["dy"][n_rows:].ne(0).sum()) == 0
    check_moe("g_wg", k["g_wg"], *ref["g_wg"], report=report)
    for gname in ("w_gu", "w_dn"):
        check_moe("g_" + gname, k["g_" + gname], *ref["g_" + gname], report=report)
        for e in range(E):
            if int(rec["used"][e]) == 0:                       # an expert without rows leaves its pre-filled gradient untouched
                check_moe(f"g_{gname}[{e}] (empty expert)", k["g_" + gname][e], old[gname][e], None)


# ---------------------------------------------------------------------------------------------------
# reads of memory nobody wrote
# ---------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def poisoned_uninitialised_memory():
    """Inside: every torch.empty / empty_like (and every allocation torch makes for an op's output) is filled at allocation, floats with
    NaN and integers with their largest value (torch's deterministic mode with fill_uninitialized_memory).  A kernel that reads memory
    nobody wrote then reads NaN every time, instead of whatever an earlier tensor left there.  Both settings are restored on exit."""
    import torch.utils.deterministic as det
    was_det, was_warn, was_fill = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(), \
        det.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True, warn_only=True)
    det.fill_uninitialized_memory = True
    try:
        yield
    finally:
        det.fill_uninitialized_memory = was_fill
        torch.use_deterministic_algorithms(was_det, warn_only=was_warn)


# ---------------------------------------------------------------------------------------------------
# gradient views for the exact autograd tests: one arena of sentinels, and the run-twice byte comparison
# ---------------------------------------------------------------------------------------------------
DEV = "cuda"
SENT = -12345.0                                   # bf16 -12352


def randn(*shape, seed, scale=1.0):
    """Seeded bf16 normal values on the GPU."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(torch.bfloat16)


class Arena:
    """The gradient views of one case, carved out of one flat bf16 buffer as train/engine.py _pack lays the arena out, with one ALIGN unit
    of guard in front and behind.  The views hold seeded values (what earlier micro-batches left); every other element holds SENT."""

    def __init__(self, shapes, seed, scale=0.5):
        from llavamod.train.engine import ALIGN
        offs, off = [], ALIGN
        for s in shapes:
            offs.append(off)
            off += -(-math.prod(s) // ALIGN) * ALIGN
        self.buf = torch.full((off + ALIGN,), SENT, dtype=torch.bfloat16, device=DEV)
        self.owned = torch.zeros(off + ALIGN, dtype=torch.bool, device=DEV)
        self.views = []
        for i, (o, s) in enumerate(zip(offs, shapes)):
            n = math.prod(s)
            v = self.buf[o:o + n].view(s)
            v.copy_(randn(*s, seed=seed + i, scale=scale))
            self.owned[o:o + n] = True
            self.views.append(v)
        self.fresh = self.buf.clone()

    def snapshot(self):
        return [v.clone() for v in self.views]

    def check_sentinels(self, tag):
        bad = (self.buf.view(torch.int16) != self.fresh.view(torch.int16)) & ~self.owned
        n = int(bad.sum())
        assert n == 0, f"{tag}: {n} arena elements outside the views changed; first at flat index {int(torch.nonzero(bad)[0])}"


def no_nan(tag, **ts):
    for name, t in ts.items():
        if t is not None:
            assert not bool(torch.isnan(t).any()), f"{tag}: NaN in {name}"


def same_bytes(tag, a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        iv = torch.int16 if x.element_size() == 2 else torch.int32
        assert x.shape == y.shape and torch.equal(x.view(iv), y.view(iv)), f"{tag}: output {i} differs between two identical runs"


def twice(tag, run, label="AUTOGRAD"):
    """run(report) -> list of output tensors; run(None), which checks nothing, must give the same bytes."""
    report = {}
    first = run(report)
    same_bytes(tag, first, run(None))
    worst = max(report, key=report.get)
    print(f"\n{label} {tag}: worst err/bound {report[worst]:.3g} ({worst}; {len(report)} checks)")


# ---------------------------------------------------------------------------------------------------
# kernels.DistillHeadFn (lm_head GEMM + fused KL/CE + the lm_head backward): float64 stage references
# ---------------------------------------------------------------------------------------------------
def distill_head_reference_fp64(h, W, t, labels, T, vocab, w_kd, w_ce, distill_all, g, rows=None, logits=None, dlogits=None, old=None,
                                store=torch.float64, block_rows=256, block_cols=16384):
    """Float64 restatement of kernels.DistillHeadFn, stage by stage, with the bounds of tests/helpers.py for each stage.

    h [N, H] the hidden rows, W [V_s, H] the lm_head, labels [N] flat (B = N / T sequences), g the upstream scalar of `total`, old [V_s, H]
    the lm_head gradient view before the call (zeros when None).  rows = (perm, count) as kernels.active_rows gives them: then t, logits and
    dlogits hold row perm[j] of the batch in their row j < count (the compact layout); without rows they hold every row in order.
    t [., >= vocab] are the teacher logits.  logits / dlogits [., V_s] are the kernel's stages: each stage takes its input from them when
    given, else from this reference's own previous stage (float64, unrounded).  Works on h's device in blocks.

    Returns a dict (`store` is the dtype of the [n, V_s] and [V_s, H] results):
      act          [n] the original index of every active row (KD or CE mask), ascending
      logits, logits_tol [n, V_s]   h[act] W^T and _gemm_tol(K = H)
      kl           kl_reference_fp64 of the logits (placed on their original rows) against t, over the first vocab columns
      align, ce, total              total = w_kd align + w_ce ce (w_ce = 0 drops ce, NaN included, as the Function does)
      dh, dh_tol   [N, H]  g (d W) over the first vocab columns of d = the d logits of the active rows, zero on the other rows.  The bound is
                   |g| _gemm_tol(d W, |d| |W|, K = V_s) for the GEMM (stored in bf16), then one fp32 product with g and one bf16 rounding
      dW, dW_tol   [V_s, H]  old + d^T (g h[act]) (rows vocab and above: old, exact), with _gemm_tol(K = n) + 2^-23 |ref| for the fp32 add to the
                   old value and, when g is not a power of two, 2^-8 |d|^T |g h| for the bf16 operand g h"""
    f64 = torch.float64
    dev = h.device
    N, H = h.shape
    Vs = W.shape[0]
    gs = float(g)
    labels = labels.reshape(-1).to(dev)
    m_kd, m_ce, _ = kl_row_masks(labels, T, distill_all)
    act = torch.nonzero(m_kd | m_ce)[:, 0]
    n = act.numel()
    if rows is not None:
        perm, count = rows
        assert int(count) == n and torch.equal(perm[:n].long().to(dev), act), "rows do not list the active rows"
        src = torch.arange(n, device=dev)                              # row of the compact tensors that holds act[i]
    else:
        src = act
    W64 = W.to(f64)
    W64a = W64.abs()
    h_act = h[act].to(f64)
    out = dict(act=act)

    lg = torch.zeros(n, Vs, dtype=store, device=dev)
    lt = torch.zeros_like(lg)
    for r0 in range(0, n, block_rows):
        a = h_act[r0:r0 + block_rows]
        ref = a @ W64.t()
        lg[r0:r0 + block_rows] = ref.to(store)
        lt[r0:r0 + block_rows] = _gemm_tol(ref, a.abs() @ W64a.t(), H).to(store)
        del ref
    out["logits"], out["logits_tol"] = lg, lt

    def placed(x, idx):                                                # rows idx of x on the original rows act, zero elsewhere
        full = torch.zeros(N, vocab, dtype=x.dtype, device=dev)
        full[act] = x[idx, :vocab]
        return full

    s_full = placed(logits, src) if logits is not None else placed(lg, torch.arange(n, device=dev))
    kl = kl_reference_fp64(s_full, placed(t, src), labels, T, vocab, w_kd, w_ce, distill_all, g_dtype=store)
    del s_full
    out["kl"], out["align"], out["ce"] = kl, kl["align"], kl["ce"]
    out["total"] = w_kd * kl["align"] + (w_ce * kl["ce"] if w_ce != 0.0 else 0.0)

    d = dlogits[src, :vocab] if dlogits is not None else kl["g"][act]  # [n, vocab]
    Wv, Wva = W64[:vocab], W64a[:vocab]
    dh = torch.zeros(N, H, dtype=f64, device=dev)
    dh_tol = torch.zeros_like(dh)
    for r0 in range(0, n, block_rows):
        db = d[r0:r0 + block_rows].to(f64)
        ref0 = db @ Wv
        r = act[r0:r0 + block_rows]
        dh[r] = gs * ref0
        dh_tol[r] = (1 + BF16_U) * abs(gs) * _gemm_tol(ref0, db.abs() @ Wva, Vs) + (BF16_U + FP32_U) * (gs * ref0).abs()
        del db, ref0
    out["dh"], out["dh_tol"] = dh, dh_tol

    gh = gs * h_act
    exact_scale = gs != 0.0 and math.frexp(gs)[0] == 0.5                # g h is exact in bf16
    dW = (old.to(store) if old is not None else torch.zeros(Vs, H, dtype=store, device=dev)).clone()
    dW_tol = torch.zeros_like(dW)
    for v0 in range(0, vocab, block_cols):
        v1 = min(vocab, v0 + block_cols)
        db = d[:, v0:v1].to(f64)
        o = dW[v0:v1].to(f64)
        c = db.t() @ gh
        cm = db.abs().t() @ gh.abs()
        ref = o + c
        tol = _gemm_tol(ref, o.abs() + cm, n) + 2.0 ** -23 * ref.abs()
        if not exact_scale:
            tol = tol + BF16_U * cm
        dW[v0:v1], dW_tol[v0:v1] = ref.to(store), tol.to(store)
        del db, o, c, cm, ref, tol
    out["dW"], out["dW_tol"] = dW, dW_tol
    return out
