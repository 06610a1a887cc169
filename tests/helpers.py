"""Shared fixtures for the GPU parity tests, smoke() and bench.py: tiny config-1 models, seeded batches, and the
oracle-side evaluation of the same step."""
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
#                ex2.approx (2^-22.5) / the degree-4 polynomial of the LMOD_KL_POLY arm (3.7e-6)                                <= 3.7e-6
#              sum 1.6e-5.  The fp32 roundings of -cb*p and of the fma ca*q + (-cb*p) add at most 2^-23 (ca q + cb p), i.e. 1.2e-7 to eps;
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
