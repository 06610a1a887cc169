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
