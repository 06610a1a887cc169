/* lmod.h -- C ABI of liblmod_b200.so: the H100 (sm_90a) kernels behind the LLaVA-MoD
 * distillation step.
 *
 * The reference (shufangxun/LLaVA-MoD) has NO plugin / FFI interface -- it is pure Python on
 * PyTorch (SURVEY.md section 8b).  The boundary this library replaces is therefore the set of
 * PyTorch call sites on the hot path; every entry point cites the reference lines whose GPU
 * work it takes over.  Conventions (all entry points):
 *   - plain pointers and sizes, no torch types; device pointers are BORROWED for the call;
 *   - no allocation, no host sync, no stream creation inside; work is enqueued on `stream`
 *     (a cudaStream_t passed as void*);  re-entrant across streams;
 *   - return 0 on success, negative lmod_status on error; lmod_last_error() gives a
 *     thread-local message;
 *   - bf16 tensors are row-major; `ld*` are row strides in ELEMENTS.
 */
#ifndef LMOD_H_
#define LMOD_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  LMOD_OK = 0,
  LMOD_ERR_ARG = -1,      /* bad argument (shape / alignment / null)         */
  LMOD_ERR_CUDA = -2,     /* CUDA runtime error (see lmod_last_error)        */
  LMOD_ERR_UNSUPPORTED = -3
} lmod_status;

const char* lmod_last_error(void);
int lmod_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches claim) */
int64_t lmod_launch_count(void);
void lmod_launch_count_reset(void);

/* ------------------------------------------------------------------------------------------
 * K16 + K15: fused mimic-KL (+ shifted LM cross-entropy) forward AND backward over the vocab.
 * Replaces AlignTrainer.get_p / get_logp / compute_align_loss (llavamod/train/align_trainer.py:
 * 473-475, 497-499, 509-526) and the model's shifted CE (llava_qwen1_5_moe.py:413-421).
 *   s_logits [N, ld_s] bf16 student, t_logits [N, ld_t] bf16 teacher, labels [N] int64
 *   (post-splice, row n = b*T + t).  V = vocab slice (151936).  Per row n:
 *     x_n   = sum_v p_T(v) * log q_S(v)           (0 where log q_S is +-inf)
 *     nll_n = lse_S - s[labels[n+1]]              (t < T-1 and label != -100)
 *   dlogits[n,v] = w_kd*m_n/n_kd*(q_S - p_T) + w_ce*c_n/n_ce*(q_S - onehot)  (bf16; may alias s_logits)
 *   with m_n = labels[n] != -100 (or 1 if distill_all), c_n = CE mask, counts from lmod_kl_counts.
 *   row_out [N,4] fp32 = {x_n, nll_n, lse_S, lse_T};  dlogits may be NULL (forward only).
 */
int lmod_kl_counts(const int64_t* labels, int64_t n_rows, int64_t seq_len, int distill_all,
                   float* counts2 /* {n_kd, n_ce} */, void* stream);
int lmod_kl_fwd_bwd(const void* s_logits, int64_t ld_s, const void* t_logits, int64_t ld_t,
                    const int64_t* labels, int64_t n_rows, int64_t seq_len, int64_t vocab,
                    int distill_all, float w_kd, float w_ce, const float* counts2,
                    float* row_out, void* dlogits, int64_t ld_d, void* stream);
/* Same over the batch's ACTIVE rows only (rows whose KD mask or CE mask is set; the reference computes every row and multiplies the rest
 * by zero, align_trainer.py:512-526): s_logits / t_logits / dlogits hold row j = original row perm[j] for j < *count (device scalars from
 * lmod_active_rows); labels and row_out stay indexed by the original row (row_out of inactive rows is not written and not read by
 * lmod_kl_finalize).  perm == count == NULL: identical to lmod_kl_fwd_bwd. */
int lmod_kl_fwd_bwd_rows(const void* s_logits, int64_t ld_s, const void* t_logits, int64_t ld_t,
                         const int64_t* labels, int64_t n_rows, int64_t seq_len, int64_t vocab,
                         int distill_all, float w_kd, float w_ce, const float* counts2,
                         float* row_out, void* dlogits, int64_t ld_d, const int32_t* perm, const int32_t* count, void* stream);
/* Active-row compaction for the loss head (csrc/rows.cu).  active(n) = labels[n] != -100 (or distill_all) || (n is not the last position of
 * its sequence && labels[n+1] != -100) -- the union of the KD mask (align_trainer.py:512-515) and the shifted-CE mask
 * (llava_qwen1_5_moe.py:413-421).  perm [n_rows] int32: perm[j] = original row of the j-th active row (ascending), -1 for j >= *count.
 * gather: dst[j,:] = src[perm[j],:] for j < *count (perm NULL = identity), zeros for *count <= j < round_up(*count, pad_to), rows beyond
 * untouched.  scatter: dst[perm[j],:] = src[j,:] for j < *count (dst zeroed by the caller).  All counts live in device memory: no host
 * synchronisation, usable inside a captured CUDA graph. */
int lmod_active_rows(const int64_t* labels, int64_t n_rows, int64_t seq_len, int distill_all, int32_t* perm, int32_t* count, void* stream);
int lmod_gather_rows(const void* src, int64_t ld_src, const int32_t* perm, const int32_t* count, int64_t max_rows, int64_t cols,
                     int64_t pad_to, void* dst, int64_t ld_dst, void* stream);
int lmod_scatter_rows(const void* src, int64_t ld_src, const int32_t* perm, const int32_t* count, int64_t max_rows, int64_t cols,
                      void* dst, int64_t ld_dst, void* stream);
/* reduces row_out into {align_loss, ce_loss, n_kd, n_ce} (align = -sum m x / n_kd ; 0/0 -> NaN kept,
 * align_trainer.py:526) */
int lmod_kl_finalize(const float* row_out, const int64_t* labels, int64_t n_rows, int64_t seq_len,
                     int distill_all, float* out4, void* stream);

/* ------------------------------------------------------------------------------------------
 * K17: DPO per-token log-prob gather.  Replaces DPOTrainer.get_logp (dpo_trainer.py:483-495):
 * labels shifted by one, NO vocab slice, log_softmax + gather + masked sequence sum.
 *   fwd: tok_logp [N] fp32 (0 for masked rows), lse [N] fp32, seq_logp [B] fp32
 *   bwd: dlogits[n,v] = g_seq[b]*mask_n*(onehot - q)   (bf16; may alias logits)
 */
int lmod_logp_gather_fwd(const void* logits, int64_t ld, const int64_t* labels, int64_t batch,
                         int64_t seq_len, int64_t vocab, float* tok_logp, float* lse,
                         float* seq_logp, int average, void* stream);
int lmod_logp_gather_bwd(const void* logits, int64_t ld, const int64_t* labels, int64_t batch,
                         int64_t seq_len, int64_t vocab, const float* lse, const float* g_seq,
                         int average, void* dlogits, int64_t ld_d, void* stream);

/* API-compat materialising forms of get_p / get_logp (fp32 [N,V] outputs) and compute_align_loss
 * on materialised inputs (align_trainer.py:473-528). */
int lmod_softmax_rows(const void* logits_bf16, int64_t ld, int64_t n_rows, int64_t vocab,
                      int log_mode, float* out, int64_t ld_out, void* stream);
int lmod_align_loss_dense(const float* logp, const float* probs, int64_t ld, const int64_t* labels,
                          int64_t n_rows, int64_t vocab, int distill_all, float* row_x,
                          float* out_loss, void* stream);

/* ------------------------------------------------------------------------------------------
 * K10 + K11: DeepSpeed-0.9.5 top-2 gate + capacity + token scatter in one call (two plain launches: gate, then seat+scatter).
 * Replaces deepspeed.moe.sharded_moe.TopKGate/top2gating + the dispatch einsum
 * (call site llava_qwen1_5_moe.py:536-546; SURVEY.md Appendix A steps 1-9).
 *   x [S,H] bf16, wg [E,H] fp32, noise [S,E] fp32 (Gumbel, explicit input).
 *   outputs: logits [S,E] fp32, gates [S,E] fp32, idx [S,2] int32, row [S,2] int32 (-1 = dropped),
 *            w [S,2] fp32 (normalised, 0 if dropped), offsets [E+1] int32 (row ranges per expert),
 *            meta [4+E] fp32 {l_aux, capacity, rows_total, 0, exp_counts...}, xp [2S,H] bf16 permuted.
 *   ws: lmod_moe_route_ws_elems(S, E) int32 elements of device scratch owned by this call (no initialisation needed; the
 *       two kernels of the op -- gate, then seat+scatter -- exchange per-tile expert counts through it).  Ordinary launches of
 *       ceil(S/16) small CTAs: no cooperative launch, no grid barrier, safe to run concurrently on several streams.
 */
/* layout: 0 = compact expert rows ; 1 = capacity-padded slabs (offsets[e] = e*C) ; 2 = compact with every group padded to a
 * multiple of 128 rows (what lmod_grouped_gemm_bf16 wants).  The padding rows of xp (alignment / unused capacity) are zeroed by the
 * op itself, so xp needs no initialisation; rows past offsets[E] are not touched.
 * meta = {l_aux, capacity, rows_used, rows_end(=offsets[E]), exp_counts[E]}. */
int lmod_moe_capacity(int64_t S, int E, double capacity_factor, int64_t min_capacity);
int lmod_moe_route_scatter(const void* x, const float* wg, const float* noise, int64_t S, int64_t H,
                           int E, double capacity_factor, int64_t min_capacity, int layout,
                           float* logits, float* gates, int32_t* idx, int32_t* row, float* w,
                           int32_t* offsets, float* meta, void* xp, int32_t* ws, void* stream);
int64_t lmod_moe_route_ws_elems(int64_t S, int E);
/* Top-1 form (DeepSpeed-0.9.5 top1gating with random token selection, --top_k_experts 1): the same arguments and outputs, with
 *   uniform [S,E] fp32 in [0,1) in place of the noise: among the tokens routed to expert e, the C with the largest uniform[s, e] keep
 *   their seat (ties: the lower token index), seated in token order.  C = lmod_moe_capacity_top1 = ceil(S/E * cf) raised to
 *   min_capacity.  idx[:,1] = row[:,1] = -1, w[:,1] = 0, w[:,0] = the raw gate of a kept token (not renormalised), 0 if dropped.
 *   meta and offsets as for top-2, rows per expert min(n_e, C).  Three plain launches (gate, selection, seat+scatter).
 *   Fails before any launch if S < min_capacity or C > S (top1gating's own failure cases).
 *   ws: lmod_moe_route_top1_ws_elems(S, E) int32 elements.  The combine, scatter-backward and router-gradient entry points below serve
 *   the top-1 record unchanged; its gate backward is lmod_moe_gate_bwd_top1. */
int lmod_moe_capacity_top1(int64_t S, int E, double capacity_factor, int64_t min_capacity);
int lmod_moe_route_scatter_top1(const void* x, const float* wg, const float* uniform, int64_t S, int64_t H,
                                int E, double capacity_factor, int64_t min_capacity, int layout,
                                float* logits, float* gates, int32_t* idx, int32_t* row, float* w,
                                int32_t* offsets, float* meta, void* xp, int32_t* ws, void* stream);
int64_t lmod_moe_route_top1_ws_elems(int64_t S, int E);
/* combine einsum("sec,ecm->sm") with bf16-rounded weights + optional residual add (Appendix A step 11,
 * llava_qwen1_5_moe.py:167) */
int lmod_moe_gather_combine(const void* y, const int32_t* row, const float* w, const void* residual,
                            int64_t S, int64_t H, void* out, void* stream);
/* backward of gather_combine: dY rows + d(w) per choice */
int lmod_moe_combine_bwd(const void* dout, const void* y, const int32_t* row, const float* w,
                         int64_t S, int64_t H, void* dy, float* dw, void* stream);
/* backward of the gate: (dw, l_aux upstream grad) -> dlogits [S,E] fp32 */
int lmod_moe_gate_bwd(const float* gates, const int32_t* idx, const int32_t* row, const float* dw,
                      const float* meta, const float* g_laux, int64_t S, int E, float* dlogits,
                      void* stream);
/* top-1 gate backward: dgates[s, idx1] += dw1 for a kept token (no renormalisation), plus the l_aux term, through the softmax */
int lmod_moe_gate_bwd_top1(const float* gates, const int32_t* idx, const int32_t* row, const float* dw,
                           const float* meta, const float* g_laux, int64_t S, int E, float* dlogits,
                           void* stream);
/* dx[s] = dxp[row1] + dxp[row2] + sum_e dlogits[s,e]*wg[e] (+ dres) ; and dwg partial sums */
int lmod_moe_scatter_bwd(const void* dxp, const int32_t* row, const float* dlogits, const float* wg,
                         const void* dres, int64_t S, int64_t H, int E, void* dx, void* stream);
int lmod_moe_wg_grad(const void* x, const float* dlogits, int64_t S, int64_t H, int E,
                     float* ws /* [32,E,H] */, float* dwg /* [E,H], accumulated (+=) */, void* stream);
/* Residual-MoE (DeepSpeed MoE(use_residual=True), SURVEY.md Appendix A "Residual"): the routed output moe [S,H] (gather_combine without
 * residual) and the dense MLP's output mlp [S,H] mixed per token by a two-way softmax of the coefficient Linear, plus the residual add.
 * All bf16; one warp per token, 16-byte loads, no host sync.
 *   z = bf16(x Wc^T + bc) (fp32 accumulate; bc may be NULL), coef = bf16(softmax_fp32(z)) [S,2],
 *   out = bf16(res + bf16(bf16(moe*c0) + bf16(mlp*c1))).  wc [2,H], bc [2]. */
int lmod_moe_residual_mix(const void* x, const void* moe, const void* mlp, const void* res, const void* wc, const void* bc,
                          int64_t S, int64_t H, void* out, void* coef, void* stream);
/* fp32 elements of the workspace lmod_moe_residual_mix_bwd needs for the coefficient's gradient (no initialisation needed) */
int64_t lmod_moe_residual_ws_elems(int64_t H);
/* Backward of the mix for upstream g (the residual's gradient is g itself):
 *   d_moe = bf16(g*c0), d_mlp = bf16(g*c1) [S,H]; dz [S,2] fp32 = c (dc - <c,dc>) with dc_j = sum_h g*{moe,mlp} (fp32);
 *   dx_coef = bf16(dz Wc) [S,H], the coefficient's share of dx (callers accumulate the other addends onto it).
 *   dwc [2,H] / dbc [2] bf16 gradient views, accumulated (+=) by a fixed-partition two-stage reduction (bit-reproducible); either may
 *   be NULL (frozen), and with both NULL x and ws are not read.  ws: lmod_moe_residual_ws_elems(H) fp32 elements. */
int lmod_moe_residual_mix_bwd(const void* g, const void* x, const void* moe, const void* mlp, const void* coef, const void* wc,
                              int64_t S, int64_t H, void* d_moe, void* d_mlp, float* dz, void* dx_coef, float* ws, void* dwc,
                              void* dbc, void* stream);

/* ------------------------------------------------------------------------------------------
 * K4/K6/K9/K2/K1 element-wise + norm kernels (modeling_qwen2.py:105-110,159-184,199-200;
 * multimodal_projector/builder.py:57-61; transformers CLIP LayerNorm/quick_gelu).
 */
int lmod_rmsnorm_fwd(const void* x, const void* res /* optional: x := x + res first */, const void* w,
                     int64_t rows, int64_t H, float eps, void* y, void* x_out /* x+res, optional */,
                     float* rstd, void* stream);
int lmod_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres,
                     int64_t rows, int64_t H, void* dx, void* stream);
/* RMSNorm weight gradient (autograd of `self.weight * hidden_states.to(input_dtype)`, qwen1_5/modeling_qwen2.py:110):
 * wgrad[h] += bf16( sum_r bf16(dy[r,h] * bf16(x[r,h] * rstd[r])) ).  x is the tensor the forward normalised (x_out of lmod_rmsnorm_fwd when a
 * residual was fused), rstd its per-row output.  ws_zeroed: fp32 [H] workspace that must be zero on entry and is zero again on return.
 * Only needed when the norm weights train (dense-student distillation, full SFT); the sparse recipes freeze them. */
int lmod_rmsnorm_wgrad(const void* dy, const void* x, const float* rstd, int64_t rows, int64_t H, float* ws_zeroed, void* wgrad, void* stream);

/* Token-embedding gradient behind the multimodal splice (nn.Embedding backward; llava_arch.py:262-274): for every token t,
 * grad[t, :] = bf16(grad[t, :] + bf16(sum over the rows r with src[r] == t of dout[r, :])), the sum in fp32 in row order, so the result
 * is deterministic.  Rows that hold image patches or padding carry src < 0, as in lmod_splice_embed, and add nothing.
 * order [n_rows] int64: the row indices grouped by token, a stable sort of src with the rows src < 0 last (llava_arch.embed_grad_order).
 * H % 8 == 0; dout and grad 16-byte aligned. */
int lmod_embed_grad(const void* dout, const int64_t* src, const int64_t* order, int64_t n_rows, int64_t H, void* grad, void* stream);
int lmod_layernorm_fwd(const void* x, const void* w, const void* b, int64_t rows, int64_t H, float eps,
                       void* y, void* stream);
/* rotate-half RoPE applied in place to q [rows, nh*hd] and k [rows, nkv*hd] (rows of a fused QKV buffer via ld).
 * cos/sin tables are the reference's bf16 cache ([max_pos, hd], modeling_qwen2.py:127-136) gathered by position_ids. */
int lmod_rope(void* q, int64_t ld_q, int nh, void* k, int64_t ld_k, int nkv, int hd,
              const void* cos_table, const void* sin_table, const int64_t* position_ids, int64_t rows,
              int backward, void* stream);
int lmod_silu_mul_fwd(const void* gate_up, int64_t ld, int64_t rows, int64_t I, void* out, void* stream);
int lmod_silu_mul_bwd(const void* dout, const void* gate_up, int64_t ld, int64_t rows, int64_t I,
                      void* dgate_up, void* stream);
/* act: 0 = gelu(erf), 1 = quick_gelu ; in place allowed; optional bias [n] added first */
int lmod_bias_act_fwd(const void* x, const void* bias, int64_t rows, int64_t n, int act, void* y,
                      void* stream);
int lmod_gelu_bwd(const void* dy, const void* x_pre, int64_t count, void* dx, void* stream);
int lmod_add(const void* a, const void* b, int64_t count, void* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * K3: multimodal splice (llava_arch.py:228-320): src [B*T'] int64 plan (>=0 token id, -1-k image
 * row k, other = padding), img_index [B*T'] int64.
 */
int lmod_splice_embed(const void* embed_w, const void* feats, const int64_t* src, const int64_t* img_index,
                      int64_t n_rows, int64_t H, int64_t n_patches, void* out, void* stream);
int lmod_splice_embed_bwd(const void* dout, const int64_t* src, const int64_t* img_index, int64_t n_rows,
                          int64_t H, int64_t n_patches, void* dfeats /* pre-zeroed */, void* stream);

/* ------------------------------------------------------------------------------------------
 * K19: fused AdamW on flat buffers (fp32 master/moments, bf16 model copy), global-norm clip.
 * Replaces DeepSpeed ZeRO-2 + CPUAdam (align_trainer.py:404-417; zero2_offload.json).
 */
int lmod_sumsq(const void* g_bf16_or_f32, int is_f32, int64_t count, float* out_accum /* += */, void* stream);
int lmod_adamw(float* master, float* m, float* v, const void* grad, int grad_is_f32, void* model_bf16,
               int64_t count, float lr, float beta1, float beta2, float eps, float wd, int64_t step,
               const float* gnorm_sq /* optional */, float max_norm, float grad_scale, void* stream);
/* The same step with 8-bit block-wise moments: the reference's --optim adamw_bnb_8bit / adamw_8bit, which HF's
 * Trainer.get_optimizer_cls_and_kwargs maps to bitsandbytes' 8-bit AdamW (align_trainer.py:409-429).  m8 / v8 [count] uint8 codes of
 * bitsandbytes' signed / unsigned dynamic maps; absmax_m / absmax_v [ceil(count / 2048)] fp32 scales, one per 2048-element block from
 * the start of the buffer.  grad and model are bf16 (model optional).  master, m8, v8, grad, model 16B aligned; count % 8 == 0; step >= 1.
 * Semantics (block rule, rounding, NaN): DESIGN.md section 5. */
int lmod_adamw_8bit(float* master, uint8_t* m8, uint8_t* v8, float* absmax_m, float* absmax_v, const void* grad_bf16,
                    void* model_bf16, int64_t count, float lr, float beta1, float beta2, float eps, float wd, int64_t step,
                    const float* gnorm_sq /* optional */, float max_norm, float grad_scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * K5/K8/K9/K12/K14: hand-written wgmma + TMA GEMM  D[M,N] (+)= A[M,K] * B[N,K]^T, bf16 in, fp32 register accumulate.
 * Replaces the nn.Linear call sites (modeling_qwen2.py:199-200,678-680,726,1176) and their autograd (dgrad / wgrad).
 *   a_mn_major / b_mn_major: 0 = operand stored K-major ([rows,K], "T"), 1 = stored MN-major ([K,rows], "N"), so that
 *   dgrad (B = W as stored) and wgrad (A = dY^T, B = X^T) need no transposed copies.
 *   epilogue bit0: D = bf16(D + acc).  bias [N] optional.  d_f32_accum != NULL: fp32 D32[M,ldd] += acc instead of D.
 *   epilogue bits 8..: split-K factor.  (The fused SwiGLU forward is lmod_gemm_swiglu below.)
 * Grouped form = DeepSpeed Experts.forward on COMPACT rows (offsets from lmod_moe_route_scatter, 128-row aligned):
 *   mode 0 fwd  : D[rows_g,N] = A[rows_g,K] * B[g][N,K]^T     mode 1 dgrad: D[rows_g,N] = A[rows_g,K] * B[g][K,N]
 *   mode 2 wgrad: D[g][M,N] (+)= A[rows_g,M]^T * B[rows_g,N]
 */
int lmod_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major,
                   void* D, int64_t ldd, int64_t M, int64_t N, int64_t K, const void* bias, int epilogue,
                   float* d_f32_accum, void* stream);
/* lmod_gemm_bf16 with extents read from DEVICE memory at kernel start (dense problems only): M_eff = min(M, *m_rows_dev),
 * K_eff = min(K, round_up(*k_rows_dev, 64)); either pointer may be NULL (static extent).  Tensor maps and the launch grid are sized for the
 * static M / K; tiles beyond the effective extent are skipped, an empty reduction contributes zero.  Dynamic M: the last tile stores
 * all its rows, up to min(M, round_up(M_eff, 128)) (A's rows there times B; rows at or past that are untouched).  Dynamic K: rows
 * [*k_rows_dev, round_up(*k_rows_dev, 64)) of both MN-major operands are read, must be finite, and one of the two must be zero there
 * (lmod_gather_rows zero-fills the hidden rows; an m_rows_dev GEMM of them writes zero rows); rows past that are never read. */
int lmod_gemm_bf16_dyn(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major,
                       void* D, int64_t ldd, int64_t M, int64_t N, int64_t K, const void* bias, int epilogue,
                       float* d_f32_accum, const int32_t* m_rows_dev, const int32_t* k_rows_dev, void* stream);
/* q|k|v projection with apply_rotary_pos_emb (modeling_qwen2.py:678-691,159-184) in the GEMM epilogue: D[M,(nh+2nkv)*hd] = A W^T + bias,
 * q and k heads rotated with cos/sin [max_pos, hd] (bf16) at position_ids[row], v untouched.  Bit-identical to lmod_gemm_bf16 followed by
 * lmod_rope (same bf16 roundings).  hd in {64,128}. */
int lmod_gemm_qkv_rope(const void* A, int64_t lda, const void* W, int64_t ldb, const void* bias, void* D, int64_t ldd, int64_t M, int64_t K,
                       int nh, int nkv, int hd, const void* cos_table, const void* sin_table, const int64_t* position_ids, void* stream);
/* Fused SwiGLU MLP input, forward only (Qwen2MLP act_fn(gate_proj(x)) * up_proj(x), modeling_qwen2.py:199-200; DeepSpeed Experts.forward
 * of the sparse layers): ONE GEMM against the fused gate|up weight W_gu [2I, K] exactly as the checkpoint stores it (gate rows, then up
 * rows; no re-layout) whose epilogue applies SwiGLU: act[M, I] = bf16(bf16(silu(g)) * u), g / u = the bf16-rounded GEMM outputs
 * (bit-identical to lmod_gemm_bf16 + lmod_silu_mul_fwd).  I %% 128 == 0.  h1 must be NULL (ld_h1 is ignored): the pre-activations are
 * not stored; a backward runs lmod_gemm_bf16 + lmod_silu_mul_fwd, which keeps them.
 * Grouped form: compact expert rows, W_gu [G, 2I, K], offsets from lmod_moe_route_scatter (128-row aligned). */
int lmod_gemm_swiglu(const void* A, int64_t lda, const void* W_gu, int64_t ldb, void* act, int64_t ld_act, void* h1, int64_t ld_h1,
                     int64_t M, int64_t I, int64_t K, void* stream);
int lmod_grouped_gemm_swiglu(const void* A, int64_t lda, const void* W_gu, int64_t ldb, void* act, int64_t ld_act, void* h1, int64_t ld_h1,
                             const int32_t* offsets, int G, int64_t max_rows, int64_t I, int64_t K, void* stream);
int lmod_grouped_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, void* D, int64_t ldd,
                           const int32_t* offsets, int G, int64_t max_rows, int64_t M, int64_t N, int64_t K,
                           int mode, int epilogue, void* stream);

/* ------------------------------------------------------------------------------------------
 * FP8 (e4m3) frozen teacher: the decoder linears of a model that is never differentiated, on e4m3 wgmma (csrc/gemm_fp8.cu, csrc/quant.cu).
 * Quantiser (fp32, per row; stated in full at the top of csrc/quant.cu):
 *     amax  = max_k |x[k]|, NaN-propagating (any NaN -> NaN; +-inf -> inf)
 *     scale = amax == 0 ? 1 : amax / 448          (NaN -> NaN, inf -> inf)
 *     q[k]  = e4m3_rn(clamp(x[k] / scale, +-448)), the clamp passing NaN through
 * A row holding a NaN gets scale NaN and NaN bytes; a row holding an inf gets scale inf, NaN bytes at its infinite elements and +-0
 * elsewhere; either way that row of every e4m3 GEMM output is NaN and no other row changes.  e4m3 subnormal operands (2^-9 .. 0.875 *
 * 2^-6) are exact on the tensor core, not flushed.  Weights [N,K] are quantised per output channel with the same function, once;
 * activations per token by the kernel that produces the GEMM input.  GEMM: D[m,n] = (acc[m,n] * s_a[m]) * s_w[n] in fp32 (acc = the wgmma fp32 sum of the e4m3 products), then bias
 * / RoPE / SwiGLU with the expressions and bf16 roundings of the bf16 forms above.  Forward only, K-major operands only.
 * lmod_quant_rows_e4m3: x [M,K] bf16 (row stride ld) -> q [M,K] bytes + scale [M]; in front of o_proj (modeling_qwen2.py:726) and down_proj
 *   (:200), and for the weights.  K %% 16 == 0.
 * lmod_rmsnorm_quant_e4m3: lmod_rmsnorm_fwd (Qwen2RMSNorm :105-110 with the residual add of :796,808) writing q / scale instead of the bf16
 *   row -- bit-equal to lmod_quant_rows_e4m3 of lmod_rmsnorm_fwd's y; x_out as there.  In front of q|k|v (:678-680) and gate|up (:199).
 * lmod_gemm_e4m3: nn.Linear forward (o_proj :726, down_proj :200).  lda / ldb: row strides of the e4m3 operands in bytes (multiples of 16);
 *   bias (and cos / sin of the q|k|v form) 4-byte aligned.
 * lmod_gemm_e4m3_qkv_rope: lmod_gemm_qkv_rope (:678-691,159-184) on e4m3 operands; bit-identical to lmod_gemm_e4m3 + lmod_rope.
 * lmod_gemm_e4m3_swiglu: lmod_gemm_swiglu (:199-200) on e4m3 operands, W8_gu [2I,K] / s_w [2I] the fused gate|up weight; no pre-activations
 *   are kept; bit-identical to lmod_gemm_e4m3 + lmod_silu_mul_fwd.  I %% 128 == 0. */
int lmod_quant_rows_e4m3(const void* x, int64_t ld, void* q, float* scale, int64_t M, int64_t K, void* stream);
int lmod_rmsnorm_quant_e4m3(const void* x, const void* res, const void* w, int64_t rows, int64_t H, float eps, void* q, float* scale,
                            void* x_out, void* stream);
int lmod_gemm_e4m3(const void* A8, int64_t lda, const float* s_a, const void* W8, int64_t ldb, const float* s_w, const void* bias, void* D,
                   int64_t ldd, int64_t M, int64_t N, int64_t K, void* stream);
int lmod_gemm_e4m3_qkv_rope(const void* A8, int64_t lda, const float* s_a, const void* W8, int64_t ldb, const float* s_w, const void* bias,
                            void* D, int64_t ldd, int64_t M, int64_t K, int nh, int nkv, int hd, const void* cos_table,
                            const void* sin_table, const int64_t* position_ids, void* stream);
int lmod_gemm_e4m3_swiglu(const void* A8, int64_t lda, const float* s_a, const void* W8_gu, int64_t ldb, const float* s_w, void* act,
                          int64_t ld_act, int64_t M, int64_t I, int64_t K, void* stream);

/* ------------------------------------------------------------------------------------------
 * K7: flash-attention FORWARD on wgmma/TMA (modeling_qwen2.py:713-721 causal; CLIP non-causal), reading the fused RoPE'd
 * QKV buffer [batch*seq, (nh+2*nkv)*hd] in place (GQA by index).  hd in {64,128}.  out [batch*seq, nh*hd];
 * lse [batch, nh, seq] fp32 (natural-log LSE of the scaled scores, consumed by lmod_attn_bwd) or NULL.
 * Padded batches (the additive 4-D mask of modeling_qwen2.py:1035-1040; the varlen un-pad of :600-641): kv_lo / kv_hi are int32
 * [batch] device arrays giving the real key range [kv_lo[b], kv_hi[b]) of every batch row (right or left padding); a query row with
 * no visible key attends to all keys (HF _unmask_unattended).  Both NULL = no padding.  Padding needs causal = 1: a non-causal
 * call with kv_lo / kv_hi is rejected (LMOD_ERR_ARG), since those un-masked rows are not what a key-padding mask would give. */
int lmod_attn_fwd(const void* qkv, int64_t ld_qkv, int64_t batch, int64_t seq, int nh, int nkv, int hd, int causal,
                  float softmax_scale, void* out, int64_t ld_o, float* lse, const int32_t* kv_lo, const int32_t* kv_hi,
                  void* stream);
/* flash-attention BACKWARD on wgmma/TMA (autograd of the call above): dqkv (fused dq|dk|dv, same layout as qkv) from qkv, out, dout, lse.
 * dq32_ws: fp32 [batch*seq, nh*hd] workspace (zeroed inside), dsum_ws: fp32 [batch, nh, seq] workspace; kv_lo / kv_hi as above. */
int lmod_attn_bwd(const void* qkv, int64_t ld_qkv, const void* out, int64_t ld_o, const void* dout, int64_t ld_do,
                  const float* lse, int64_t batch, int64_t seq, int nh, int nkv, int hd, int causal, float softmax_scale,
                  void* dqkv, int64_t ld_dqkv, float* dq32_ws, float* dsum_ws, const int32_t* kv_lo, const int32_t* kv_hi,
                  void* stream);

/* ------------------------------------------------------------------------------------------
 * KV-cache decoding (csrc/decode.cu).  The cache of a layer is one K and one V buffer [batch, nkv, max_len, hd] bf16 (HF's legacy layout);
 * sequence b holds rows [0, len[b]).
 * lmod_kv_append: DynamicCache.update (the reference's cache_utils.py) -- copies the k and v heads of n_new rows per sequence of the fused,
 *   RoPE'd QKV buffer [batch*n_new, (nh+2*nkv)*hd] (row stride ld_qkv) to cache rows offsets[b] + [0, n_new), offsets int32 [batch] on the
 *   device.  Bit-exact; no other row is written (rows that would land at or past max_len are skipped; callers bounds-check).  hd %% 8 == 0.
 * lmod_attn_decode: the past_key_value path of Qwen2SdpaAttention.forward (modeling_qwen2.py:652-728) for one new query per sequence:
 *   q [batch, ld_q] (query heads at columns [h*hd, (h+1)*hd), e.g. the fused QKV rows) against cache rows [0, len[b]), len int32 [batch] on
 *   the device; GQA by index (query head h reads KV head h / (nh/nkv), nh/nkv <= 8).  out [batch, nh*hd] bf16 (row stride ld_o); lse
 *   [batch, nh] fp32 (natural-log LSE of the scaled scores) or NULL.  hd in {64,128}.  Split-KV: the launch grid depends on max_len, not
 *   on len, so a captured graph serves every step.  ws: fp32 workspace of at least lmod_attn_decode_ws_elems(...) elements. */
int lmod_kv_append(const void* qkv, int64_t ld_qkv, int64_t batch, int64_t n_new, int nh, int nkv, int hd, const int32_t* offsets,
                   void* k_cache, void* v_cache, int64_t max_len, void* stream);
/* lmod_kv_append_rows: the prefill of a padded batch -- of the n_rows rows per sequence of the fused QKV buffer [batch*n_rows, ...], copies
 *   rows [src_lo[b], src_hi[b]) of sequence b to cache rows offsets[b] + (r - src_lo[b]), so each sequence's real rows land packed from
 *   offsets[b].  src_lo / src_hi / offsets int32 [batch] on the device (the ranges the attention kernels mask with).  Bit-exact, no host
 *   sync; no other row is written (rows at or past max_len are skipped; callers bounds-check).  hd %% 8 == 0. */
int lmod_kv_append_rows(const void* qkv, int64_t ld_qkv, int64_t batch, int64_t n_rows, int nh, int nkv, int hd, const int32_t* src_lo,
                        const int32_t* src_hi, const int32_t* offsets, void* k_cache, void* v_cache, int64_t max_len, void* stream);
int64_t lmod_attn_decode_ws_elems(int64_t batch, int nh, int nkv, int hd, int64_t max_len);
int lmod_attn_decode(const void* q, int64_t ld_q, const void* k_cache, const void* v_cache, const int32_t* len, int64_t batch, int nh,
                     int nkv, int hd, int64_t max_len, float softmax_scale, void* out, int64_t ld_o, float* lse, float* ws,
                     int64_t ws_elems, void* stream);
/* lmod_attn_decode_chunk: the past_key_value path of Qwen2SdpaAttention.forward for T >= 1 new queries per sequence (the verify step of
 *   assisted decoding, HF generate(assistant_model=...)): q [batch*T, ld_q] (row b*T + t), their k / v already appended by lmod_kv_append
 *   (n_new = T), len int32 [batch] the lengths after the append.  Row t attends to cache rows [0, len[b] - T + t + 1).  out [batch*T, nh*hd]
 *   (row stride ld_o), lse [batch*T, nh] or NULL.  Row t gives the same bytes, in out and lse, as lmod_attn_decode on that row alone with
 *   len = len[b] - T + t + 1.  hd in {64,128}, nh/nkv <= 8.  ws: fp32 workspace of at least lmod_attn_decode_chunk_ws_elems(...). */
int64_t lmod_attn_decode_chunk_ws_elems(int64_t batch, int64_t T, int nh, int nkv, int hd, int64_t max_len);
int lmod_attn_decode_chunk(const void* q, int64_t ld_q, const void* k_cache, const void* v_cache, const int32_t* len, int64_t batch,
                           int64_t T, int nh, int nkv, int hd, int64_t max_len, float softmax_scale, void* out, int64_t ld_o, float* lse,
                           float* ws, int64_t ws_elems, void* stream);
/* lmod_attn_decode_shared: one new query for each of n sequences per prompt that share the prompt's K / V (num_return_sequences): q
 *   [batch*n, ld_q] (row b*n + j: copy j of prompt b).  Prompt b's keys [0, prefix_len[b]) are rows of the prefix buffers
 *   [batch, nkv, p_max, hd]; copy j's keys from prefix_len[b] on are rows of its suffix buffers [batch*n, nkv, s_max, hd] (key i at suffix
 *   row i - prefix_len[b]).  len int32 [batch*n] total keys per sequence, prefix_len int32 [batch], both on the device; len - prefix_len
 *   <= s_max.  A 64-key block wholly inside the prefix is read once for all copies a CTA serves (min(n, 8 / (nh/nkv)) of them).  max_len:
 *   the length the expanded per-sequence cache would have; the splits are lmod_attn_decode's at that max_len, so every row's out and lse
 *   are the bytes lmod_attn_decode gives on that row's materialised cache (its prefix rows, then its suffix rows).  out [batch*n, nh*hd]
 *   (row stride ld_o), lse [batch*n, nh] or NULL.  hd in {64,128}, nh/nkv <= 8, any n >= 1.  ws: fp32 workspace of at least
 *   lmod_attn_decode_shared_ws_elems(...). */
int64_t lmod_attn_decode_shared_ws_elems(int64_t batch, int64_t n, int nh, int nkv, int hd, int64_t max_len);
int lmod_attn_decode_shared(const void* q, int64_t ld_q, const void* k_prefix, const void* v_prefix, const int32_t* prefix_len, int64_t p_max,
                            const void* k_suffix, const void* v_suffix, int64_t s_max, const int32_t* len, int64_t batch, int64_t n, int nh,
                            int nkv, int hd, int64_t max_len, float softmax_scale, void* out, int64_t ld_o, float* lse, float* ws,
                            int64_t ws_elems, void* stream);
/* lmod_kv_beam_reorder: beam search's cache reorder (HF _reorder_cache / index_select over the beams), in place.  bufs: device array of
 *   n_bufs pointers to bf16 buffers [prompts*n, nkv, cap, hp] (every layer's K and V in one launch); rows int32 [prompts], parent int32
 *   [prompts*n] with values in [0, n), both on the device.  For every buffer, prompt b, beam j, KV head h and row r < rows[b]:
 *   new[b*n + j, h, r, :hd] = old[b*n + parent[b*n + j], h, r, :hd], byte for byte.  Rows at or past rows[b] (clamped to cap) and columns
 *   [hd, hp) are not written; any map works in place (cycles, many beams from one), and a prompt whose map is the identity moves nothing.
 *   Everything read is on the device, so the launch can be captured.  hd %% 8 == 0, hd <= hp <= 128, n <= 128; n == 1 launches nothing.
 *   Callers check the ranges (a parent outside [0, n) leaves its beam unwritten). */
int lmod_kv_beam_reorder(void* const* bufs, int n_bufs, int64_t prompts, int64_t n, int nkv, int64_t cap, int hd, int hp, const int32_t* rows,
                         const int32_t* parent, void* stream);

/* ------------------------------------------------------------------------------------------
 * Assisted decoding (csrc/spec.cu).
 * lmod_spec_accept: HF's assisted-generation acceptance (generation/utils.py: the greedy candidate match of _assisted_decoding, and
 *   _speculative_sampling) for one round of k drafted tokens.  target_logits fp32 [batch, k+1, V_t]: row j holds the target's logits after
 *   the inputs [last, d_1 .. d_j], so it scores d_{j+1}; row k gives the bonus token.  draft_tokens int64 [batch, k].
 *   u == NULL (greedy): n_acc = the largest n with d_{j+1} == argmax(row j) (first index on ties) for every j < n; next = argmax(row n_acc).
 *   u fp32 [batch, k+1] (sampling; draft_logits fp32 [batch, k, V_d], both logit sets after the logits processors, -inf = probability 0,
 *   draft probability 0 for ids >= V_d): accept d_{j+1} while u_j * q_j(d_{j+1}) <= p_j(d_{j+1}) (fp32 softmaxes); at the first rejection
 *   next ~ normalize(max(0, p_j - q_j)), after k acceptances next ~ p_k, by inverse CDF with u_k over a fixed-order scan.
 *   Writes n_acc int32 [batch] and next int64 [batch]; len_target / len_draft int32 [batch] (either may be NULL) -= k - n_acc[b].  No host
 *   sync. */
int lmod_spec_accept(const float* target_logits, int64_t V_t, const float* draft_logits, int64_t V_d, const int64_t* draft_tokens,
                     const float* u, int64_t batch, int k, int32_t* n_acc, int64_t* next, int32_t* len_target, int32_t* len_draft,
                     void* stream);


#ifdef __cplusplus
}
#endif
#endif /* LMOD_H_ */
