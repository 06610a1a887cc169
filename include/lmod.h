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
/* dx[s] = dxp[row1] + dxp[row2] + sum_e dlogits[s,e]*wg[e] (+ dres) ; and dwg partial sums */
int lmod_moe_scatter_bwd(const void* dxp, const int32_t* row, const float* dlogits, const float* wg,
                         const void* dres, int64_t S, int64_t H, int E, void* dx, void* stream);
int lmod_moe_wg_grad(const void* x, const float* dlogits, int64_t S, int64_t H, int E,
                     float* ws /* [32,E,H] */, float* dwg /* [E,H], accumulated (+=) */, void* stream);

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

/* Token-embedding gradient behind the multimodal splice (nn.Embedding backward; llava_arch.py:262-274): for every row with src[row] >= 0,
 * grad[src[row], :] += dout[row, :] (bf16 atomics; rows that hold image patches or padding carry src < 0, as in lmod_splice_embed). */
int lmod_embed_grad(const void* dout, const int64_t* src, int64_t n_rows, int64_t H, void* grad, void* stream);
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

/* ------------------------------------------------------------------------------------------
 * K5/K8/K9/K12/K14: hand-written wgmma + TMA GEMM  D[M,N] (+)= A[M,K] * B[N,K]^T, bf16 in, fp32 register accumulate.
 * Replaces the nn.Linear call sites (modeling_qwen2.py:199-200,678-680,726,1176) and their autograd (dgrad / wgrad).
 *   a_mn_major / b_mn_major: 0 = operand stored K-major ([rows,K], "T"), 1 = stored MN-major ([K,rows], "N"), so that
 *   dgrad (B = W as stored) and wgrad (A = dY^T, B = X^T) need no transposed copies.
 *   epilogue bit0: D = bf16(D + acc).  bias [N] optional.  d_f32_accum != NULL: fp32 D32[M,ldd] += acc instead of D.
 *   epilogue bits 8..: split-K factor.  (The fused SwiGLU forms are lmod_gemm_swiglu / lmod_gemm_silu_bwd below.)
 * Grouped form = DeepSpeed Experts.forward on COMPACT rows (offsets from lmod_moe_route_scatter, 128-row aligned):
 *   mode 0 fwd  : D[rows_g,N] = A[rows_g,K] * B[g][N,K]^T     mode 1 dgrad: D[rows_g,N] = A[rows_g,K] * B[g][K,N]
 *   mode 2 wgrad: D[g][M,N] (+)= A[rows_g,M]^T * B[rows_g,N]
 */
int lmod_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major,
                   void* D, int64_t ldd, int64_t M, int64_t N, int64_t K, const void* bias, int epilogue,
                   float* d_f32_accum, void* stream);
/* lmod_gemm_bf16 with extents read from DEVICE memory at kernel start (dense problems only): M_eff = min(M, *m_rows_dev),
 * K_eff = min(K, round_up(*k_rows_dev, 64)); either pointer may be NULL (static extent).  Tensor maps and the launch grid are sized for the
 * static M / K; tiles beyond the effective extent are skipped, an empty reduction contributes zero.  Rows of A (or of both MN-major
 * operands, for a dynamic K) between the count and the next tile boundary must hold finite values (lmod_gather_rows zero-fills them). */
int lmod_gemm_bf16_dyn(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major,
                       void* D, int64_t ldd, int64_t M, int64_t N, int64_t K, const void* bias, int epilogue,
                       float* d_f32_accum, const int32_t* m_rows_dev, const int32_t* k_rows_dev, void* stream);
/* Fused SwiGLU MLP input (Qwen2MLP act_fn(gate_proj(x)) * up_proj(x), modeling_qwen2.py:199-200; DeepSpeed Experts.forward of the sparse
 * layers): ONE GEMM against the fused gate|up weight W_gu [2I, K] exactly as the checkpoint stores it (gate rows, then up rows; no
 * re-layout) whose epilogue applies SwiGLU: act[M, I] = bf16(bf16(silu(g)) * u), g / u = the bf16-rounded GEMM outputs (bit-identical to
 * lmod_gemm_bf16 + lmod_silu_mul_fwd).  h1 (optional, [M, 2I]) receives the pre-activations for the backward.  I %% 128 == 0.
 * Grouped form: compact expert rows, W_gu [G, 2I, K], offsets from lmod_moe_route_scatter (128-row aligned).
 * Backward: lmod_gemm_silu_bwd computes dh1[M, 2I] = silu_mul_bwd(dY W_dn, h1) in the epilogue of the down_proj dgrad GEMM
 * (dY [M, K], W_dn [K, I] as stored), so the [M, I] dact tensor is never written; grouped form W_dn [G, K, I]. */
/* D[M,N] = bf16( bf16(A W^T + bias) + R ): a projection written straight into the residual stream -- o_proj / down_proj of
 * Qwen2DecoderLayer.forward (`hidden_states = residual + hidden_states`, modeling_qwen2.py:796,808) and out_proj / fc2 of the CLIP encoder
 * layers.  The GEMM output is rounded to bf16 before the add, as the reference materialises it: bit-identical to lmod_gemm_bf16 + lmod_add.
 * A [M,K], W [N,K] (both K-major), bias [N] or NULL, R [M,N] (row stride ld_r); D may alias R. */
int lmod_gemm_residual(const void* A, int64_t lda, const void* W, int64_t ldb, const void* bias, const void* R, int64_t ld_r,
                       void* D, int64_t ldd, int64_t M, int64_t N, int64_t K, void* stream);
/* q|k|v projection with apply_rotary_pos_emb (modeling_qwen2.py:678-691,159-184) in the GEMM epilogue: D[M,(nh+2nkv)*hd] = A W^T + bias,
 * q and k heads rotated with cos/sin [max_pos, hd] (bf16) at position_ids[row], v untouched.  Bit-identical to lmod_gemm_bf16 followed by
 * lmod_rope (same bf16 roundings).  hd in {64,128}. */
int lmod_gemm_qkv_rope(const void* A, int64_t lda, const void* W, int64_t ldb, const void* bias, void* D, int64_t ldd, int64_t M, int64_t K,
                       int nh, int nkv, int hd, const void* cos_table, const void* sin_table, const int64_t* position_ids, void* stream);
int lmod_gemm_swiglu(const void* A, int64_t lda, const void* W_gu, int64_t ldb, void* act, int64_t ld_act, void* h1, int64_t ld_h1,
                     int64_t M, int64_t I, int64_t K, void* stream);
int lmod_grouped_gemm_swiglu(const void* A, int64_t lda, const void* W_gu, int64_t ldb, void* act, int64_t ld_act, void* h1, int64_t ld_h1,
                             const int32_t* offsets, int G, int64_t max_rows, int64_t I, int64_t K, void* stream);
int lmod_gemm_silu_bwd(const void* dY, int64_t lda, const void* W_dn, int64_t ldb, const void* h1, int64_t ld_h1, void* dh1, int64_t ld_dh1,
                       int64_t M, int64_t I, int64_t K, void* stream);
int lmod_grouped_gemm_silu_bwd(const void* dY, int64_t lda, const void* W_dn, int64_t ldb, const void* h1, int64_t ld_h1, void* dh1,
                               int64_t ld_dh1, const int32_t* offsets, int G, int64_t max_rows, int64_t I, int64_t K, void* stream);
int lmod_grouped_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, void* D, int64_t ldd,
                           const int32_t* offsets, int G, int64_t max_rows, int64_t M, int64_t N, int64_t K,
                           int mode, int epilogue, void* stream);

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
int64_t lmod_attn_decode_ws_elems(int64_t batch, int nh, int nkv, int hd, int64_t max_len);
int lmod_attn_decode(const void* q, int64_t ld_q, const void* k_cache, const void* v_cache, const int32_t* len, int64_t batch, int nh,
                     int nkv, int hd, int64_t max_len, float softmax_scale, void* out, int64_t ld_o, float* lse, float* ws,
                     int64_t ws_elems, void* stream);


#ifdef __cplusplus
}
#endif
#endif /* LMOD_H_ */
