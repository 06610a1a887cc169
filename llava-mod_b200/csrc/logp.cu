// logp.cu -- DPO log-prob gather (K17) and the materialising API-compat forms of get_p / get_logp /
// compute_align_loss.
//
// Reference: llavamod/train/dpo_trainer.py:483-495 (shift, log_softmax over the FULL vocab, gather,
// masked sequence sum) and llavamod/train/align_trainer.py:473-475,497-499,509-526.
// All kernels are HBM-streaming: 16-byte read-only loads, per-thread online log-sum-exp, warp-shuffle
// + shared-memory block reduction, one CTA per row.
#include "common.cuh"

namespace {

constexpr int LP_THREADS = 256;

struct OnlineLse {
  float m, z;
  __device__ __forceinline__ void init() { m = -INFINITY; z = 0.f; }
  __device__ __forceinline__ void add8(const uint4& v) {
    float x[8] = {bf16lo(v.x), bf16hi(v.x), bf16lo(v.y), bf16hi(v.y), bf16lo(v.z), bf16hi(v.z), bf16lo(v.w), bf16hi(v.w)};
    float vm = fmaxf(fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3])), fmaxf(fmaxf(x[4], x[5]), fmaxf(x[6], x[7])));
    if (vm > m) { z *= ex2f((m - vm) * LOG2E_F); m = vm; }     // m == -inf: z is 0 and stays 0 (ex2(-inf)=0)
    // While m is still -inf (every element so far -inf) the exponent is taken against 0, so a -inf element adds ex2(-inf) = 0;
    // against m it would be -inf - (-inf) = NaN, which no later rescale clears (the same guard as kl.cu).
    const float nm = isinf(m) ? 0.f : -m * LOG2E_F;
#pragma unroll
    for (int j = 0; j < 8; ++j) z += ex2f(fmaf(x[j], LOG2E_F, nm));
  }
  __device__ __forceinline__ void add1(float x) {
    if (x > m) { z *= ex2f((m - x) * LOG2E_F); m = x; }
    z += ex2f((x - (isinf(m) ? 0.f : m)) * LOG2E_F);
  }
};

// combine (m,z) pairs across the block; result lse broadcast
__device__ __forceinline__ float block_lse(OnlineLse o, float* red) {
  float M = block_max(o.m, red);
  float Mu = isinf(M) ? 0.f : M;
  float zz = isinf(o.m) ? 0.f : o.z * ex2f((o.m - Mu) * LOG2E_F);
  float Z = block_sum(zz, red);
  return Mu + lg2f(Z) * LN2_F;
}

__global__ void __launch_bounds__(LP_THREADS) logp_fwd_kernel(
    const __nv_bfloat16* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels, int64_t T,
    int vocab, float* __restrict__ tok_logp, float* __restrict__ lse_out) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;              // row = b*T + t ; predicts labels[row+1]
  const int64_t tpos = row % T;
  int64_t lab = LMOD_IGNORE_INDEX;
  if (tpos + 1 < T) lab = labels[row + 1];
  if (lab == LMOD_IGNORE_INDEX) {               // masked: per_token_logps * 0 (dpo_trainer.py:493-495)
    if (threadIdx.x == 0) { tok_logp[row] = 0.f; lse_out[row] = 0.f; }
    return;
  }
  const __nv_bfloat16* r = logits + row * ld;
  OnlineLse o; o.init();
  const int nvec = vocab >> 3;
  const uint4* rv = reinterpret_cast<const uint4*>(r);
  int i = threadIdx.x;
  for (; i + 3 * LP_THREADS < nvec; i += 4 * LP_THREADS) {   // 4 independent 16B loads in flight
    uint4 a = ldg_nc_v4(rv + i), b = ldg_nc_v4(rv + i + LP_THREADS), c = ldg_nc_v4(rv + i + 2 * LP_THREADS),
          d = ldg_nc_v4(rv + i + 3 * LP_THREADS);
    o.add8(a); o.add8(b); o.add8(c); o.add8(d);
  }
  for (; i < nvec; i += LP_THREADS) o.add8(ldg_nc_v4(rv + i));
  for (int j = (nvec << 3) + threadIdx.x; j < vocab; j += LP_THREADS) o.add1(__bfloat162float(r[j]));
  float lse = block_lse(o, red);
  if (threadIdx.x == 0) {
    tok_logp[row] = __bfloat162float(r[lab]) - lse;
    lse_out[row] = lse;
  }
}

__global__ void logp_seq_sum_kernel(const float* __restrict__ tok_logp, const int64_t* __restrict__ labels,
                                    int64_t T, int average, float* __restrict__ seq_logp) {
  __shared__ float red[32];
  const int64_t b = blockIdx.x;
  float s = 0.f, c = 0.f;
  for (int64_t t = threadIdx.x; t + 1 < T; t += blockDim.x) {
    if (labels[b * T + t + 1] != LMOD_IGNORE_INDEX) { s += tok_logp[b * T + t]; c += 1.f; }
  }
  s = block_sum(s, red); c = block_sum(c, red);
  if (threadIdx.x == 0) seq_logp[b] = average ? s / c : s;
}

__global__ void __launch_bounds__(LP_THREADS) logp_bwd_kernel(
    const __nv_bfloat16* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels, int64_t T,
    int vocab, const float* __restrict__ lse_in, const float* __restrict__ g_seq, const float* __restrict__ inv_cnt,
    __nv_bfloat16* __restrict__ d, int64_t ld_d) {
  const int64_t row = blockIdx.x;
  const int64_t tpos = row % T, b = row / T;
  int64_t lab = LMOD_IGNORE_INDEX;
  if (tpos + 1 < T) lab = labels[row + 1];
  const int nvec = vocab >> 3;
  uint4* dv = reinterpret_cast<uint4*>(d + row * ld_d);
  if (lab == LMOD_IGNORE_INDEX) {
    uint4 z = make_uint4(0, 0, 0, 0);
    for (int i = threadIdx.x; i < nvec; i += LP_THREADS) stg_v4(dv + i, z);
    for (int j = (nvec << 3) + threadIdx.x; j < vocab; j += LP_THREADS) d[row * ld_d + j] = __float2bfloat16(0.f);
    return;
  }
  float g = g_seq[b];
  if (inv_cnt) g *= inv_cnt[b];
  const float e0 = -lse_in[row] * LOG2E_F;
  const uint4* rv = reinterpret_cast<const uint4*>(logits + row * ld);
  for (int i = threadIdx.x; i < nvec; i += LP_THREADS) {
    uint4 v = ldg_nc_v4(rv + i);
    float x[8] = {bf16lo(v.x), bf16hi(v.x), bf16lo(v.y), bf16hi(v.y), bf16lo(v.z), bf16hi(v.z), bf16lo(v.w), bf16hi(v.w)};
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = -g * ex2f(fmaf(x[j], LOG2E_F, e0));
    const unsigned rel = (unsigned)((int)lab - i * 8);
    if (rel < 8u) {
#pragma unroll
      for (int j = 0; j < 8; ++j) if (rel == (unsigned)j) o[j] += g;
    }
    uint4 w;
    w.x = pack_bf16x2(o[0], o[1]); w.y = pack_bf16x2(o[2], o[3]); w.z = pack_bf16x2(o[4], o[5]); w.w = pack_bf16x2(o[6], o[7]);
    stg_v4(dv + i, w);
  }
  for (int j = (nvec << 3) + threadIdx.x; j < vocab; j += LP_THREADS) {
    float q = ex2f(fmaf(__bfloat162float(logits[row * ld + j]), LOG2E_F, e0));
    d[row * ld_d + j] = __float2bfloat16(-g * q + ((int64_t)j == lab ? g : 0.f));
  }
}

// ---- API-compat materialising kernels ----------------------------------------------------------
__global__ void __launch_bounds__(LP_THREADS) softmax_rows_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld,
                                                                 int vocab, int log_mode, float* __restrict__ out,
                                                                 int64_t ld_out) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const __nv_bfloat16* r = logits + row * ld;
  OnlineLse o; o.init();
  for (int j = threadIdx.x; j < vocab; j += LP_THREADS) o.add1(__bfloat162float(r[j]));
  float lse = block_lse(o, red);
  float* w = out + row * ld_out;
  for (int j = threadIdx.x; j < vocab; j += LP_THREADS) {
    float x = __bfloat162float(r[j]);
    w[j] = log_mode ? (x - lse) : ex2f((x - lse) * LOG2E_F);
  }
}

__global__ void __launch_bounds__(LP_THREADS) align_dense_rows_kernel(const float* __restrict__ logp,
                                                                     const float* __restrict__ probs, int64_t ld,
                                                                     int vocab, float* __restrict__ row_x) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  float a = 0.f;
  for (int j = threadIdx.x; j < vocab; j += LP_THREADS) {
    float l = logp[row * ld + j];
    a += isinf(l) ? 0.f : probs[row * ld + j] * l;      // align_trainer.py:509-510
  }
  a = block_sum(a, red);
  if (threadIdx.x == 0) row_x[row] = a;
}

__global__ void align_dense_final_kernel(const float* __restrict__ row_x, const int64_t* __restrict__ labels, int64_t n,
                                         int distill_all, float* __restrict__ out) {
  __shared__ float red[32];
  float s = 0.f, c = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    bool m = distill_all || labels[i] != LMOD_IGNORE_INDEX;
    if (m) { s += row_x[i]; c += 1.f; }
  }
  s = block_sum(s, red); c = block_sum(c, red);
  if (threadIdx.x == 0) out[0] = -s / c;
}

}  // namespace

extern "C" int lmod_logp_gather_fwd(const void* logits, int64_t ld, const int64_t* labels, int64_t batch,
                                    int64_t seq_len, int64_t vocab, float* tok_logp, float* lse, float* seq_logp,
                                    int average, void* stream) {
  LMOD_CHECK_ARG(logits && labels && tok_logp && lse && seq_logp, "lmod_logp_gather_fwd: null pointer");
  LMOD_CHECK_ARG(batch > 0 && seq_len > 0 && vocab > 0 && ld >= vocab && ld % 8 == 0 && (uintptr_t)logits % 16 == 0,
                 "lmod_logp_gather_fwd: ld must be a multiple of 8 and logits 16B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  logp_fwd_kernel<<<(unsigned)(batch * seq_len), LP_THREADS, 0, st>>>((const __nv_bfloat16*)logits, ld, labels, seq_len,
                                                                     (int)vocab, tok_logp, lse);
  LMOD_LAUNCH_OK();
  logp_seq_sum_kernel<<<(unsigned)batch, 256, 0, st>>>(tok_logp, labels, seq_len, average, seq_logp);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_logp_gather_bwd(const void* logits, int64_t ld, const int64_t* labels, int64_t batch,
                                    int64_t seq_len, int64_t vocab, const float* lse, const float* g_seq, int average,
                                    void* dlogits, int64_t ld_d, void* stream) {
  LMOD_CHECK_ARG(logits && labels && lse && g_seq && dlogits, "lmod_logp_gather_bwd: null pointer");
  LMOD_CHECK_ARG(ld % 8 == 0 && ld_d % 8 == 0 && ld >= vocab && ld_d >= vocab && (uintptr_t)logits % 16 == 0 &&
                     (uintptr_t)dlogits % 16 == 0, "lmod_logp_gather_bwd: bad strides / alignment");
  LMOD_CHECK_ARG(!average, "lmod_logp_gather_bwd: average_log_prob backward needs a scratch buffer (unsupported)");
  cudaStream_t st = (cudaStream_t)stream;
  logp_bwd_kernel<<<(unsigned)(batch * seq_len), LP_THREADS, 0, st>>>((const __nv_bfloat16*)logits, ld, labels, seq_len,
                                                                     (int)vocab, lse, g_seq, nullptr,
                                                                     (__nv_bfloat16*)dlogits, ld_d);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_softmax_rows(const void* logits_bf16, int64_t ld, int64_t n_rows, int64_t vocab, int log_mode,
                                 float* out, int64_t ld_out, void* stream) {
  LMOD_CHECK_ARG(logits_bf16 && out && n_rows > 0 && vocab > 0 && ld >= vocab && ld_out >= vocab, "lmod_softmax_rows: bad arguments");
  softmax_rows_kernel<<<(unsigned)n_rows, LP_THREADS, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)logits_bf16, ld,
                                                                                 (int)vocab, log_mode, out, ld_out);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_align_loss_dense(const float* logp, const float* probs, int64_t ld, const int64_t* labels,
                                     int64_t n_rows, int64_t vocab, int distill_all, float* row_x, float* out_loss,
                                     void* stream) {
  LMOD_CHECK_ARG(logp && probs && labels && row_x && out_loss && n_rows > 0 && vocab > 0 && ld >= vocab,
                 "lmod_align_loss_dense: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  align_dense_rows_kernel<<<(unsigned)n_rows, LP_THREADS, 0, st>>>(logp, probs, ld, (int)vocab, row_x);
  LMOD_LAUNCH_OK();
  align_dense_final_kernel<<<1, 1024, 0, st>>>(row_x, labels, n_rows, distill_all, out_loss);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
