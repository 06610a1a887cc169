// rows.cu -- supervised-row compaction for the loss head.
//
// The reference pushes every position of the sequence through both lm_heads and the vocabulary-wide loss and then multiplies the
// masked ones by zero (align_trainer.py:512-526 `masked_fill` / mask product; llava_qwen1_5_moe.py:413-421 ignore_index).  With LLaVA
// data ~40-60 % of the positions (system prompt, image patches, the question) carry neither a KD mask nor a CE target, so here the
// student / teacher lm_head GEMMs, the fused KL+CE kernel and the lm_head backward GEMMs run on the batch's ACTIVE rows only:
//   lmod_active_rows  -> perm[j] = original row of the j-th active row, count (device scalars, no host sync, CUDA-graph friendly)
//   lmod_gather_rows  -> compact copy of the hidden states (rows count..round_up(count,pad) zero-filled, so the rows past count that
//                        a partial GEMM tile computes are exact zeros)
//   The lm_head wgrad reduces over rows [0, round_up(count, 64)) of BOTH the hidden rows and dlogits, and 0 * NaN is NaN: dlogits rows
//   [count, round_up(count, 64)) must be finite too.  The KL kernel writes rows < count only; the m_dev logits GEMM stores its whole
//   last 128-row tile (gemm.cu), which puts exact zeros (zero hidden rows times W) into those rows before the KL kernel runs.
//   lmod_scatter_rows -> d hidden back to its original rows
// The GEMMs read the dynamic extents from device memory (lmod_gemm_bf16_dyn).  Results are identical: a row that contributes
// exactly zero to the loss contributes exactly zero gradient.
#include "common.cuh"

namespace {

// active(row) = KD mask || CE mask, the same predicate kl_stream_kernel evaluates: labels[row] != -100 (or distill_all) ||
// (row is not the last of its sequence && labels[row+1] != -100)
__global__ void __launch_bounds__(1024) active_rows_kernel(const int64_t* __restrict__ labels, int64_t n, int64_t T, int distill_all,
                                                          int32_t* __restrict__ perm, int32_t* __restrict__ count) {
  __shared__ int warp_tot[32];
  __shared__ int base_s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) base_s = 0;
  __syncthreads();
  for (int64_t start = 0; start < n; start += blockDim.x) {
    const int64_t row = start + threadIdx.x;
    bool act = false;
    if (row < n) {
      act = distill_all || labels[row] != LMOD_IGNORE_INDEX;
      if (!act && (row % T) + 1 < T) act = labels[row + 1] != LMOD_IGNORE_INDEX;
    }
    const unsigned m = __ballot_sync(0xffffffffu, act);
    if (lane == 0) warp_tot[warp] = __popc(m);
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; ++w) before += warp_tot[w];
    const int pos = base_s + before + __popc(m & ((1u << lane) - 1u));
    if (act) perm[pos] = (int32_t)row;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += warp_tot[w];
      base_s += tot;
    }
    __syncthreads();
  }
  const int total = base_s;
  for (int64_t j = total + threadIdx.x; j < n; j += blockDim.x) perm[j] = -1;
  if (threadIdx.x == 0) *count = total;
}

// one warp per destination row; perm == null: identity (a dynamic-count row copy)
__global__ void __launch_bounds__(256) gather_rows_kernel(const __nv_bfloat16* __restrict__ src, int64_t ld_src, const int32_t* __restrict__ perm,
                                                         const int32_t* __restrict__ count, int64_t max_rows, int cols, int pad_to,
                                                         __nv_bfloat16* __restrict__ dst, int64_t ld_dst) {
  const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= max_rows) return;
  const int c = *count;
  const int64_t padded = ((int64_t)c + pad_to - 1) / pad_to * pad_to;
  uint4* to = reinterpret_cast<uint4*>(dst + j * ld_dst);
  if (j < c) {
    const int64_t r = perm ? perm[j] : j;
    const uint4* from = reinterpret_cast<const uint4*>(src + r * ld_src);
    for (int v = lane; v < (cols >> 3); v += 32) to[v] = ldg_nc_v4(from + v);
  } else if (j < padded) {
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (int v = lane; v < (cols >> 3); v += 32) to[v] = z;
  }
}

// dst[perm[j], :] = src[j, :] * scale for j < count (dst pre-zeroed by the caller)
__global__ void __launch_bounds__(256) scatter_rows_kernel(const __nv_bfloat16* __restrict__ src, int64_t ld_src, const int32_t* __restrict__ perm,
                                                          const int32_t* __restrict__ count, int64_t max_rows, int cols,
                                                          __nv_bfloat16* __restrict__ dst, int64_t ld_dst) {
  const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= max_rows || j >= *count) return;
  const uint4* from = reinterpret_cast<const uint4*>(src + j * ld_src);
  uint4* to = reinterpret_cast<uint4*>(dst + (int64_t)perm[j] * ld_dst);
  for (int v = lane; v < (cols >> 3); v += 32) to[v] = from[v];
}

}  // namespace

extern "C" int lmod_active_rows(const int64_t* labels, int64_t n_rows, int64_t seq_len, int distill_all, int32_t* perm, int32_t* count, void* stream) {
  LMOD_CHECK_ARG(labels && perm && count && n_rows > 0 && seq_len > 0 && n_rows % seq_len == 0 && n_rows < ((int64_t)1 << 31),
                 "lmod_active_rows: bad arguments (n_rows=%lld seq_len=%lld)", (long long)n_rows, (long long)seq_len);
  active_rows_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(labels, n_rows, seq_len, distill_all, perm, count);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_gather_rows(const void* src, int64_t ld_src, const int32_t* perm, const int32_t* count, int64_t max_rows, int64_t cols,
                                int64_t pad_to, void* dst, int64_t ld_dst, void* stream) {
  LMOD_CHECK_ARG(src && count && dst && max_rows > 0 && cols > 0 && cols % 8 == 0 && ld_src % 8 == 0 && ld_dst % 8 == 0 && pad_to >= 1,
                 "lmod_gather_rows: bad arguments (cols and strides must be multiples of 8 elements)");
  gather_rows_kernel<<<(unsigned)((max_rows * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)src, ld_src, perm, count, max_rows, (int)cols, (int)pad_to, (__nv_bfloat16*)dst, ld_dst);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_scatter_rows(const void* src, int64_t ld_src, const int32_t* perm, const int32_t* count, int64_t max_rows, int64_t cols,
                                 void* dst, int64_t ld_dst, void* stream) {
  LMOD_CHECK_ARG(src && perm && count && dst && max_rows > 0 && cols > 0 && cols % 8 == 0 && ld_src % 8 == 0 && ld_dst % 8 == 0,
                 "lmod_scatter_rows: bad arguments");
  scatter_rows_kernel<<<(unsigned)((max_rows * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)src, ld_src, perm, count, max_rows, (int)cols, (__nv_bfloat16*)dst, ld_dst);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
