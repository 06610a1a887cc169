// quant.cu -- row-wise e4m3 quantisation of bf16 rows for the FP8 (e4m3) frozen teacher (gemm_fp8.cu consumes the bytes and the scales).
//
// The quantiser, in fp32, for one row x[0..K) (bf16 values are exact in fp32):
//     amax  = max_k |x[k]|, NaN-propagating (any NaN -> NaN; +-inf -> inf)
//     scale = amax == 0 ? 1 : amax / 448          (NaN -> NaN, inf -> inf)
//     q[k]  = e4m3_rn(clamp(x[k] / scale, +-448)), the clamp passing NaN through
// with IEEE divisions, round to nearest (one for the scale, one per element: not a reciprocal multiply), the clamp after the division and
// before the conversion to e4m3 (the "fn" format: largest finite value 448, NaN 0x7F / 0xFF) round-to-nearest-even.  Subnormal scales are
// kept (no flush to zero); an all-zero row gets scale 1 and zero bytes.  x ~= scale * q.
// Non-finite rows: a row holding a NaN gets scale NaN and NaN bytes; a row holding an inf gets scale inf, NaN bytes at its infinite
// elements and +-0 elsewhere.  Either way every column of that row of an e4m3 GEMM is NaN, as in the bf16 teacher, and no other row
// changes.  (fmaxf / fminf return the non-NaN operand, which would turn such a row into finite -448's: hence max_nan (common.cuh) and
// clamp448 below.)
// tests/fp8_oracle.py restates exactly this; lmod_quant_rows_e4m3 and lmod_rmsnorm_quant_e4m3 are bit-equal to it.
//
// One CTA of 128 threads per row.  The row is read from global memory once (16-byte loads), parked in shared memory while the block
// reduces its amax, and converted from there with 16-byte stores.  No host sync, no workspace: graph-capturable.
#include <cuda_fp8.h>
#include "common.cuh"

namespace {

constexpr int QUANT_THREADS = 128;
constexpr int QUANT_MAX_K = 96 * 1024;      // the row (2 bytes per element) has to fit the CTA's shared memory

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  f[0] = bf16lo(u.x); f[1] = bf16hi(u.x); f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
  f[4] = bf16lo(u.z); f[5] = bf16hi(u.z); f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]); o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
  return o;
}
// clamp that returns NaN when the operand is NaN (PTX max.NaN / min.NaN, sm_80+; max_nan is in common.cuh)
__device__ __forceinline__ float clamp448(float v) {
  float r;
  asm("max.NaN.f32 %0, %1, 0fC3E00000;\n\tmin.NaN.f32 %0, %0, 0f43E00000;" : "=f"(r) : "f"(v));     // -448, 448
  return r;
}
__device__ __forceinline__ float amax8(const uint4& u, float m) {
  float f[8];
  unpack8(u, f);
#pragma unroll
  for (int j = 0; j < 8; ++j) m = max_nan(m, fabsf(f[j]));
  return m;
}
// block_max of common.cuh with max_nan: a NaN in any thread's amax reaches every thread
__device__ __forceinline__ float block_max_nan(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = lane < QUANT_THREADS / 32 ? red[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r = max_nan(r, __shfl_xor_sync(0xffffffffu, r, o));
  return r;
}
__device__ __forceinline__ uint32_t e4m3x4(const float* f, float scale) {
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = clamp448(__fdiv_rn(f[j], scale));
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v[0], v[1]), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v[2], v[3]), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
// second pass: the bf16 row in shared memory (K % 16 == 0) -> e4m3 bytes, 16 per thread and store
__device__ __forceinline__ void convert_row(const uint4* srow, int K, float amax, uint8_t* q, float* scale_out) {
  const float scale = amax == 0.f ? 1.f : __fdiv_rn(amax, 448.f);
  if (threadIdx.x == 0) *scale_out = scale;
  uint4* qr = reinterpret_cast<uint4*>(q);
  for (int c = threadIdx.x; c < (K >> 4); c += QUANT_THREADS) {
    float a[8], b[8];
    unpack8(srow[2 * c], a);
    unpack8(srow[2 * c + 1], b);
    qr[c] = make_uint4(e4m3x4(a, scale), e4m3x4(a + 4, scale), e4m3x4(b, scale), e4m3x4(b + 4, scale));
  }
}

__global__ void __launch_bounds__(QUANT_THREADS) quant_rows_e4m3_kernel(const __nv_bfloat16* __restrict__ x, int64_t ld, int K,
                                                                       uint8_t* __restrict__ q, float* __restrict__ scale) {
  extern __shared__ uint4 srow[];
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ld);
  float m = 0.f;
  for (int v = threadIdx.x; v < (K >> 3); v += QUANT_THREADS) {
    const uint4 u = ldg_nc_v4(xr + v);
    srow[v] = u;
    m = amax8(u, m);
  }
  m = block_max_nan(m, red);                 // its barriers also publish srow
  convert_row(srow, K, m, q + row * K, scale + row);
}

// Qwen2RMSNorm with the decoder layer's residual add fused in, as rmsnorm_fwd_kernel of elementwise.cu computes it -- the same
// per-thread order of the sum of squares (128 threads, 8-element vectors strided by the CTA), the same block reduction, the same bf16
// roundings: y = bf16(w * bf16(x' * rstd)), x' = bf16(x + res) -- with y quantised instead of written.
__global__ void __launch_bounds__(QUANT_THREADS) rmsnorm_quant_e4m3_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                                                                          const __nv_bfloat16* __restrict__ w, int H, float eps,
                                                                          uint8_t* __restrict__ q, float* __restrict__ scale,
                                                                          __nv_bfloat16* __restrict__ x_out) {
  extern __shared__ uint4 srow[];
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int hv = H >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
  const uint4* rr = res ? reinterpret_cast<const uint4*>(res + row * H) : nullptr;
  uint4* xo = x_out ? reinterpret_cast<uint4*>(x_out + row * H) : nullptr;
  float ss = 0.f;
  for (int v = threadIdx.x; v < hv; v += QUANT_THREADS) {
    uint4 u = ldg_nc_v4(xr + v);
    float f[8];
    unpack8(u, f);
    if (rr) {
      float g[8];
      unpack8(ldg_nc_v4(rr + v), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = bf16_round(f[j] + g[j]);
      u = pack8(f);
    }
    if (xo) xo[v] = u;
    srow[v] = u;                             // each thread reads back only what it wrote until the block reduction below
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)H + eps);
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  float m = 0.f;
  for (int v = threadIdx.x; v < hv; v += QUANT_THREADS) {
    float f[8], wf[8];
    unpack8(srow[v], f);
    unpack8(__ldg(wr + v), wf);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = wf[j] * bf16_round(f[j] * rstd);
    const uint4 y = pack8(f);
    srow[v] = y;
    m = amax8(y, m);
  }
  m = block_max_nan(m, red);
  convert_row(srow, H, m, q + row * H, scale + row);
}

template <typename Kern>
int row_smem(Kern kern, bool* done) {
  if (!*done) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, QUANT_MAX_K * 2));
    *done = true;
  }
  return LMOD_OK;
}

}  // namespace

// q[M,K] (e4m3 bytes, row stride K), scale[M] = quantise the rows of x [M,K] bf16 (row stride ld) as the header of this file states.
// The input of o_proj (the attention output) and of down_proj (the SwiGLU activation) of an FP8 teacher layer, and its weights at
// switch-on.  K % 16 == 0, ld % 8 == 0, x and q 16-byte aligned.
extern "C" int lmod_quant_rows_e4m3(const void* x, int64_t ld, void* q, float* scale, int64_t M, int64_t K, void* stream) {
  LMOD_CHECK_ARG(x && q && scale && M > 0 && K > 0, "lmod_quant_rows_e4m3: null pointer or empty problem");
  LMOD_CHECK_ARG(K % 16 == 0 && K <= QUANT_MAX_K && ld % 8 == 0 && ld >= K && (uintptr_t)x % 16 == 0 && (uintptr_t)q % 16 == 0,
                 "lmod_quant_rows_e4m3: K must be a multiple of 16 up to %d, ld a multiple of 8, pointers 16-byte aligned", QUANT_MAX_K);
  static bool attr = false;
  if (int rc = row_smem(quant_rows_e4m3_kernel, &attr)) return rc;
  quant_rows_e4m3_kernel<<<(unsigned)M, QUANT_THREADS, (size_t)K * 2, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, ld, (int)K, (uint8_t*)q, scale);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

// lmod_rmsnorm_fwd (Qwen2RMSNorm, modeling_qwen2.py:105-110, residual add of :796,808 fused in) whose normalised row goes out as e4m3
// bytes q [rows,H] + scale [rows] instead of bf16: bit-equal to lmod_quant_rows_e4m3(lmod_rmsnorm_fwd(...)); x_out as there.  Feeds the
// q|k|v and gate|up projections of an FP8 teacher layer.  H % 16 == 0.
extern "C" int lmod_rmsnorm_quant_e4m3(const void* x, const void* res, const void* w, int64_t rows, int64_t H, float eps, void* q, float* scale,
                                       void* x_out, void* stream) {
  LMOD_CHECK_ARG(x && w && q && scale && rows > 0 && H > 0 && H % 16 == 0 && H <= QUANT_MAX_K,
                 "lmod_rmsnorm_quant_e4m3: bad arguments (H %% 16 == 0, H <= %d required)", QUANT_MAX_K);
  static bool attr = false;
  if (int rc = row_smem(rmsnorm_quant_e4m3_kernel, &attr)) return rc;
  rmsnorm_quant_e4m3_kernel<<<(unsigned)rows, QUANT_THREADS, (size_t)H * 2, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x, (const __nv_bfloat16*)res, (const __nv_bfloat16*)w, (int)H, eps, (uint8_t*)q, scale, (__nv_bfloat16*)x_out);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
