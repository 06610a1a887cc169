// gemm_epilogue.cuh -- what the wgmma GEMM kernels share besides sm90.cuh: the tile height and the epilogue device
// functions (bias, RoPE, SwiGLU, the 16-byte store transpose).  Included by gemm.cu (bf16) and gemm_fp8.cu (e4m3), so that the fused
// epilogues of both round exactly alike.
#pragma once
#include "sm90.cuh"

namespace {

constexpr int BM = 128;

// The epilogue works on what one thread holds of a wgmma accumulator: two adjacent columns (col, col + 1) of one row.
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ void bias2(const __nv_bfloat16* b, float& f0, float& f1) {
  const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(b));
  f0 += bf16lo(w); f1 += bf16hi(w);
}
// rotate one (x1, x2) pair of columns of a head: x = bf16(acc + bias); o1 = bf16(bf16(x1 c) + bf16(-x2 s)), o2 = bf16(bf16(x2 c) + bf16(x1 s))
// (the expression of rope_vec_kernel).  a1 / a2: fp32 accumulators of the first-half / second-half columns, b1 / b2: their bias (or null).
__device__ __forceinline__ void rope_store2(float a10, float a11, float a20, float a21, const __nv_bfloat16* b1, const __nv_bfloat16* b2,
                                            const __nv_bfloat16* cs, const __nv_bfloat16* sn, __nv_bfloat16* d1, __nv_bfloat16* d2) {
  float x1[2] = {a10, a11}, x2[2] = {a20, a21};
  if (b1) { bias2(b1, x1[0], x1[1]); bias2(b2, x2[0], x2[1]); }
  const uint32_t cw = __ldg(reinterpret_cast<const uint32_t*>(cs)), sw = __ldg(reinterpret_cast<const uint32_t*>(sn));
  const float c[2] = {bf16lo(cw), bf16hi(cw)}, s[2] = {bf16lo(sw), bf16hi(sw)};
  float o1[2], o2[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float y1 = bf16_round(x1[j]), y2 = bf16_round(x2[j]);
    o1[j] = bf16_round(y1 * c[j]) + bf16_round(-y2 * s[j]);
    o2[j] = bf16_round(y2 * c[j]) + bf16_round(y1 * s[j]);
  }
  *reinterpret_cast<uint32_t*>(d1) = pack_bf16x2(o1[0], o1[1]);
  *reinterpret_cast<uint32_t*>(d2) = pack_bf16x2(o2[0], o2[1]);
}
// act = bf16(bf16(silu(g)) * u) on bf16-rounded GEMM outputs: the expression of silu_mul_fwd_kernel (bit-identical to GEMM + that kernel)
__device__ __forceinline__ void swiglu_store2(float g0, float g1, float u0, float u1, __nv_bfloat16* act, __nv_bfloat16* h1g, __nv_bfloat16* h1u) {
  const float gb[2] = {bf16_round(g0), bf16_round(g1)}, ub[2] = {bf16_round(u0), bf16_round(u1)};
  float f[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) f[j] = bf16_round(gb[j] * sigmoid_f(gb[j])) * ub[j];
  *reinterpret_cast<uint32_t*>(act) = pack_bf16x2(f[0], f[1]);
  if (h1g) {
    *reinterpret_cast<uint32_t*>(h1g) = pack_bf16x2(gb[0], gb[1]);
    *reinterpret_cast<uint32_t*>(h1u) = pack_bf16x2(ub[0], ub[1]);
  }
}
// 4 x 4 transpose within each quad of lanes: lane q holds w[j] = word j of its own; afterwards w[j] = word q of lane j (the lane index
// within the quad is q).  The sender picks the word its receiver needs, so no register is indexed dynamically.
__device__ __forceinline__ uint32_t pick4(const uint32_t (&w)[4], int i) { return i == 0 ? w[0] : i == 1 ? w[1] : i == 2 ? w[2] : w[3]; }
__device__ __forceinline__ void quad_transpose(uint32_t (&w)[4], int q) {
  uint32_t o[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int s = (q + r) & 3;                               // lane s sends its word q, chosen there as word (s - r) & 3
    const uint32_t v = r == 0 ? pick4(w, q) : __shfl_sync(0xffffffffu, pick4(w, (q - r) & 3), s, 4);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = (j == s) ? v : (r == 0 ? 0u : o[j]);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) w[j] = o[j];
}

}  // namespace
