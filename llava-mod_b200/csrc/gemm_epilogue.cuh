// gemm_epilogue.cuh -- what the wgmma GEMM kernels share besides sm90.cuh: the tile height and the epilogue device
// functions (bias, RoPE, SwiGLU, the 16-byte store transpose).  Included by gemm.cu (bf16) and gemm_fp8.cu (e4m3), so that the fused
// epilogues of both round exactly alike.
#pragma once
#include "sm90.cuh"

namespace {

constexpr int BM = 128;

// The epilogue starts from what one thread holds of a wgmma accumulator: two adjacent columns (col, col + 1) of one row.  Whatever is
// rounded to bf16 first (or, where nothing is, the fp32 words) is traded across the quad with quad_transpose, after which each lane holds
// 8 consecutive columns of the row; the functions below finish the element-wise work on such a block, loading their side inputs and
// storing their outputs 16 bytes at a time.  Every operation after the first rounding is per element, so this is exact.
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ void bias2(const __nv_bfloat16* b, float& f0, float& f1) {
  const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(b));
  f0 += bf16lo(w); f1 += bf16hi(w);
}
__device__ __forceinline__ void unpack8w(const uint32_t (&w)[4], float (&f)[8]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) { f[2 * j] = bf16lo(w[j]); f[2 * j + 1] = bf16hi(w[j]); }
}
__device__ __forceinline__ void unpack8v(const uint4 v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  unpack8w(w, f);
}
__device__ __forceinline__ uint4 pack8v(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}
// 16-byte stores.  st16 is a plain C++ store, which leaves the compiler free to move the next block's loads (bias, cos / sin, side
// inputs) ahead of it; st16_asm is one st.global.v4 whatever the compiler would make of the words -- the e4m3 kernel's compiler splits
// the C++ store of its RoPE and SwiGLU blocks into four 32-bit ones.
__device__ __forceinline__ void st16(__nv_bfloat16* d, const uint4 v) { *reinterpret_cast<uint4*>(d) = v; }
__device__ __forceinline__ void st16_asm(__nv_bfloat16* d, const uint4 v) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" :: "l"(d), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}
// rotate 8 (x1, x2) column pairs of a head, x1 / x2 = bf16(acc + bias) of the first-half / second-half block:
// o1 = bf16(bf16(x1 c) + bf16(-x2 s)), o2 = bf16(bf16(x2 c) + bf16(x1 s)) (the expression of rope_vec_kernel).  cs / sn: the 8 first-half
// columns of the cos / sin row of the position.
__device__ __forceinline__ void rope8(const uint32_t (&w1)[4], const uint32_t (&w2)[4], const __nv_bfloat16* cs, const __nv_bfloat16* sn,
                                      uint4& r1, uint4& r2) {
  float x1[8], x2[8], c[8], s[8], o1[8], o2[8];
  unpack8w(w1, x1); unpack8w(w2, x2);
  unpack8v(__ldg(reinterpret_cast<const uint4*>(cs)), c);
  unpack8v(__ldg(reinterpret_cast<const uint4*>(sn)), s);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o1[j] = bf16_round(x1[j] * c[j]) + bf16_round(-x2[j] * s[j]);
    o2[j] = bf16_round(x2[j] * c[j]) + bf16_round(x1[j] * s[j]);
  }
  r1 = pack8v(o1);
  r2 = pack8v(o2);
}
// act = bf16(bf16(silu(g)) * u) of one packed column pair of the bf16-rounded GEMM outputs: the expression of silu_mul_fwd_kernel
// (bit-identical to GEMM + that kernel).  Computed before the transpose, so that only the activation has to be traded.
__device__ __forceinline__ uint32_t swiglu2(const uint32_t wg, const uint32_t wu) {
  const float g0 = bf16lo(wg), g1 = bf16hi(wg);
  return pack_bf16x2(bf16_round(g0 * sigmoid_f(g0)) * bf16lo(wu), bf16_round(g1 * sigmoid_f(g1)) * bf16hi(wu));
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
