// sm90.cuh -- shared wgmma / TMA / mbarrier helpers for the hand-written tensor-core kernels (gemm.cu, attn.cu, attn_bwd.cu).  sm_90a.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "sm90_wgmma.cuh"

namespace {

// ---------------------------------------------------------------------------------------------------------------------------------
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes (or ~20 us pass) instead of spinning through
// issue slots the math warps need; the spin bound (~2.6 s) turns a protocol bug into a trap instead of a hung GPU.
// No printf (or any other call) here: a call anywhere in a wgmma kernel makes ptxas serialize every MMA in it (C7510).
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t phase) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase), "r"(20000u) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t phase) {
  if (mbar_try_wait(bar, phase)) return;
  uint32_t spins = 0;
  while (!mbar_try_wait_hint(bar, phase)) {
    if (++spins > (1u << 17)) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               :: "r"(smem_u32(smem_dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

// wgmma shared-memory matrix descriptor (sm_90): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout SWIZZLE_128B = 1 [62,64).
// K-major 128B-swizzled tile (rows x 64 bf16, 8-row atoms of 1024 B): LBO unused, SBO = 1024, +32 B per 16-element k step.
// MN-major 128B-swizzled tile (blocks of 64 mn x k rows): LBO = bytes between 64-wide mn blocks, SBO = 1024 (8 k rows), +2048 B per k step.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// keeps the compiler from moving register reads / writes of an accumulator across the asynchronous MMAs that own it
template <int N>
__device__ __forceinline__ void reg_fence(float* d) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}
template <int N>
__device__ __forceinline__ void reg_fence_u(uint32_t* d) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i]) :: "memory");
}
// register re-allocation between warpgroups: the TMA warpgroup gives registers back, the math warpgroups take them
template <int R> __device__ __forceinline__ void regs_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(R)); }
template <int R> __device__ __forceinline__ void regs_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(R)); }
// named barrier over the `n` threads of the math warpgroups
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(n) : "memory"); }

// ---- host: TMA tensor maps ------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D bf16 tensor map over a row-major [outer, inner] matrix with row stride ld (elements), 128B swizzle, zero fill out of bounds
int make_map(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner, uint32_t box_outer) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { lmod_set_error("cuTensorMapEncodeTiled entry point not available"); return LMOD_ERR_CUDA; }
  // cuTensorMapEncodeTiled is a DRIVER call: a thread that has not touched the CUDA runtime yet (autograd's backward thread, when one of
  // our GEMMs is the first thing it runs) has no current context and gets CUDA_ERROR_INVALID_CONTEXT; a runtime call binds the primary one
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { (void)cudaFree(nullptr); ctx_bound = true; }
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstr[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { lmod_set_error("cuTensorMapEncodeTiled failed (%d): inner=%llu outer=%llu ld=%llu", (int)r, (unsigned long long)inner,
                                          (unsigned long long)outer, (unsigned long long)ld); return LMOD_ERR_CUDA; }
  return LMOD_OK;
}

}  // namespace
