// gemm_fp8.cu -- e4m3 wgmma + TMA GEMM for sm_90a, forward only:  D[m,n] = s_a[m] * s_w[n] * sum_k a8[m,k] * w8[n,k]
//
// The decoder linears of a frozen FP8 teacher (modeling_qwen2.py:678-680 q/k/v, :726 o_proj, :199-200 gate/up/down): a8 [M,K] are the
// activation rows quantised per token (quant.cu), w8 [N,K] the weight quantised per output channel at switch-on, both e4m3 bytes stored
// K-major -- the one operand form 8-bit wgmma has.  The epilogue computes (acc * s_a[m]) * s_w[n] in fp32, in that order, and then
// continues exactly as gemm.cu does from its accumulator: (+bias) -> bf16, or the RoPE / SwiGLU expressions of gemm_epilogue.cuh.
//
// Accumulation.  The 8-bit MMA of sm_90 does not keep a full fp32 running sum: it aligns the addends of an instruction to the largest
// one and drops what falls below about 13 fractional bits, towards zero.  Left alone over K = 4096 that is a biased error of 1.6 % of
// sum|a||w| on same-signed products (4 bf16 ulps; measured, DESIGN.md section 4).  So the wgmma accumulator only ever holds PROMOTE_KB
// k-blocks (512 elements): then it is drained, added into a second register set with ordinary fp32 adds, and restarted.  Two register
// sets of 64 per thread are what fits, hence 128-column tiles only.
//
// Structure: gemm_wgmma_kernel's (gemm.cu) -- one persistent CTA per SM, 384 threads; warpgroup 0's thread 0 is the TMA producer,
// warpgroups 1 and 2 each own 64 rows of the 128 x BN tile, full / empty mbarrier ring, one k-block of MMAs in flight while the previous
// stage is handed back.  A stage row is 128 one-byte elements: the same 128-byte swizzled rows and stage bytes as the bf16 kernel, so the
// ring depth is that of its 128-column tiles (6 stages), and a k-block is four wgmma m64n128k32.
// Not here, on purpose: MN-major operands, split-K, grouped rows, accumulation into D, device extents -- nothing frozen uses them.
#include "gemm_epilogue.cuh"

namespace {

constexpr int BK8 = 128;                              // one-byte elements per stage row
constexpr int BN8 = 128;                              // accumulator columns per tile
constexpr int A8_STAGE_BYTES = BM * BK8;              // 16 KB
constexpr int STAGES8 = 6;
constexpr int STAGE8_BYTES = A8_STAGE_BYTES + BN8 * BK8;
constexpr int SMEM8 = STAGES8 * STAGE8_BYTES + 1024;  // + alignment slack
constexpr int PROMOTE_KB = 4;                         // k-blocks summed inside the tensor core before the fp32 promotion
constexpr int GEMM8_THREADS = 384;

struct Fp8Params {
  __nv_bfloat16* D;
  int64_t ldd;
  const __nv_bfloat16* bias;       // [N] or null
  const float* sa;                 // [M] activation scales
  const float* sw;                 // [N] weight scales ([2I] for the SwiGLU form)
  int M, N, K;
  int bn;                          // output columns per tile
  // fused SwiGLU: W is the fused gate|up weight [2I, K]; N = I; a tile is 64 act columns whose accumulator holds [64 gate | 64 up]
  int swiglu_I;                    // 0 = off
  // fused rotary embedding of the q|k|v projection (see GemmParams of gemm.cu)
  const __nv_bfloat16* rope_cos;
  const __nv_bfloat16* rope_sin;
  const int64_t* rope_pos;
  int rope_hd, rope_cols;
};

// tile index -> (m0, n0): M fastest, so that consecutive CTAs share the weight tile in L2
__device__ __forceinline__ bool get_tile8(const Fp8Params& p, int t, int& m0, int& n0) {
  const int num_m = (p.M + BM - 1) / BM, num_n = (p.N + p.bn - 1) / p.bn;
  if (t >= num_m * num_n) return false;
  m0 = (t % num_m) * BM; n0 = (t / num_m) * p.bn;
  return true;
}

__device__ __forceinline__ void mma_kblock8(float* acc, uint32_t sa, uint32_t sb, uint32_t accumulate) {
#pragma unroll
  for (int k = 0; k < BK8 / 32; ++k) {
    const uint64_t da = gmma_desc(sa + k * 32, 16, 1024), db = gmma_desc(sb + k * 32, 16, 1024);
    wgmma_e4m3_ss_n128(acc, da, db, (k > 0) ? 1u : accumulate);
  }
}

__device__ __forceinline__ float2 scale2(const float* sw, int col, int n) {
  return col < n ? __ldg(reinterpret_cast<const float2*>(sw + col)) : make_float2(0.f, 0.f);
}

__global__ void __launch_bounds__(GEMM8_THREADS, 1)
gemm_e4m3_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const Fp8Params p) {
  constexpr int BN = BN8, STAGES = STAGES8, STAGE_BYTES = STAGE8_BYTES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);   // SW128 needs 1024 B
  const int wg = threadIdx.x >> 7;
  const int nk = (p.K + BK8 - 1) / BK8;                    // TMA zero-fills the tail of a K that is not a multiple of 128

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    mbar_fence_init();
    asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_b) : "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      int m0, n0;
      for (int ti = blockIdx.x; get_tile8(p, ti, m0, n0); ti += gridDim.x) {
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait_bounded(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A8_STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          tma_load_2d(sa, &tma_a, kb * BK8, m0, &full_bar[stage]);                         // box (128 k, 128 rows)
          if (p.swiglu_I) {                                                                // box (128 k, 64 rows): gate rows, then the matching up rows
            tma_load_2d(sb, &tma_b, kb * BK8, n0, &full_bar[stage]);
            tma_load_2d(sb + 64 * BK8, &tma_b, kb * BK8, p.swiglu_I + n0, &full_bar[stage]);
          } else {
            tma_load_2d(sb, &tma_b, kb * BK8, n0, &full_bar[stage]);                       // box (128 k, BN rows)
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  // ===================== math warpgroups: MMA + epilogue =====================
  regs_alloc<232>();
  const int c = wg - 1;                                    // rows [64c, 64c + 64) of every tile
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  float part[BN / 2], acc[BN / 2];                         // the tensor core's partial sum of up to PROMOTE_KB k-blocks; the fp32 total
  uint32_t stage = 0, phase = 0;
  int m0, n0;
  for (int ti = blockIdx.x; get_tile8(p, ti, m0, n0); ti += gridDim.x) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kg = 0; kg < nk; kg += PROMOTE_KB) {
      const int n = min(PROMOTE_KB, nk - kg);
      uint32_t prev = 0;
      for (int j = 0; j < n; ++j) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + c * (64 * BK8), sb = smem_u32(smem + stage * STAGE_BYTES + A8_STAGE_BYTES);
        wgmma_fence();
        mma_kblock8(part, sa, sb, j > 0 ? 1u : 0u);
        wgmma_commit();
        if (j > 0) {                                       // the previous k-block's MMAs are done: hand its stage back
          wgmma_wait<1>();
          if (wg_leader) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();                                     // on every path, before the registers are read (a conditional wait: C7517)
      if (wg_leader) mbar_arrive(&empty_bar[prev]);
      reg_fence<BN / 2>(part);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
    }

    // accumulator fragment: register 4i + 2h + e holds row 16w + lane/4 + 8h, column 8i + 2(lane%4) + e of this warpgroup's 64 x BN block.
    // The forms are those of gemm_wgmma_kernel on the scaled accumulators (acc * s_a[m]) * s_w[n]: each rounds to bf16, trades the packed
    // column pairs of a transpose group (4 blocks of 8 columns) across the quad, and stores 16-byte blocks.
    const int row0 = m0 + c * 64 + w * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3), q = lane & 3;
    const float sar[2] = {row0 < p.M ? __ldg(p.sa + row0) : 0.f, row0 + 8 < p.M ? __ldg(p.sa + row0 + 8) : 0.f};
    if (p.swiglu_I) {
      // accumulator columns [0,64) = gate, [64,128) = up of the same 64 act columns (I % 128 == 0: all in range)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        float2 sg[4], su[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = n0 + 8 * (4 * k + j) + cq;
          sg[j] = scale2(p.sw, col, p.N); su[j] = scale2(p.sw + p.swiglu_I, col, p.N);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t wa[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int i = 4 * k + j;
            wa[j] = swiglu2(pack_bf16x2(acc[4 * i + 2 * h] * sar[h] * sg[j].x, acc[4 * i + 2 * h + 1] * sar[h] * sg[j].y),
                            pack_bf16x2(acc[4 * (i + 8) + 2 * h] * sar[h] * su[j].x, acc[4 * (i + 8) + 2 * h + 1] * sar[h] * su[j].y));
          }
          quad_transpose(wa, q);
          const int row = row0 + 8 * h;
          if (row < p.M) st16_asm(p.D + (int64_t)row * p.ldd + n0 + 8 * (4 * k + q), make_uint4(wa[0], wa[1], wa[2], wa[3]));
        }
      }
      continue;
    }
    int64_t pos[2] = {0, 0};                               // the rotary positions of the thread's two rows
    if (p.rope_cos) {
#pragma unroll
      for (int h = 0; h < 2; ++h) if (row0 + 8 * h < p.M) pos[h] = __ldg(p.rope_pos + row0 + 8 * h);
    }
#pragma unroll
    for (int k = 0; k < BN / 32; ++k) {
      const int cg = n0 + 32 * k;                          // first column of the group (the same in every lane)
      if (cg >= p.N) continue;
      if (p.rope_cos && cg < p.rope_cols) {
        // q / k head columns: a group of the first half of a head is rotated together with its partner group half a head further on
        // (k + 2 for hd 128, k + 1 for hd 64; a head never straddles a tile); the partner is skipped
        const int half = p.rope_hd >> 1, hoff = cg % p.rope_hd;
        if (hoff >= half) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t w1[4], w2[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int i1 = 4 * k + j, col = n0 + 8 * i1 + cq;
            const int i2a = (i1 + 4) % (BN / 8), i2b = (i1 + 8) % (BN / 8);
            const float2 s1 = scale2(p.sw, col, p.N), s2 = scale2(p.sw, col + half, p.N);
            const float a20 = half == 32 ? acc[4 * i2a + 2 * h] : acc[4 * i2b + 2 * h];
            const float a21 = half == 32 ? acc[4 * i2a + 2 * h + 1] : acc[4 * i2b + 2 * h + 1];
            float x10 = acc[4 * i1 + 2 * h] * sar[h] * s1.x, x11 = acc[4 * i1 + 2 * h + 1] * sar[h] * s1.y;
            float x20 = a20 * sar[h] * s2.x, x21 = a21 * sar[h] * s2.y;
            if (p.bias) { bias2(p.bias + col, x10, x11); bias2(p.bias + col + half, x20, x21); }
            w1[j] = pack_bf16x2(x10, x11);
            w2[j] = pack_bf16x2(x20, x21);
          }
          quad_transpose(w1, q);
          quad_transpose(w2, q);
          const int row = row0 + 8 * h;
          if (row >= p.M) continue;
          const int64_t cs = pos[h] * p.rope_hd + hoff + 8 * q;
          __nv_bfloat16* d = p.D + (int64_t)row * p.ldd + cg + 8 * q;
          uint4 o1, o2;
          rope8(w1, w2, p.rope_cos + cs, p.rope_sin + cs, o1, o2);
          st16_asm(d, o1);
          st16_asm(d + half, o2);
        }
        continue;
      }
      // plain bf16 output (+bias)
      float2 s[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) s[j] = scale2(p.sw, cg + 8 * j + cq, p.N);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t wd[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = cg + 8 * j + cq;
          float f0 = acc[4 * (4 * k + j) + 2 * h] * sar[h] * s[j].x, f1 = acc[4 * (4 * k + j) + 2 * h + 1] * sar[h] * s[j].y;
          if (p.bias && col < p.N) bias2(p.bias + col, f0, f1);
          wd[j] = pack_bf16x2(f0, f1);
        }
        quad_transpose(wd, q);
        const int row = row0 + 8 * h, col8 = cg + 8 * q;
        if (row < p.M && col8 < p.N) st16(p.D + (int64_t)row * p.ldd + col8, make_uint4(wd[0], wd[1], wd[2], wd[3]));
      }
    }
  }
}

// 2-D tensor map over a row-major [outer, inner] matrix of bytes with row stride ld, 128B swizzle, zero fill out of bounds
int make_map_u8(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner, uint32_t box_outer) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { lmod_set_error("cuTensorMapEncodeTiled entry point not available"); return LMOD_ERR_CUDA; }
  static thread_local bool ctx_bound = false;              // see make_map: the driver call needs a current context
  if (!ctx_bound) { (void)cudaFree(nullptr); ctx_bound = true; }
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstr[1] = {ld};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { lmod_set_error("cuTensorMapEncodeTiled failed (%d): inner=%llu outer=%llu ld=%llu (bytes)", (int)r,
                                          (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld); return LMOD_ERR_CUDA; }
  return LMOD_OK;
}

int launch8(const CUtensorMap& ta, const CUtensorMap& tb, const Fp8Params& p, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(gemm_e4m3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM8));
    attr = true;
  }
  const int tiles = ((p.M + BM - 1) / BM) * ((p.N + p.bn - 1) / p.bn);
  const int grid = tiles < lmod_num_sms() ? tiles : lmod_num_sms();
  gemm_e4m3_kernel<<<grid, GEMM8_THREADS, SMEM8, st>>>(ta, tb, p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

struct Rope8 { const void* cos; const void* sin; const int64_t* pos; int hd; int cols; };

// swiglu_I != 0: W has 2I rows and a tile is 64 act columns (64 gate + 64 up accumulator columns)
int gemm8(const char* who, const void* A, int64_t lda, const float* sa, const void* W, int64_t ldb, const float* sw, const void* bias, void* D,
          int64_t ldd, int64_t M, int64_t N, int64_t K, int64_t swiglu_I, const Rope8* rope, cudaStream_t st) {
  LMOD_CHECK_ARG(A && sa && W && sw && D && M > 0 && N > 0 && K > 0, "%s: null pointer or empty problem", who);
  LMOD_CHECK_ARG(K % 16 == 0 && lda % 16 == 0 && ldb % 16 == 0 && ldd % 8 == 0 && N % 8 == 0 && (uintptr_t)A % 16 == 0 && (uintptr_t)W % 16 == 0 &&
                 (uintptr_t)D % 16 == 0 && (uintptr_t)sw % 8 == 0,
                 "%s: K and the e4m3 row strides must be multiples of 16, N and ldd of 8, pointers 16-byte aligned (TMA, 16-byte stores)", who);
  LMOD_CHECK_ARG((uintptr_t)bias % 4 == 0 && (!rope || ((uintptr_t)rope->cos % 4 == 0 && (uintptr_t)rope->sin % 4 == 0)),
                 "%s: bias, cos and sin must be 4-byte aligned (the epilogue reads bias two bf16 at a time)", who);
  LMOD_CHECK_ARG(!rope || ((uintptr_t)rope->cos % 16 == 0 && (uintptr_t)rope->sin % 16 == 0 && rope->hd % 8 == 0),
                 "%s: cos and sin must be 16-byte aligned and head_dim a multiple of 8 (the epilogue reads them 8 bf16 at a time)", who);
  Fp8Params p = {};
  p.D = (__nv_bfloat16*)D; p.ldd = ldd; p.bias = (const __nv_bfloat16*)bias; p.sa = sa; p.sw = sw;
  p.M = (int)M; p.N = (int)N; p.K = (int)K; p.swiglu_I = (int)swiglu_I;
  p.bn = swiglu_I ? BN8 / 2 : BN8;
  if (rope) { p.rope_cos = (const __nv_bfloat16*)rope->cos; p.rope_sin = (const __nv_bfloat16*)rope->sin; p.rope_pos = rope->pos; p.rope_hd = rope->hd; p.rope_cols = rope->cols; }
  CUtensorMap ta, tb;
  if (int rc = make_map_u8(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK8, BM)) return rc;
  if (int rc = make_map_u8(&tb, W, (uint64_t)K, (uint64_t)(swiglu_I ? 2 * swiglu_I : N), (uint64_t)ldb, BK8, p.bn)) return rc;
  return launch8(ta, tb, p, st);
}

}  // namespace

// D[M,N] = bf16( s_a[m] s_w[n] (A8 W8^T)[m,n] + bias[n] ): nn.Linear forward of a frozen decoder projection (o_proj modeling_qwen2.py:726,
// down_proj :200; q|k|v and gate|up when their fused forms below do not apply) on e4m3 operands.  A8 [M,K] / W8 [N,K] e4m3 bytes with
// row strides lda / ldb (bytes); s_a [M], s_w [N] fp32; bias [N] bf16 or NULL.
extern "C" int lmod_gemm_e4m3(const void* A8, int64_t lda, const float* s_a, const void* W8, int64_t ldb, const float* s_w, const void* bias,
                              void* D, int64_t ldd, int64_t M, int64_t N, int64_t K, void* stream) {
  return gemm8("lmod_gemm_e4m3", A8, lda, s_a, W8, ldb, s_w, bias, D, ldd, M, N, K, 0, nullptr, (cudaStream_t)stream);
}

// lmod_gemm_qkv_rope on e4m3 operands (Qwen2Attention q/k/v_proj + apply_rotary_pos_emb, modeling_qwen2.py:678-691,159-184).
// Bit-identical to lmod_gemm_e4m3 + lmod_rope.  hd in {64, 128}.
extern "C" int lmod_gemm_e4m3_qkv_rope(const void* A8, int64_t lda, const float* s_a, const void* W8, int64_t ldb, const float* s_w,
                                       const void* bias, void* D, int64_t ldd, int64_t M, int64_t K, int nh, int nkv, int hd,
                                       const void* cos_table, const void* sin_table, const int64_t* position_ids, void* stream) {
  LMOD_CHECK_ARG(cos_table && sin_table && position_ids && nh > 0 && nkv > 0, "lmod_gemm_e4m3_qkv_rope: null pointer");
  LMOD_CHECK_ARG(hd == 64 || hd == 128, "lmod_gemm_e4m3_qkv_rope: head_dim %d not fused (64 and 128 are; use lmod_gemm_e4m3 + lmod_rope)", hd);
  Rope8 r = {cos_table, sin_table, position_ids, hd, (nh + nkv) * hd};
  return gemm8("lmod_gemm_e4m3_qkv_rope", A8, lda, s_a, W8, ldb, s_w, bias, D, ldd, M, (int64_t)(nh + 2 * nkv) * hd, K, 0, &r, (cudaStream_t)stream);
}

// lmod_gemm_swiglu on e4m3 operands (Qwen2MLP act_fn(gate_proj(x)) * up_proj(x), modeling_qwen2.py:199-200), forward only, so no
// pre-activations are kept: W8_gu [2I,K] and s_w [2I] are the fused gate|up weight as quantised (gate rows, then up rows).
// Bit-identical to lmod_gemm_e4m3 + lmod_silu_mul_fwd.  I % 128 == 0.
extern "C" int lmod_gemm_e4m3_swiglu(const void* A8, int64_t lda, const float* s_a, const void* W8_gu, int64_t ldb, const float* s_w, void* act,
                                     int64_t ld_act, int64_t M, int64_t I, int64_t K, void* stream) {
  LMOD_CHECK_ARG(I > 0 && I % 128 == 0, "lmod_gemm_e4m3_swiglu: intermediate size %lld is not a multiple of 128 (use lmod_gemm_e4m3 + lmod_silu_mul_fwd)",
                 (long long)I);
  return gemm8("lmod_gemm_e4m3_swiglu", A8, lda, s_a, W8_gu, ldb, s_w, nullptr, act, ld_act, M, I, K, I, nullptr, (cudaStream_t)stream);
}
