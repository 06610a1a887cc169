// attn_bwd.cu -- flash-attention BACKWARD on wgmma / TMA (sm_90a).
//
// Backward of Qwen2SdpaAttention's scaled_dot_product_attention (modeling_qwen2.py:713-721) for the sparse student: given the fused
// RoPE'd QKV buffer, the forward output O, dO and the log-sum-exp of the forward kernel, produces dQ|dK|dV in one fused buffer.
//
// One CTA owns a block of 128 keys of one (batch, kv-head) and sweeps the 64-query blocks (and the query heads of its GQA group) that can
// see it.  Warpgroup 0 is the TMA producer (K_j, V_j once; Q_i / dO_i through a 2-stage ring); math warpgroups 1 and 2 own 64 keys each
// and keep their dK_j, dV_j accumulators in registers for the whole sweep.  Per (key block, query block):
//     S^T  = K_j Q_i^T,  dP^T = V_j dO_i^T      (wgmma, both operands from shared memory, M = 64 keys, N = 64 queries)
//     P^T  = exp2(S^T c - lse),  dS^T = P^T (dP^T - D) scale      (registers; lse / D per query column)
//     dV_j += P^T dO_i,  dK_j += dS^T Q_i       (wgmma, A = P^T / dS^T straight from registers, B = dO_i / Q_i MN-major)
//     dQ_i  = dS K_j                            (wgmma over all 128 keys, A = dS written to 128B-swizzled shared memory by both math
//                                                warpgroups, MN-major; B = K_j MN-major) -- computed by warpgroup 1 + (i mod 2) and
//                                                added into an fp32 workspace with red.global.add (a key block only holds a partial dQ)
#include "sm90.cuh"

namespace {

constexpr int BKVB = 128, BQB = 64;
constexpr int ATB_THREADS = 384;     // TMA warpgroup + two math warpgroups
constexpr int NQ = 2;                // Q_i / dO_i ring

struct AttnBwdParams {
  const float* lse;       // [B, nh, T]
  const float* dsum;      // [B, nh, T]  D = rowsum(dO * O)
  float* dq32;            // [B*T, nh*hd] fp32 workspace (zero-initialised)
  __nv_bfloat16* dqkv;    // fused gradient buffer; this kernel writes the k and v columns
  int64_t ld_dqkv, ld_dq32;
  int B, T, nh, nkv;
  int causal;
  float scale, scale_log2;
  const int32_t* kv_lo;   // padded batches: real key range per batch row (see attn.cu); NULL = no padding
  const int32_t* kv_hi;
};

__device__ __forceinline__ void red_add_v2(float* dst, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" :: "l"(dst), "f"(a), "f"(b) : "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_rs_b_mn(float* d, const uint32_t* a, uint64_t db, uint32_t acc) {
  if constexpr (N == 128) wgmma_rs_n128<1>(d, a, db, acc);
  else wgmma_rs_n64<1>(d, a, db, acc);
}

template <int HD>
__global__ void __launch_bounds__(ATB_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tma_kv, const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_do,
                const AttnBwdParams p) {
  constexpr int KSUB = HD / 64;
  constexpr int KV_BYTES = BKVB * HD * 2;              // one of K_j / V_j
  constexpr int Q_BYTES = BQB * HD * 2;                // one of Q_i / dO_i
  constexpr int DS_BYTES = BKVB * BQB * 2;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t kv_full, q_full[NQ], q_empty[NQ];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sK = smem;
  uint8_t* sV = sK + KV_BYTES;
  uint8_t* sQ = sV + KV_BYTES;                         // stage s: Q at sQ + s*2*Q_BYTES, dO right after
  uint8_t* sDS = sQ + NQ * 2 * Q_BYTES;                // 2 buffers of DS_BYTES (by iteration parity)
  const int wg = threadIdx.x >> 7;

  // heavy key blocks (small j under the causal mask) are scheduled first: j is the slowest grid index
  const int j = blockIdx.z, hk = blockIdx.x, b = blockIdx.y;
  const int group = p.nh / p.nkv;
  const int kv0 = j * BKVB;
  const int nq = (p.T + BQB - 1) / BQB;
  int lo = 0, hi = p.T;
  if (p.kv_lo) { lo = p.kv_lo[b]; hi = p.kv_hi[b]; }
  const bool all_pad = hi <= lo;
  const bool padded = (lo > 0) || (hi < p.T);
  // un-masked query rows (rows in front of a left-padded sequence see every key) make every query block a partner of this key block
  const int i_start = (p.causal && lo == 0 && !all_pad) ? (kv0 / BQB) : 0;
  const int n_i = nq - i_start;                        // query blocks per head for this key block
  const int n_it = n_i * group;
  const int row_base = b * p.T;
  const int col_k = (p.nh + hk) * HD, col_v = (p.nh + p.nkv + hk) * HD;

  if (threadIdx.x == 0) {
    mbar_init(&kv_full, 1);
    for (int s = 0; s < NQ; ++s) { mbar_init(&q_full[s], 1); mbar_init(&q_empty[s], 2); }
    mbar_fence_init();
    asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_kv) : "memory");
    asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_q) : "memory");
    asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_do) : "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    regs_dealloc<40>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(&kv_full, 2 * KV_BYTES);
#pragma unroll
      for (int i = 0; i < KSUB; ++i) {
        tma_load_2d(sK + i * (BKVB * 128), &tma_kv, col_k + 64 * i, row_base + kv0, &kv_full);
        tma_load_2d(sV + i * (BKVB * 128), &tma_kv, col_v + 64 * i, row_base + kv0, &kv_full);
      }
      for (int it = 0; it < n_it; ++it) {
        const int s = it % NQ;
        const int h = hk * group + it / n_i, qi = i_start + it % n_i;
        mbar_wait_bounded(&q_empty[s], ((it / NQ) & 1) ^ 1);
        uint8_t* q = sQ + s * 2 * Q_BYTES;
        uint8_t* d = q + Q_BYTES;
        mbar_expect_tx(&q_full[s], 2 * Q_BYTES);
#pragma unroll
        for (int i = 0; i < KSUB; ++i) {
          tma_load_2d(q + i * (BQB * 128), &tma_q, h * HD + 64 * i, row_base + qi * BQB, &q_full[s]);
          tma_load_2d(d + i * (BQB * 128), &tma_do, h * HD + 64 * i, row_base + qi * BQB, &q_full[s]);
        }
      }
    }
    return;
  }

  // ===================== math warpgroups =====================
  regs_alloc<232>();
  const int c = wg - 1;
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int kr = c * 64 + w * 16 + (lane >> 2);        // key row (within the block) of fragment rows h = 0; h = 1 is kr + 8
  const int cq = 2 * (lane & 3);
  const uint32_t aK = smem_u32(sK), aV = smem_u32(sV);
  float dk[HD / 2], dv[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
  mbar_wait(&kv_full, 0);
  for (int it = 0; it < n_it; ++it) {
    const int s = it % NQ, buf = it & 1;
    const int h = hk * group + it / n_i, qi = i_start + it % n_i;
    const int q0 = qi * BQB;
    const uint32_t aQ = smem_u32(sQ + s * 2 * Q_BYTES), aDO = aQ + Q_BYTES;
    const int64_t lbase = ((int64_t)b * p.nh + h) * p.T;
    // only the blocks on the causal diagonal and the ragged tail need per-element masks
    const bool masked = padded || (q0 + BQB > p.T) || (kv0 + BKVB > p.T) || (p.causal && q0 < kv0 + BKVB - 1);

    float sacc[32], dpacc[32];
    mbar_wait(&q_full[s], (it / NQ) & 1);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {
      const uint32_t ko = (k / 4), ki = (k % 4) * 32;
      wgmma_ss_n64<0, 0>(sacc, gmma_desc(aK + ko * (BKVB * 128) + c * (64 * 128) + ki, 16, 1024), gmma_desc(aQ + ko * (BQB * 128) + ki, 16, 1024), k > 0 ? 1u : 0u);
    }
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {
      const uint32_t ko = (k / 4), ki = (k % 4) * 32;
      wgmma_ss_n64<0, 0>(dpacc, gmma_desc(aV + ko * (BKVB * 128) + c * (64 * 128) + ki, 16, 1024), gmma_desc(aDO + ko * (BQB * 128) + ki, 16, 1024), k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<32>(sacc);
    reg_fence<32>(dpacc);

    // P^T, dS^T: fragment register 4i + 2hh + e = key kr + 8hh, query q0 + 8i + cq + e
    uint32_t pa[4][4], da[4][4];
    uint8_t* dsb = sDS + buf * DS_BYTES;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int qa = min(q0 + 8 * i + cq, p.T - 1), qb = min(q0 + 8 * i + cq + 1, p.T - 1);   // rows >= T are masked below
      const float2 l2 = make_float2(__ldg(p.lse + lbase + qa) * LOG2E_F, __ldg(p.lse + lbase + qb) * LOG2E_F);
      const float2 dd = make_float2(__ldg(p.dsum + lbase + qa), __ldg(p.dsum + lbase + qb));
      float pv[4], ds[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kv = kv0 + kr + 8 * (e >> 1), qidx = q0 + 8 * i + cq + (e & 1);
        bool ok = true;
        if (masked) {
          const bool seen = (all_pad || qidx < lo) ? true : (kv >= lo && kv < hi && (!p.causal || kv <= qidx));
          ok = (qidx < p.T) && (kv < p.T) && seen;
        }
        const float lsev = (e & 1) ? l2.y : l2.x, dsv = (e & 1) ? dd.y : dd.x;
        pv[e] = ok ? ex2f(fmaf(sacc[4 * i + e], p.scale_log2, -lsev)) : 0.f;
        ds[e] = pv[e] * (dpacc[4 * i + e] - dsv) * p.scale;
      }
      pa[i >> 1][(i & 1) * 2 + 0] = pack_bf16x2(pv[0], pv[1]);
      pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(pv[2], pv[3]);
      da[i >> 1][(i & 1) * 2 + 0] = pack_bf16x2(ds[0], ds[1]);
      da[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(ds[2], ds[3]);
      // dS for dQ = dS K: row = key, 64 queries contiguous (MN-major A operand), 128B swizzle (16-byte chunk ^ (row & 7))
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = kr + 8 * hh;
        *reinterpret_cast<uint32_t*>(dsb + row * 128 + ((i ^ (row & 7)) << 4) + 2 * cq) = da[i >> 1][(i & 1) * 2 + hh];
      }
    }
    fence_proxy_async();                               // generic-proxy smem writes -> visible to the tensor core (async proxy)
    named_bar(1, 256);                                 // both halves of dS are in shared memory

    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {                   // reduction over the 64 queries of the block
      wgmma_rs_b_mn<HD>(dv, pa[kk], gmma_desc(aDO + kk * 2048, BQB * 128, 1024), 1u);
      wgmma_rs_b_mn<HD>(dk, da[kk], gmma_desc(aQ + kk * 2048, BQB * 128, 1024), 1u);
    }
    wgmma_commit();
    if ((it & 1) == c) {
      // dQ_i = dS K_j over the 128 keys, 64 head-dim columns per pass
      const int row = q0 + w * 16 + (lane >> 2);
      float* dst = p.dq32 + (int64_t)(row_base + row) * p.ld_dq32 + h * HD + cq;
#pragma unroll
      for (int ps = 0; ps < KSUB; ++ps) {
        float dq[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKVB / 16; ++k)
          wgmma_ss_n64<1, 1>(dq, gmma_desc(smem_u32(dsb) + k * 2048, BQB * 128, 1024),
                             gmma_desc(aK + ps * (BKVB * 128) + k * 2048, BKVB * 128, 1024), k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence<32>(dq);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
            if (row + 8 * hh < p.T) red_add_v2(dst + (int64_t)8 * hh * p.ld_dq32 + ps * 64 + 8 * i, dq[4 * i + 2 * hh], dq[4 * i + 2 * hh + 1]);
      }
    }
    wgmma_wait<0>();
    reg_fence<HD / 2>(dv);
    reg_fence<HD / 2>(dk);
    reg_fence_u<16>(&pa[0][0]);
    reg_fence_u<16>(&da[0][0]);
    if (wg_leader) mbar_arrive(&q_empty[s]);
  }

  // ---- dK_j, dV_j epilogue ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int kv = kv0 + kr + 8 * hh;
    if (kv >= p.T) continue;
    __nv_bfloat16* dkrow = p.dqkv + (int64_t)(row_base + kv) * p.ld_dqkv + col_k + cq;
    __nv_bfloat16* dvrow = p.dqkv + (int64_t)(row_base + kv) * p.ld_dqkv + col_v + cq;
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      *reinterpret_cast<uint32_t*>(dkrow + 8 * i) = pack_bf16x2(dk[4 * i + 2 * hh], dk[4 * i + 2 * hh + 1]);
      *reinterpret_cast<uint32_t*>(dvrow + 8 * i) = pack_bf16x2(dv[4 * i + 2 * hh], dv[4 * i + 2 * hh + 1]);
    }
  }
}

// D[b,h,t] = sum_d dO[t,h,d] * O[t,h,d]   (one warp per (t,h))
template <int HD>
__global__ void __launch_bounds__(256) attn_dsum_kernel(const __nv_bfloat16* __restrict__ o, int64_t ld_o, const __nv_bfloat16* __restrict__ dout,
                                                       int64_t ld_do, int B, int T, int nh, float* __restrict__ dsum) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (int64_t)B * T * nh) return;
  const int h = (int)(w % nh);
  const int64_t row = w / nh;                      // b*T + t
  const uint32_t* po = reinterpret_cast<const uint32_t*>(o + row * ld_o + h * HD);
  const uint32_t* pd = reinterpret_cast<const uint32_t*>(dout + row * ld_do + h * HD);
  float a = 0.f;
#pragma unroll
  for (int i = lane; i < HD / 2; i += 32) {
    const uint32_t x = __ldg(po + i), y = __ldg(pd + i);
    a = fmaf(bf16lo(x), bf16lo(y), a);
    a = fmaf(bf16hi(x), bf16hi(y), a);
  }
  a = warp_sum(a);
  if (lane == 0) dsum[((row / T) * nh + h) * (int64_t)T + (row % T)] = a;
}

// dq32 [rows, nh*hd] fp32 -> q columns of the fused bf16 gradient buffer
__global__ void attn_dq_convert_kernel(const float* __restrict__ dq32, int64_t ld32, int64_t rows, int cols, __nv_bfloat16* __restrict__ dqkv, int64_t ld) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // one thread per 8 columns
  const int cv = cols >> 3;
  if (i >= rows * cv) return;
  const int64_t row = i / cv;
  const int c = (int)(i % cv) * 8;
  const float4 a = *reinterpret_cast<const float4*>(dq32 + row * ld32 + c), b2 = *reinterpret_cast<const float4*>(dq32 + row * ld32 + c + 4);
  uint4 w;
  w.x = pack_bf16x2(a.x, a.y); w.y = pack_bf16x2(a.z, a.w); w.z = pack_bf16x2(b2.x, b2.y); w.w = pack_bf16x2(b2.z, b2.w);
  *reinterpret_cast<uint4*>(dqkv + row * ld + c) = w;
}

template <int HD>
int launch_attn_bwd(const CUtensorMap& tkv, const CUtensorMap& tq, const CUtensorMap& tdo, const AttnBwdParams& p, cudaStream_t st) {
  constexpr int SMEM = 2 * BKVB * HD * 2 + NQ * 2 * BQB * HD * 2 + 2 * BKVB * BQB * 2 + 1024;
  static bool attr = false;
  if (!attr) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(attn_bwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr = true;
  }
  dim3 grid(p.nkv, p.B, (p.T + BKVB - 1) / BKVB);
  attn_bwd_kernel<HD><<<grid, ATB_THREADS, SMEM, st>>>(tkv, tq, tdo, p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

}  // namespace

// qkv / dqkv: fused [batch*seq, (nh+2nkv)*hd]; out, dout: [batch*seq, nh*hd]; lse [batch, nh, seq] from lmod_attn_fwd.
// dq32_ws: fp32 [batch*seq, nh*hd] workspace, dsum_ws: fp32 [batch, nh, seq] workspace (both written here; dq32 is zeroed inside).
// kv_lo / kv_hi: as in lmod_attn_fwd (padded batches), or NULL.
extern "C" int lmod_attn_bwd(const void* qkv, int64_t ld_qkv, const void* out, int64_t ld_o, const void* dout, int64_t ld_do, const float* lse,
                             int64_t batch, int64_t seq, int nh, int nkv, int hd, int causal, float softmax_scale, void* dqkv, int64_t ld_dqkv,
                             float* dq32_ws, float* dsum_ws, const int32_t* kv_lo, const int32_t* kv_hi, void* stream) {
  LMOD_CHECK_ARG((kv_lo == nullptr) == (kv_hi == nullptr), "lmod_attn_bwd: kv_lo and kv_hi come together");
  LMOD_CHECK_ARG(causal || kv_lo == nullptr, "lmod_attn_bwd: key padding (kv_lo / kv_hi) is only supported with causal = 1 (see lmod_attn_fwd)");
  LMOD_CHECK_ARG(qkv && out && dout && lse && dqkv && dq32_ws && dsum_ws && batch > 0 && seq > 0 && nh % nkv == 0, "lmod_attn_bwd: bad arguments");
  LMOD_CHECK_ARG(hd == 64 || hd == 128, "lmod_attn_bwd: head_dim %d not built (64 and 128 are)", hd);
  LMOD_CHECK_ARG(ld_qkv % 8 == 0 && ld_o % 8 == 0 && ld_do % 8 == 0 && ld_dqkv % 8 == 0, "lmod_attn_bwd: strides must be multiples of 8");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t rows = batch * seq;
  const int qcols = nh * hd;
  LMOD_CUDA_OK(cudaMemsetAsync(dq32_ws, 0, (size_t)rows * qcols * sizeof(float), st));
  {
    const int64_t warps = rows * nh;
    const unsigned blocks = (unsigned)((warps * 32 + 255) / 256);
    if (hd == 128) attn_dsum_kernel<128><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)out, ld_o, (const __nv_bfloat16*)dout, ld_do, (int)batch, (int)seq, nh, dsum_ws);
    else attn_dsum_kernel<64><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)out, ld_o, (const __nv_bfloat16*)dout, ld_do, (int)batch, (int)seq, nh, dsum_ws);
    LMOD_LAUNCH_OK();
  }
  CUtensorMap tkv, tq, tdo;
  const uint64_t cols = (uint64_t)(nh + 2 * nkv) * hd;
  int rc = make_map(&tkv, qkv, cols, (uint64_t)rows, (uint64_t)ld_qkv, 64, BKVB);
  if (rc) return rc;
  rc = make_map(&tq, qkv, cols, (uint64_t)rows, (uint64_t)ld_qkv, 64, BQB);
  if (rc) return rc;
  rc = make_map(&tdo, dout, (uint64_t)qcols, (uint64_t)rows, (uint64_t)ld_do, 64, BQB);
  if (rc) return rc;
  AttnBwdParams p;
  p.lse = lse; p.dsum = dsum_ws; p.dq32 = dq32_ws; p.dqkv = (__nv_bfloat16*)dqkv; p.ld_dqkv = ld_dqkv; p.ld_dq32 = qcols;
  p.B = (int)batch; p.T = (int)seq; p.nh = nh; p.nkv = nkv; p.causal = causal; p.scale = softmax_scale; p.scale_log2 = softmax_scale * LOG2E_F;
  p.kv_lo = kv_lo; p.kv_hi = kv_hi;
  rc = (hd == 128) ? launch_attn_bwd<128>(tkv, tq, tdo, p, st) : launch_attn_bwd<64>(tkv, tq, tdo, p, st);
  if (rc) return rc;
  const int64_t n = rows * (qcols / 8);
  attn_dq_convert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dq32_ws, qcols, rows, qcols, (__nv_bfloat16*)dqkv, ld_dqkv);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
