// attn.cu -- flash-attention FORWARD on wgmma / TMA (sm_90a), bf16 in, fp32 softmax + accumulation in registers.
//
// Replaces F.scaled_dot_product_attention of Qwen2SdpaAttention.forward (modeling_qwen2.py:713-721, causal, no padding) and the CLIP
// tower's non-causal self-attention (transformers CLIPVisionModel via clip_encoder.py:54).  Operates directly on the fused, RoPE'd
// QKV projection output [B*T, (nh + 2*nkv)*hd] -- no head transposes, GQA by index (repeat_kv :204-213 never materialises).
//
// One CTA = one (batch, head, 128-query block), three warpgroups:
//   warpgroup 0, thread 0 : TMA producer -- Q tile once, then K_j and V_j blocks (128B swizzle) into NST-stage rings with their own
//                           full / empty barriers; gives its registers to the math warpgroups (setmaxnreg)
//   warpgroups 1, 2       : 64 query rows each.  S_j = Q K_j^T (wgmma, both operands from shared memory, N = BKV) -> mask, online
//                           softmax in registers (exp2, row max / sum across the 4 threads of a row) -> P_j as bf16 A fragments
//                           (the S accumulator layout is the A-fragment layout) -> O += P_j V_j (wgmma, A from registers, V MN-major)
//                           -> epilogue O / l -> bf16 -> global, LSE
// Padded batches (right or left padding, per-row key range [kv_lo, kv_hi)) run on the same kernel: the CTA walks only the key blocks
// its rows can see and masks per element; rows with no visible key are un-masked as in the reference's 4-D mask.
#include <stdlib.h>
#include "sm90.cuh"

namespace {

constexpr int BQ = 128;
constexpr int ATT_THREADS = 384;          // TMA warpgroup + two math warpgroups
template <int HD> struct AttCfg {
  static constexpr int BKV = (HD == 64) ? 128 : 64;   // keys per block: S (BKV/2) + O (HD/2) accumulator registers per thread
  static constexpr int NST = 4;
  static constexpr int KSUB = HD / 64;               // 64-column sub-tiles along the head dimension
  static constexpr int Q_BYTES = BQ * HD * 2, KV_BYTES = BKV * HD * 2;
  static constexpr int SMEM = Q_BYTES + 2 * NST * KV_BYTES + 1024;
};

struct AttnParams {
  __nv_bfloat16* out;
  float* lse;            // [B, nh, T] natural-log LSE of the scaled scores (flash-attn's softmax_lse), may be null
  int64_t ld_o;
  int B, T, nh, nkv;
  int causal;
  float scale_log2;      // softmax_scale * log2(e)
  // padded batches (the reference's additive 4-D mask, modeling_qwen2.py:1035-1040): per batch row the keys [kv_lo, kv_hi) are real
  // tokens, everything else is padding.  Query rows that see no key at all (left padding) are un-masked like HF's
  // _unmask_unattended: they attend to every key of the row, causal mask dropped.  NULL = no padding.
  const int32_t* kv_lo;
  const int32_t* kv_hi;
};

template <int N, int TB>
__device__ __forceinline__ void wgmma_ss_kmajor(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (N == 128) wgmma_ss_n128<0, TB>(d, da, db, acc);
  else wgmma_ss_n64<0, TB>(d, da, db, acc);
}
template <int N>
__device__ __forceinline__ void wgmma_rs_mn(float* d, const uint32_t* a, uint64_t db, uint32_t acc) {
  if constexpr (N == 128) wgmma_rs_n128<1>(d, a, db, acc);
  else wgmma_rs_n64<1>(d, a, db, acc);
}

template <int HD>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_kv, const AttnParams p) {
  using C = AttCfg<HD>;
  constexpr int BKV = C::BKV, NST = C::NST, KSUB = C::KSUB;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t q_full, k_full[NST], k_empty[NST], v_full[NST], v_empty[NST];

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = smem;
  uint8_t* sK0 = smem + C::Q_BYTES;                   // K stage s at sK0 + s*KV_BYTES
  uint8_t* sV0 = sK0 + NST * C::KV_BYTES;             // V stage s at sV0 + s*KV_BYTES
  const int wg = threadIdx.x >> 7;

  // Grid = (heads, batch, query blocks): heads vary fastest and the heavy (late) causal query blocks of ALL heads are handed out first
  const int nqb = (p.T + BQ - 1) / BQ;
  const int qb = p.causal ? (nqb - 1 - (int)blockIdx.z) : (int)blockIdx.z;
  const int h = (int)blockIdx.x, b = blockIdx.y;
  const int hk = h / (p.nh / p.nkv);
  const int q0 = qb * BQ;
  int lo = 0, hi = p.T;
  if (p.kv_lo) { lo = p.kv_lo[b]; hi = p.kv_hi[b]; }
  const bool all_pad = hi <= lo;
  // key blocks this query block walks: [jb, jb + nblk).  A block that holds an un-masked row (no visible key) walks every key.
  int kbeg = lo, kend = p.causal ? min(hi, q0 + BQ) : hi;
  if (all_pad || q0 < lo) { kbeg = 0; kend = p.T; }
  const int jb = kbeg / BKV;
  const int nblk = (kend + BKV - 1) / BKV - jb;
  const int row_base = b * p.T;                       // row of token 0 of this batch in the fused buffer
  const int col_q = h * HD, col_k = (p.nh + hk) * HD, col_v = (p.nh + p.nkv + hk) * HD;

  if (threadIdx.x == 0) {
    mbar_init(&q_full, 1);
    for (int s = 0; s < NST; ++s) { mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 2); mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 2); }
    mbar_fence_init();
    asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_q) : "memory");
    asm volatile("prefetch.tensormap [%0];" :: "l"(&tma_kv) : "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer: Q once, then K_j and V_j =====================
    regs_dealloc<40>();
    if (threadIdx.x == 0 && nblk > 0) {
      mbar_expect_tx(&q_full, C::Q_BYTES);
#pragma unroll
      for (int i = 0; i < KSUB; ++i) tma_load_2d(sQ + i * (BQ * 128), &tma_q, col_q + 64 * i, row_base + q0, &q_full);
      for (int j = 0; j < nblk; ++j) {
        const int s = j % NST;
        const uint32_t ph = ((j / NST) & 1) ^ 1;
        mbar_wait_bounded(&k_empty[s], ph);
        mbar_expect_tx(&k_full[s], C::KV_BYTES);
#pragma unroll
        for (int i = 0; i < KSUB; ++i) tma_load_2d(sK0 + s * C::KV_BYTES + i * (BKV * 128), &tma_kv, col_k + 64 * i, row_base + (jb + j) * BKV, &k_full[s]);
        mbar_wait_bounded(&v_empty[s], ph);
        mbar_expect_tx(&v_full[s], C::KV_BYTES);
#pragma unroll
        for (int i = 0; i < KSUB; ++i) tma_load_2d(sV0 + s * C::KV_BYTES + i * (BKV * 128), &tma_kv, col_v + 64 * i, row_base + (jb + j) * BKV, &v_full[s]);
      }
    }
    return;
  }

  // ===================== math warpgroups =====================
  regs_alloc<232>();
  const int c = wg - 1;
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  // fragment rows: r + 8h (h = 0, 1) of the 128-row block; columns 8i + cq + e
  const int r = c * 64 + w * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  int klo[2], khi[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qrow = q0 + r + 8 * hh;
    klo[hh] = lo; khi[hh] = p.causal ? min(hi, qrow + 1) : hi;
    if (all_pad || qrow < lo) { klo[hh] = 0; khi[hh] = p.T; }
  }
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  const uint32_t aQ = smem_u32(sQ) + c * (64 * 128);
  if (nblk > 0) mbar_wait(&q_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int s = j % NST;
    const uint32_t ph = (j / NST) & 1;
    float sacc[BKV / 2];
    mbar_wait(&k_full[s], ph);
    const uint32_t aK = smem_u32(sK0 + s * C::KV_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k)
      wgmma_ss_kmajor<BKV, 0>(sacc, gmma_desc(aQ + (k / 4) * (BQ * 128) + (k % 4) * 32, 16, 1024),
                              gmma_desc(aK + (k / 4) * (BKV * 128) + (k % 4) * 32, 16, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<BKV / 2>(sacc);
    if (wg_leader) mbar_arrive(&k_empty[s]);

    const int kv0 = (jb + j) * BKV;
    if (kv0 < max(klo[0], klo[1]) || kv0 + BKV > min(khi[0], khi[1])) {
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int hh = e >> 1, kv = kv0 + 8 * i + cq + (e & 1);
          if (kv < klo[hh] || kv >= khi[hh]) sacc[4 * i + e] = -INFINITY;
        }
    }
    float alpha[2], neg_m[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i) mx = fmaxf(mx, fmaxf(sacc[4 * i + 2 * hh], sacc[4 * i + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[hh], mx * p.scale_log2);
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;   // no visible key so far: keep everything finite (P = exp2(-inf) = 0)
      alpha[hh] = ex2f(m[hh] - m_use);                         // m = -inf -> 0
      m[hh] = m_new;
      neg_m[hh] = -m_use;
    }
    uint32_t pa[BKV / 16][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) {
      float pv[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        pv[e] = ex2f(fmaf(sacc[4 * i + e], p.scale_log2, neg_m[e >> 1]));
        rs[e >> 1] += pv[e];
      }
      pa[i >> 1][(i & 1) * 2 + 0] = pack_bf16x2(pv[0], pv[1]);
      pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(pv[2], pv[3]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) l[hh] = fmaf(l[hh], alpha[hh], rs[hh]);
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      o[4 * i + 0] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }

    mbar_wait(&v_full[s], ph);
    const uint32_t aV = smem_u32(sV0 + s * C::KV_BYTES);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)        // V_j as B operand, MN-major: 64-wide hd blocks BKV*128 B apart, 16 keys = 2048 B per k step
      wgmma_rs_mn<HD>(o, pa[kk], gmma_desc(aV + kk * 2048, BKV * 128, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<HD / 2>(o);
    if (wg_leader) mbar_arrive(&v_empty[s]);
  }

  // ---- epilogue: normalise, store, LSE ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float lt = l[hh];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv = (lt > 0.f) ? 1.f / lt : 0.f;
    const int qrow = q0 + r + 8 * hh;
    if (qrow < p.T) {
      __nv_bfloat16* orow = p.out + (int64_t)(row_base + qrow) * p.ld_o + col_q + cq;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i)
        *reinterpret_cast<uint32_t*>(orow + 8 * i) = pack_bf16x2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
      if (p.lse && (lane & 3) == 0) p.lse[((int64_t)b * p.nh + h) * p.T + qrow] = (m[hh] + lg2f(lt)) * LN2_F;
    }
  }
}

template <int HD>
int launch_attn(const CUtensorMap& tq, const CUtensorMap& tkv, const AttnParams& p, cudaStream_t st) {
  constexpr int SMEM = AttCfg<HD>::SMEM;
  static bool attr = false;
  if (!attr) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr = true;
  }
  const dim3 grid(p.nh, p.B, (p.T + BQ - 1) / BQ);
  attn_fwd_kernel<HD><<<grid, ATT_THREADS, SMEM, st>>>(tq, tkv, p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

}  // namespace

// qkv: fused projection output [batch*seq, (nh + 2*nkv)*hd] bf16 (q heads | k heads | v heads), row stride ld_qkv.
// out: [batch*seq, nh*hd] (row stride ld_o).  lse: [batch, nh, seq] fp32 or NULL.  hd in {64, 128}.
// kv_lo / kv_hi: int32 [batch] device arrays, the real (un-padded) key range of every batch row, or both NULL for no padding.
extern "C" int lmod_attn_fwd(const void* qkv, int64_t ld_qkv, int64_t batch, int64_t seq, int nh, int nkv, int hd, int causal,
                             float softmax_scale, void* out, int64_t ld_o, float* lse, const int32_t* kv_lo, const int32_t* kv_hi,
                             void* stream) {
  LMOD_CHECK_ARG((kv_lo == nullptr) == (kv_hi == nullptr), "lmod_attn_fwd: kv_lo and kv_hi come together");
  // The kernel un-masks every query row in front of kv_lo (no visible key under the causal mask).  Without the causal mask those rows
  // would see [kv_lo, kv_hi) under a key-padding mask, so the combination would silently give a different answer: refuse it.
  LMOD_CHECK_ARG(causal || kv_lo == nullptr, "lmod_attn_fwd: key padding (kv_lo / kv_hi) is only supported with causal = 1");
  LMOD_CHECK_ARG(qkv && out && batch > 0 && seq > 0 && nh > 0 && nkv > 0 && nh % nkv == 0, "lmod_attn_fwd: bad arguments");
  LMOD_CHECK_ARG(hd == 64 || hd == 128, "lmod_attn_fwd: head_dim %d not built (64 and 128 are)", hd);
  LMOD_CHECK_ARG(ld_qkv % 8 == 0 && ld_o % 8 == 0 && ((uintptr_t)qkv % 16 == 0) && ((uintptr_t)out % 16 == 0), "lmod_attn_fwd: alignment");
  CUtensorMap tq, tkv;
  const uint64_t cols = (uint64_t)(nh + 2 * nkv) * hd, rows = (uint64_t)(batch * seq);
  int rc = make_map(&tq, qkv, cols, rows, (uint64_t)ld_qkv, 64, BQ);
  if (rc) return rc;
  rc = make_map(&tkv, qkv, cols, rows, (uint64_t)ld_qkv, 64, hd == 128 ? AttCfg<128>::BKV : AttCfg<64>::BKV);
  if (rc) return rc;
  AttnParams p;
  p.out = (__nv_bfloat16*)out; p.lse = lse; p.ld_o = ld_o; p.B = (int)batch; p.T = (int)seq; p.nh = nh; p.nkv = nkv; p.causal = causal;
  p.scale_log2 = softmax_scale * LOG2E_F;
  p.kv_lo = kv_lo; p.kv_hi = kv_hi;
  return hd == 128 ? launch_attn<128>(tq, tkv, p, (cudaStream_t)stream) : launch_attn<64>(tq, tkv, p, (cudaStream_t)stream);
}
