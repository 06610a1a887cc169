// kl.cu -- fused mimic-KL (+ shifted CE) forward+backward over the vocabulary.
//
// Replaces (reference) llavamod/train/align_trainer.py:473-475 (teacher softmax fp32), :497-499
// (student log_softmax fp32), :509-526 (product / masked_fill / vocab sum / masked mean) and
// llava_qwen1_5_moe.py:413-421 (shifted CE), i.e. >= 8 full [N,V] passes, by one kernel, kl_stream_kernel:
//
//   * a cluster of KS_CS = 2 CTAs owns a row (V = 151936 bf16 logits, student + teacher = 608 KB), each CTA one half of it; cluster cid
//     takes the rows cid, cid + ncl, ... (ncl = co-resident clusters).
//   * in each CTA a TMA producer warp streams the half row through a KS_STAGES-deep shared-memory ring of KS_CH logit pairs (1-D bulk
//     copies completing on mbarriers), twice, and 16 consumer warps work on it:
//       pass 1  online max / sum-exp / sum p_T*s of both rows, a block reduction, then the exchange between the two CTAs of the row: each
//               stores its partials into the other's shared memory (DSMEM) and arrives on the other's mbarrier, so no barrier.cluster
//               stops the producer, which runs ahead into pass 2 and the next row;
//       pass 2  the gradient, written in place over the student logits.  The last ring-full of pass-1 chunks is still held in the ring;
//               the chunks before it are fetched again and come out of L2, because pass 1 loaded them with evict_last (every last read
//               of a chunk is evict_first).
//   * on an H100 (50 MB L2, 132 SMs) two CTAs per row keep 66 rows = 40 MB in flight, so pass 2 hits L2 and HBM traffic stays the
//     algorithmic 4V bytes read + 2V written per token; one CTA per row keeps 79 MB in flight and pass 2 partly misses.  Timed on one
//     H100 (400 W limit), 885 rows x 151936: 0.338 ms with two CTAs per row against 0.415 ms with one.
//   * rows whose KD mask and CE mask are both 0 contribute nothing (reference multiplies by 0): their loads are skipped and their
//     gradient slice is zero-filled.
#include <stdio.h>
#include <stdlib.h>
#include "common.cuh"

namespace {

constexpr int KS_CS = 2;                 // CTAs per row (a cluster shares a row through DSMEM)
constexpr int KS_CH = 8192;              // logit pairs per ring stage (16 KB student + 16 KB teacher)
constexpr int KS_STAGES = 6;             // 192 KB ring
constexpr int KS_THREADS = 512;          // consumer threads (+ one producer warp)
// the exchange is a DSMEM store into the peer CTA + a remote mbarrier arrive: a row needs at least two CTAs
static_assert(KS_CS >= 2, "kl_stream_kernel exchanges partials between the CTAs of a row");
constexpr int64_t KL_MAX_VOCAB = 450560;  // largest vocabulary the entry points accept (Qwen's is 151936)

struct KlParams {
  const __nv_bfloat16* s;
  const __nv_bfloat16* t;
  const int64_t* labels;
  const float* counts;   // {n_kd, n_ce}
  float* row_out;        // [N,4]
  __nv_bfloat16* d;      // may be null / alias s
  int64_t ld_s, ld_t, ld_d;
  int64_t n_rows, seq_len;
  int vocab, slice;      // slice: elements per CTA (multiple of 8)
  int distill_all;
  float w_kd, w_ce;
  // compact mode (rows.cu): s / t / d hold only the batch's active rows, row j of them is original row perm[j] (labels, row_out);
  // the row count comes from device memory.  null = dense layout, n_rows rows.
  const int32_t* perm;
  const int32_t* count;
};

__device__ __forceinline__ uint32_t hmax2_u32(uint32_t a, uint32_t b) {
  __nv_bfloat162 r = __hmax2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
  return *reinterpret_cast<uint32_t*>(&r);
}
__device__ __forceinline__ uint32_t hmin2_u32(uint32_t a, uint32_t b) {
  __nv_bfloat162 r = __hmin2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
  return *reinterpret_cast<uint32_t*>(&r);
}

// one (student, teacher) word pair of a vector that holds an infinite student logit: align_trainer.py:509-510 drops the terms where
// log q_S is +-inf
__device__ __forceinline__ void accum_pair(uint32_t sw, uint32_t tw, float nms, float nmt, float& zs, float& zt, float& a, float& zk) {
  float s0 = bf16lo(sw), s1 = bf16hi(sw), t0 = bf16lo(tw), t1 = bf16hi(tw);
  float es0 = ex2f(fmaf(s0, LOG2E_F, nms)), es1 = ex2f(fmaf(s1, LOG2E_F, nms));
  float et0 = ex2f(fmaf(t0, LOG2E_F, nmt)), et1 = ex2f(fmaf(t1, LOG2E_F, nmt));
  zs += es0; zs += es1;
  zt += et0; zt += et1;
  if (isinf(s0)) { s0 = 0.f; et0 = 0.f; }
  if (isinf(s1)) { s1 = 0.f; et1 = 0.f; }
  zk += et0; zk += et1;      // teacher mass of the KEPT terms: x = sum_kept p_T*(s - lse_S)
  a = fmaf(et0, s0, a);
  a = fmaf(et1, s1, a);
}

struct XchgS { float ms, mt, zs, zt, a, slab, zk, pad; };

__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_addr, uint32_t rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
  return ra;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t remote_addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" :: "r"(remote_addr), "f"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t remote_bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" :: "r"(remote_bar) : "memory");
}
// bounded waits: a protocol bug traps (reported by the launch check) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t phase) {
  uint32_t ok = 0, spins = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    if (!ok && ++spins > (1u << 24)) { printf("lmod kl_stream_kernel: exchange barrier timeout (block %d thread %d)\n", blockIdx.x, threadIdx.x); __trap(); }
  }
}
__device__ __forceinline__ void ks_wait(uint64_t* bar, uint32_t phase) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, phase)) {
    if (++spins > (1u << 24)) { printf("lmod kl_stream_kernel: ring barrier timeout (block %d thread %d)\n", blockIdx.x, threadIdx.x); __trap(); }
  }
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}

// Two-lane accumulators of the online pass: lane 0 sums the even vocabulary positions of a thread, lane 1 the odd ones.  Every operation
// is rounded to nearest on its own (no contraction into other FMAs), so the summation order and the result are fixed.
struct Acc2 { float zs0, zs1, zt0, zt1, a0, a1; };
// one 32-bit word of student logits + one of teacher logits (two vocabulary positions)
__device__ __forceinline__ void accum_word(uint32_t sw, uint32_t tw, float nms, float nmt, Acc2& A) {
  const float s0 = bf16lo(sw), s1 = bf16hi(sw), t0 = bf16lo(tw), t1 = bf16hi(tw);
  const float es0 = ex2f(__fmaf_rn(s0, LOG2E_F, nms)), es1 = ex2f(__fmaf_rn(s1, LOG2E_F, nms));
  const float et0 = ex2f(__fmaf_rn(t0, LOG2E_F, nmt)), et1 = ex2f(__fmaf_rn(t1, LOG2E_F, nmt));
  A.zs0 = __fadd_rn(A.zs0, es0); A.zs1 = __fadd_rn(A.zs1, es1);
  A.zt0 = __fadd_rn(A.zt0, et0); A.zt1 = __fadd_rn(A.zt1, et1);
  A.a0 = __fmaf_rn(et0, s0, A.a0); A.a1 = __fmaf_rn(et1, s1, A.a1);
}
// gradient of one word: g = ca * q_S - cb * p_T
__device__ __forceinline__ void grad_word(uint32_t sw, uint32_t tw, float es, float et, float ca, float ncb, float& g0, float& g1) {
  const float q0 = ex2f(__fmaf_rn(bf16lo(sw), LOG2E_F, es)), q1 = ex2f(__fmaf_rn(bf16hi(sw), LOG2E_F, es));
  const float p0 = ex2f(__fmaf_rn(bf16lo(tw), LOG2E_F, et)), p1 = ex2f(__fmaf_rn(bf16hi(tw), LOG2E_F, et));
  g0 = __fmaf_rn(q0, ca, __fmaf_rn(p0, ncb, 0.f));
  g1 = __fmaf_rn(q1, ca, __fmaf_rn(p1, ncb, 0.f));
}

__device__ __forceinline__ bool kl_row_masks(const KlParams& p, int64_t row, int64_t& orow, int64_t& lab_next, bool& m_kd, bool& m_ce) {
  orow = p.perm ? (int64_t)p.perm[row] : row;
  const int64_t lab_here = p.labels[orow];
  const int64_t tpos = orow % p.seq_len;
  lab_next = LMOD_IGNORE_INDEX;
  if (tpos + 1 < p.seq_len) lab_next = p.labels[orow + 1];
  m_kd = p.distill_all ? true : (lab_here != LMOD_IGNORE_INDEX);
  m_ce = (lab_next != LMOD_IGNORE_INDEX);
  return m_kd || m_ce;
}

__global__ void __launch_bounds__(KS_THREADS + 32, 1) kl_stream_kernel(const KlParams p) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ __align__(16) XchgS xchg[2][KS_CS];                // [slot][source CTA]: written by the peers through DSMEM
  __shared__ __align__(8) uint64_t full[KS_STAGES], empty[KS_STAGES], xbar[2];
  __shared__ float red[7][KS_THREADS / 32];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank();
  const uint32_t cid = cluster_id_x(), ncl = cluster_nclusters_x();
  const int v0 = (int)rank * p.slice;
  int len = p.vocab - v0;
  len = len < 0 ? 0 : (len > p.slice ? p.slice : len);
  const int nchunks = (len + KS_CH - 1) / KS_CH;
  const bool want_grad = p.d != nullptr;
  const int held = want_grad ? min(KS_STAGES, nchunks) : 0;     // pass-1 chunks kept in the ring for pass 2

  if (tid == 0) {
    for (int i = 0; i < KS_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], KS_THREADS / 32); }
    mbar_init(&xbar[0], KS_CS); mbar_init(&xbar[1], KS_CS);
    mbar_fence_init();
  }
  __syncthreads();
  cluster_sync_all();                                            // every CTA's barriers exist before a peer arrives on them

  const int64_t n_rows = p.count ? (int64_t)*p.count : p.n_rows;

  if (warp == KS_THREADS / 32) {
    // ===================== producer warp: the chunks of every active row, pass 1 then pass 2, through the ring =====================
    if (lane == 0 && nchunks > 0) {
      const uint64_t keep = l2_policy_evict_last(), drop = l2_policy_evict_first();
      uint32_t n = 0;
      for (int64_t row = cid; row < n_rows; row += ncl) {
        int64_t orow, lab_next; bool m_kd, m_ce;
        if (!kl_row_masks(p, row, orow, lab_next, m_kd, m_ce)) continue;
        const __nv_bfloat16* srow = p.s + row * p.ld_s + v0;
        const __nv_bfloat16* trow = p.t + row * p.ld_t + v0;
        // pass 1: every chunk.  pass 2: the last `held` chunks of pass 1 are still in the ring (their stages are released only after the
        // gradient pass has used them), so only chunks [0, nchunks - held) are fetched again, into the stages as they come free
        for (int c = 0; c < nchunks; ++c, ++n) {
          const uint32_t st = n % KS_STAGES;
          if (n >= KS_STAGES) ks_wait(&empty[st], ((n / KS_STAGES) - 1) & 1);
          const int e0 = c * KS_CH, cnt = min(KS_CH, len - e0);
          uint8_t* sb = smem_raw + (size_t)st * (KS_CH * 4);
          const uint64_t pol = (want_grad && c < nchunks - held) ? keep : drop;      // what pass 2 re-reads should stay in L2, the rest not
          mbar_expect_tx(&full[st], (uint32_t)cnt * 4u);
          bulk_g2s_hint(sb, srow + e0, (uint32_t)cnt * 2u, &full[st], pol);
          bulk_g2s_hint(sb + KS_CH * 2, trow + e0, (uint32_t)cnt * 2u, &full[st], pol);
        }
        if (want_grad) {
          for (int c = 0; c < nchunks - held; ++c, ++n) {
            const uint32_t st = n % KS_STAGES;
            if (n >= KS_STAGES) ks_wait(&empty[st], ((n / KS_STAGES) - 1) & 1);
            const int e0 = c * KS_CH, cnt = min(KS_CH, len - e0);
            uint8_t* sb = smem_raw + (size_t)st * (KS_CH * 4);
            mbar_expect_tx(&full[st], (uint32_t)cnt * 4u);
            bulk_g2s_hint(sb, srow + e0, (uint32_t)cnt * 2u, &full[st], drop);
            bulk_g2s_hint(sb + KS_CH * 2, trow + e0, (uint32_t)cnt * 2u, &full[st], drop);
          }
        }
      }
    }
  } else {
    // ===================== consumers =====================
    const float n_kd = p.counts[0], n_ce = p.counts[1];
    uint32_t n = 0, it_active = 0;
    for (int64_t row = cid; row < n_rows; row += ncl) {
      int64_t orow, lab_next; bool m_kd, m_ce;
      const bool active = kl_row_masks(p, row, orow, lab_next, m_kd, m_ce);
      if (!active) {
        if (want_grad) {
          const uint4 z = make_uint4(0, 0, 0, 0);
          uint4* dst = reinterpret_cast<uint4*>(p.d + row * p.ld_d + v0);
          for (int i = tid; i < (len >> 3); i += KS_THREADS) stg_v4(dst + i, z);
        }
        if (rank == 0 && tid == 0) *reinterpret_cast<float4*>(p.row_out + orow * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
        continue;
      }
      const uint32_t xi = it_active & 1u, xpar = (it_active >> 1) & 1u;
      ++it_active;
      const int lab_local = m_ce ? (int)(lab_next - v0) : -1;     // position of the CE label inside this CTA's half row (or outside)
      // ---- pass 1: online (max, scaled sums) per thread, chunk by chunk as the ring fills ----
      // The running maxima settle after a few vectors, so the rescale branch is cold.  Infinite logits never enter a running maximum:
      // -inf terms vanish on their own, +inf keeps the degenerate outcome (sum-exp = inf).
      float m_s = -INFINITY, m_t = -INFINITY, zk = 0.f, slab = 0.f;
      Acc2 A = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int c = 0; c < nchunks; ++c, ++n) {
        const uint32_t st = n % KS_STAGES;
        const int e0 = c * KS_CH, nv = min(KS_CH, len - e0) >> 3;
        const uint4* s_buf = reinterpret_cast<const uint4*>(smem_raw + (size_t)st * (KS_CH * 4));
        const uint4* t_buf = reinterpret_cast<const uint4*>(smem_raw + (size_t)st * (KS_CH * 4) + KS_CH * 2);
        ks_wait(&full[st], (n / KS_STAGES) & 1);      // every thread polls
        for (int i = tid; i < nv; i += KS_THREADS) {
          const uint4 sv = s_buf[i], tv = t_buf[i];
          const uint32_t pmx_s = hmax2_u32(hmax2_u32(sv.x, sv.y), hmax2_u32(sv.z, sv.w));
          const uint32_t pmn_s = hmin2_u32(hmin2_u32(sv.x, sv.y), hmin2_u32(sv.z, sv.w));
          const uint32_t pmx_t = hmax2_u32(hmax2_u32(tv.x, tv.y), hmax2_u32(tv.z, tv.w));
          const float vmax_s = fmaxf(bf16lo(pmx_s), bf16hi(pmx_s)), vmin_s = fminf(bf16lo(pmn_s), bf16hi(pmn_s));
          const float vmax_t = fmaxf(bf16lo(pmx_t), bf16hi(pmx_t));
          if (vmax_s > m_s && !isinf(vmax_s)) {
            const float f = ex2f((m_s - vmax_s) * LOG2E_F);             // m_s = -inf the first time: 0 * 0
            A.zs0 *= f; A.zs1 *= f;
            m_s = vmax_s;
          }
          if (vmax_t > m_t && !isinf(vmax_t)) {
            const float f = ex2f((m_t - vmax_t) * LOG2E_F);
            A.zt0 *= f; A.zt1 *= f; A.a0 *= f; A.a1 *= f; zk *= f;
            m_t = vmax_t;
          }
          const float nms = isinf(m_s) ? 0.f : -m_s * LOG2E_F, nmt = isinf(m_t) ? 0.f : -m_t * LOG2E_F;
          if (!(isinf(vmin_s) || isinf(vmax_s))) {
            accum_word(sv.x, tv.x, nms, nmt, A);
            accum_word(sv.y, tv.y, nms, nmt, A);
            accum_word(sv.z, tv.z, nms, nmt, A);
            accum_word(sv.w, tv.w, nms, nmt, A);
          } else {
            // a vector that holds an infinite student logit: scalar path that drops those terms
            float zs = 0.f, zt = 0.f, acc = 0.f, zk_v = 0.f;
            accum_pair(sv.x, tv.x, nms, nmt, zs, zt, acc, zk_v);
            accum_pair(sv.y, tv.y, nms, nmt, zs, zt, acc, zk_v);
            accum_pair(sv.z, tv.z, nms, nmt, zs, zt, acc, zk_v);
            accum_pair(sv.w, tv.w, nms, nmt, zs, zt, acc, zk_v);
            A.zs0 += zs; A.zt0 += zt; A.a0 += acc;
            zk += zk_v - zt;                                              // zk tracks (kept - all) teacher mass; the final zk = zt + this
          }
          const unsigned rel = (unsigned)(lab_local - (e0 + i * 8));
          if (rel < 8u) slab = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(s_buf + i)[rel]);
        }
        __syncwarp();
        if (lane == 0 && c < nchunks - held) mbar_arrive(&empty[st]);       // the held tail is released by pass 2
      }
      float zs = A.zs0 + A.zs1, zt = A.zt0 + A.zt1, acc = A.a0 + A.a1;
      zk += zt;
      // ---- block reduction with the (max, scaled sums) combine ----
      {
        float Ms = warp_max(m_s), Mt = warp_max(m_t);
        const float fs = isinf(m_s) ? 0.f : ex2f((m_s - Ms) * LOG2E_F);
        const float ft = isinf(m_t) ? 0.f : ex2f((m_t - Mt) * LOG2E_F);
        zs = warp_sum(isinf(zs) ? zs : zs * fs);
        zt = warp_sum(isinf(zt) ? zt : zt * ft);
        acc = warp_sum(acc * ft); zk = warp_sum(zk * ft);
        slab = warp_sum(slab);
        if (lane == 0) { red[0][warp] = Ms; red[1][warp] = Mt; red[2][warp] = slab; red[3][warp] = zs; red[4][warp] = zt; red[5][warp] = acc; red[6][warp] = zk; }
      }
      asm volatile("bar.sync 1, %0;" :: "n"(KS_THREADS) : "memory");
      if (warp == 0) {
        constexpr int NW = KS_THREADS / 32;
        const float wms = (lane < NW) ? red[0][lane] : -INFINITY, wmt = (lane < NW) ? red[1][lane] : -INFINITY;
        const float ms = warp_max(wms), mt = warp_max(wmt);
        const float fs = isinf(wms) ? 0.f : ex2f((wms - ms) * LOG2E_F);
        const float ft = isinf(wmt) ? 0.f : ex2f((wmt - mt) * LOG2E_F);
        float a = (lane < NW) ? red[3][lane] : 0.f, b = (lane < NW) ? red[4][lane] : 0.f;
        float c2 = (lane < NW) ? red[5][lane] : 0.f, k = (lane < NW) ? red[6][lane] : 0.f, sl = (lane < NW) ? red[2][lane] : 0.f;
        a = warp_sum(isinf(a) ? a : a * fs); b = warp_sum(isinf(b) ? b : b * ft);
        c2 = warp_sum(c2 * ft); k = warp_sum(k * ft); sl = warp_sum(sl);
        if (lane < KS_CS) {
          // publish this CTA's partials into slot [xi][rank] of EVERY CTA of the cluster (lane l -> CTA l), then arrive on its barrier
          const uint32_t base = mapa_u32(smem_u32(&xchg[xi][rank]), (uint32_t)lane);
          st_cluster_f32(base + 0, (len > 0) ? ms : -INFINITY); st_cluster_f32(base + 4, (len > 0) ? mt : -INFINITY);
          st_cluster_f32(base + 8, a); st_cluster_f32(base + 12, b); st_cluster_f32(base + 16, c2); st_cluster_f32(base + 20, sl);
          st_cluster_f32(base + 24, k);
          mbar_arrive_cluster(mapa_u32(smem_u32(&xbar[xi]), (uint32_t)lane));
        }
      }
      mbar_wait_cluster(&xbar[xi], xpar);
      float lse_s, lse_t, xrow, slab_row;
      {
        float r_ms = -INFINITY, r_mt = -INFINITY, r_zs = 0.f, r_zt = 0.f, r_a = 0.f, r_sl = 0.f, r_zk = 0.f;
        if (lane < KS_CS) {
          const XchgS x = xchg[xi][lane];
          r_ms = x.ms; r_mt = x.mt; r_zs = x.zs; r_zt = x.zt; r_a = x.a; r_sl = x.slab; r_zk = x.zk;
        }
        const float Ms = warp_max(r_ms), Mt = warp_max(r_mt);
        const float Ms_u = isinf(Ms) ? 0.f : Ms, Mt_u = isinf(Mt) ? 0.f : Mt;
        const float fs = isinf(r_ms) ? 0.f : ex2f((r_ms - Ms_u) * LOG2E_F);
        const float ft = isinf(r_mt) ? 0.f : ex2f((r_mt - Mt_u) * LOG2E_F);
        const float Zs = warp_sum(r_zs * fs), Zt = warp_sum(r_zt * ft), A = warp_sum(r_a * ft), Zk = warp_sum(r_zk * ft);
        slab_row = warp_sum(r_sl);
        lse_s = Ms_u + lg2f(Zs) * LN2_F;
        lse_t = Mt_u + lg2f(Zt) * LN2_F;
        xrow = (A - lse_s * Zk) / Zt;
      }
      if (rank == 0 && tid == 0)
        *reinterpret_cast<float4*>(p.row_out + orow * 4) = make_float4(xrow, m_ce ? (lse_s - slab_row) : 0.f, lse_s, lse_t);
      // ---- pass 2: the same chunks again (L2), gradient written in place ----
      if (want_grad) {
        const float ckd = m_kd ? (p.w_kd / n_kd) : 0.f;
        const float cce = m_ce ? (p.w_ce / n_ce) : 0.f;
        const float ca = ckd + cce, cb = ckd;
        const float es = -lse_s * LOG2E_F, et = -lse_t * LOG2E_F;
        // first the chunks pass 1 left in the ring (no load, no wait: their stage is the one pass 1 filled), then the rest of the row as the
        // producer re-fetches it (L2) into the stages released here
        const uint32_t n_p1 = n - (uint32_t)nchunks;                      // sequence number of this row's first pass-1 chunk
        for (int q = 0; q < nchunks; ++q) {
          const bool in_ring = q < held;
          const int c = in_ring ? nchunks - held + q : q - held;
          const uint32_t st = (in_ring ? n_p1 + (uint32_t)c : n) % KS_STAGES;
          const int e0 = c * KS_CH, nv = min(KS_CH, len - e0) >> 3;
          const uint4* s_buf = reinterpret_cast<const uint4*>(smem_raw + (size_t)st * (KS_CH * 4));
          const uint4* t_buf = reinterpret_cast<const uint4*>(smem_raw + (size_t)st * (KS_CH * 4) + KS_CH * 2);
          uint4* dst = reinterpret_cast<uint4*>(p.d + row * p.ld_d + v0 + e0);
          if (!in_ring) { ks_wait(&full[st], (n / KS_STAGES) & 1); ++n; }
          for (int i = tid; i < nv; i += KS_THREADS) {
            const uint4 sv = s_buf[i], tv = t_buf[i];
            float g[8];
            grad_word(sv.x, tv.x, es, et, ca, -cb, g[0], g[1]);
            grad_word(sv.y, tv.y, es, et, ca, -cb, g[2], g[3]);
            grad_word(sv.z, tv.z, es, et, ca, -cb, g[4], g[5]);
            grad_word(sv.w, tv.w, es, et, ca, -cb, g[6], g[7]);
            const unsigned rel = (unsigned)(lab_local - (e0 + i * 8));
            if (rel < 8u) {
#pragma unroll
              for (int j = 0; j < 8; ++j) if (rel == (unsigned)j) g[j] -= cce;
            }
            uint4 o;
            o.x = pack_bf16x2(g[0], g[1]); o.y = pack_bf16x2(g[2], g[3]);
            o.z = pack_bf16x2(g[4], g[5]); o.w = pack_bf16x2(g[6], g[7]);
            stg_v4(dst + i, o);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[st]);
        }
      }
    }
  }
  cluster_sync_all();  // keep this CTA's shared memory and barriers alive until every peer finished its DSMEM stores
}

__global__ void kl_counts_kernel(const int64_t* __restrict__ labels, int64_t n, int64_t T, int distill_all,
                                 float* __restrict__ out) {
  __shared__ float red[32];
  float a = 0.f, b = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    a += (distill_all || labels[i] != LMOD_IGNORE_INDEX) ? 1.f : 0.f;
    if ((i % T) + 1 < T) b += (labels[i + 1] != LMOD_IGNORE_INDEX) ? 1.f : 0.f;
  }
  a = block_sum(a, red);
  b = block_sum(b, red);
  if (threadIdx.x == 0) { out[0] = a; out[1] = b; }
}

__global__ void kl_finalize_kernel(const float* __restrict__ row_out, const int64_t* __restrict__ labels,
                                   int64_t n, int64_t T, int distill_all, float* __restrict__ out) {
  __shared__ float red[32];
  float sx = 0.f, sn = 0.f, ck = 0.f, cc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    float4 r = *reinterpret_cast<const float4*>(row_out + i * 4);
    bool m = distill_all || labels[i] != LMOD_IGNORE_INDEX;
    bool c = ((i % T) + 1 < T) && labels[i + 1] != LMOD_IGNORE_INDEX;
    if (m) { sx += r.x; ck += 1.f; }
    if (c) { sn += r.y; cc += 1.f; }
  }
  sx = block_sum(sx, red); sn = block_sum(sn, red); ck = block_sum(ck, red); cc = block_sum(cc, red);
  if (threadIdx.x == 0) {
    out[0] = -sx / ck;     // 0/0 -> NaN like align_trainer.py:526
    out[1] = sn / cc;
    out[2] = ck;
    out[3] = cc;
  }
}

}  // namespace

extern "C" int lmod_kl_counts(const int64_t* labels, int64_t n_rows, int64_t seq_len, int distill_all,
                              float* counts2, void* stream) {
  LMOD_CHECK_ARG(labels && counts2 && n_rows > 0 && seq_len > 0 && n_rows % seq_len == 0,
                 "lmod_kl_counts: bad arguments (n_rows=%lld seq_len=%lld)", (long long)n_rows, (long long)seq_len);
  kl_counts_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(labels, n_rows, seq_len, distill_all, counts2);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_kl_finalize(const float* row_out, const int64_t* labels, int64_t n_rows, int64_t seq_len,
                                int distill_all, float* out4, void* stream) {
  LMOD_CHECK_ARG(row_out && labels && out4 && n_rows > 0 && seq_len > 0, "lmod_kl_finalize: bad arguments");
  kl_finalize_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(row_out, labels, n_rows, seq_len, distill_all, out4);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

static int kl_stream_launch(const KlParams& p, int64_t n_rows, cudaStream_t stream) {
  const size_t smem = (size_t)KS_STAGES * KS_CH * 4;
  static bool attr_done = false;
  if (!attr_done) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(kl_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = KS_CS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(KS_THREADS + 32); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cfg.gridDim = dim3(KS_CS);
  static int max_clusters = 0;                                   // co-resident clusters: queried once, outside any capture
  if (max_clusters <= 0) {
    cudaError_t e = cudaOccupancyMaxActiveClusters(&max_clusters, kl_stream_kernel, &cfg);
    if (e != cudaSuccess || max_clusters <= 0) { (void)cudaGetLastError(); max_clusters = lmod_num_sms() / KS_CS; }
    if (getenv("LMOD_KL_VERBOSE"))
      fprintf(stderr, "[lmod] kl_stream_kernel: cluster %d, %zu B smem, %d co-resident clusters\n", KS_CS, smem, max_clusters);
  }
  int64_t ncl = n_rows < max_clusters ? n_rows : max_clusters;
  cfg.gridDim = dim3((unsigned)(ncl * KS_CS));
  LMOD_CUDA_OK(cudaLaunchKernelEx(&cfg, kl_stream_kernel, p));
  lmod_count_launch();
  return LMOD_OK;
}

extern "C" int lmod_kl_fwd_bwd_rows(const void* s_logits, int64_t ld_s, const void* t_logits, int64_t ld_t,
                                    const int64_t* labels, int64_t n_rows, int64_t seq_len, int64_t vocab,
                                    int distill_all, float w_kd, float w_ce, const float* counts2,
                                    float* row_out, void* dlogits, int64_t ld_d, const int32_t* perm, const int32_t* count, void* stream) {
  LMOD_CHECK_ARG(s_logits && t_logits && labels && counts2 && row_out, "lmod_kl_fwd_bwd: null pointer");
  LMOD_CHECK_ARG(n_rows > 0 && seq_len > 0 && n_rows % seq_len == 0, "lmod_kl_fwd_bwd: n_rows %% seq_len != 0");
  LMOD_CHECK_ARG(vocab >= 8 && vocab % 8 == 0 && ld_s % 8 == 0 && ld_t % 8 == 0 && ld_s >= vocab && ld_t >= vocab,
                 "lmod_kl_fwd_bwd: vocab and row strides must be multiples of 8 elements (16-byte TMA bulk copies)");
  LMOD_CHECK_ARG(((uintptr_t)s_logits % 16 == 0) && ((uintptr_t)t_logits % 16 == 0), "lmod_kl_fwd_bwd: pointers must be 16B aligned");
  if (dlogits) LMOD_CHECK_ARG(ld_d % 8 == 0 && ld_d >= vocab && ((uintptr_t)dlogits % 16 == 0), "lmod_kl_fwd_bwd: bad dlogits stride");
  LMOD_CHECK_ARG(vocab <= KL_MAX_VOCAB, "lmod_kl_fwd_bwd: vocab %lld above the supported maximum %lld", (long long)vocab,
                 (long long)KL_MAX_VOCAB);
  LMOD_CHECK_ARG((perm == nullptr) == (count == nullptr), "lmod_kl_fwd_bwd_rows: perm and count go together");

  const int64_t per = (vocab + KS_CS - 1) / KS_CS;
  KlParams p;
  p.s = (const __nv_bfloat16*)s_logits; p.t = (const __nv_bfloat16*)t_logits; p.labels = labels;
  p.counts = counts2; p.row_out = row_out; p.d = (__nv_bfloat16*)dlogits;
  p.ld_s = ld_s; p.ld_t = ld_t; p.ld_d = ld_d; p.n_rows = n_rows; p.seq_len = seq_len;
  p.vocab = (int)vocab; p.slice = (int)((per + 7) / 8 * 8); p.distill_all = distill_all; p.w_kd = w_kd; p.w_ce = w_ce;
  p.perm = perm; p.count = count;
  return kl_stream_launch(p, n_rows, (cudaStream_t)stream);
}

extern "C" int lmod_kl_fwd_bwd(const void* s_logits, int64_t ld_s, const void* t_logits, int64_t ld_t,
                               const int64_t* labels, int64_t n_rows, int64_t seq_len, int64_t vocab,
                               int distill_all, float w_kd, float w_ce, const float* counts2,
                               float* row_out, void* dlogits, int64_t ld_d, void* stream) {
  return lmod_kl_fwd_bwd_rows(s_logits, ld_s, t_logits, ld_t, labels, n_rows, seq_len, vocab, distill_all, w_kd, w_ce, counts2, row_out,
                              dlogits, ld_d, nullptr, nullptr, stream);
}
