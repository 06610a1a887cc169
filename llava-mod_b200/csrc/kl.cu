// kl.cu -- fused mimic-KL (+ shifted CE) forward+backward over the vocabulary.
//
// Replaces (reference) llavamod/train/align_trainer.py:473-475 (teacher softmax fp32), :497-499
// (student log_softmax fp32), :509-526 (product / masked_fill / vocab sum / masked mean) and
// llava_qwen1_5_moe.py:413-421 (shifted CE), i.e. >= 8 full [N,V] passes, by ONE sweep:
//
//   * a row (V = 151936 bf16 logits, student + teacher = 608 KB) does not fit one SM's shared
//     memory, so a thread-block CLUSTER of 8 CTAs owns a row: each CTA pulls its 1/8 slice of both
//     rows into shared memory with 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx),
//     reduces max / sum-exp / sum p_T*s locally, exchanges 6 floats through distributed shared
//     memory (one barrier.cluster per row), then produces the gradient slice from the SAME shared
//     memory copy.  HBM traffic is therefore exactly the algorithmic 4*V bytes read + 2*V written
//     per token; nothing is re-read.
//   * two CTAs are resident per SM (<= 2 x 76 KB smem) so one CTA's loads overlap the other's math.
//   * rows whose KD mask and CE mask are both 0 contribute nothing (reference multiplies by 0):
//     their loads are skipped and their gradient slice is zero-filled.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "common.cuh"

namespace {

constexpr int KL_CHUNKS = 4;       // mbarrier-tracked load chunks per slice
constexpr int KL_MAX_CS = 8;
constexpr int KL_MIN_CTAS = 2;       // two CTAs per SM (2 x 76 KB of shared memory)
constexpr int KL_DEFAULT_MODE = 5;      // sb128: the fastest of the shared-memory-resident modes

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
  int keep_tail;         // stream kernel: 1 = the last ring-full of pass-1 chunks stays in shared memory for pass 2 (0: A/B arm, LMOD_KL_KEEP=0)
};

struct Xchg {            // per-CTA partials published to the cluster
  float ms, mt, zs, zt, a, slab, pad0, pad1;
};

__device__ __forceinline__ uint32_t hmax2_u32(uint32_t a, uint32_t b) {
  __nv_bfloat162 r = __hmax2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
  return *reinterpret_cast<uint32_t*>(&r);
}
__device__ __forceinline__ uint32_t hmin2_u32(uint32_t a, uint32_t b) {
  __nv_bfloat162 r = __hmin2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
  return *reinterpret_cast<uint32_t*>(&r);
}

template <bool CHECK_INF>
__device__ __forceinline__ void accum_pair(uint32_t sw, uint32_t tw, float nms, float nmt, float& zs,
                                           float& zt, float& a, float& zk) {
  float s0 = bf16lo(sw), s1 = bf16hi(sw), t0 = bf16lo(tw), t1 = bf16hi(tw);
  float es0 = ex2f(fmaf(s0, LOG2E_F, nms)), es1 = ex2f(fmaf(s1, LOG2E_F, nms));
  float et0 = ex2f(fmaf(t0, LOG2E_F, nmt)), et1 = ex2f(fmaf(t1, LOG2E_F, nmt));
  zs += es0; zs += es1;
  zt += et0; zt += et1;
  if (CHECK_INF) {   // align_trainer.py:509-510: terms where log q_S is +-inf are dropped
    if (isinf(s0)) { s0 = 0.f; et0 = 0.f; }
    if (isinf(s1)) { s1 = 0.f; et1 = 0.f; }
    zk += et0; zk += et1;      // teacher mass of the KEPT terms: x = sum_kept p_T*(s - lse_S)
  }
  a = fmaf(et0, s0, a);
  a = fmaf(et1, s1, a);
}

// NBUF = 1 (default): one slice buffer, two CTAs per SM hide each other's loads AND each other's barrier waits.
// NBUF = 2 (LMOD_KL_MODE=db256/db512, experiment kept for the record): one CTA per SM with two slice buffers, the loads of the cluster's
// NEXT active row issued before the math of the current one.  Measured 1.6-1.8x SLOWER: with one CTA per SM nothing fills the SM while
// the CTA sits in __syncthreads / barrier.cluster (22 % of warp samples), and only 15 clusters of 8 single-CTA SMs fit the GPCs.
template <int KL_THREADS, int NBUF>
__global__ void __launch_bounds__(KL_THREADS, NBUF == 2 ? 1 : KL_MIN_CTAS) kl_fused_kernel(const KlParams p) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ __align__(16) Xchg xchg[2];
  __shared__ __align__(8) uint64_t bars_all[NBUF][KL_CHUNKS];
  __shared__ float red[7][KL_THREADS / 32];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank(), cs = cluster_nctarank();
  const uint32_t cid = cluster_id_x(), ncl = cluster_nclusters_x();

  const size_t buf_bytes = (size_t)p.slice * 4;                 // student + teacher slice

  // this CTA's slice of the vocabulary
  const int v0 = (int)rank * p.slice;
  int len = p.vocab - v0;
  len = len < 0 ? 0 : (len > p.slice ? p.slice : len);
  const int nvec = len >> 3;                                   // 16-byte vectors (8 bf16)
  const int cvec = ((nvec + KL_CHUNKS - 1) / KL_CHUNKS);        // vectors per chunk

  if (tid == 0) {
    for (int b = 0; b < NBUF; ++b)
      for (int c = 0; c < KL_CHUNKS; ++c) mbar_init(&bars_all[b][c], 1);
    mbar_fence_init();
  }
  __syncthreads();
  cluster_sync_all();

  const float n_kd = p.counts[0], n_ce = p.counts[1];
  uint32_t it_active = 0;

  const int64_t n_rows = p.count ? (int64_t)*p.count : p.n_rows;
  for (int64_t row = cid; row < n_rows; row += ncl) {
    // ---- masks (uniform over the cluster) ----
    const int64_t orow = p.perm ? (int64_t)p.perm[row] : row;     // where this row sits in the batch: labels and row_out are indexed by it
    const int64_t lab_here = p.labels[orow];
    const int64_t tpos = orow % p.seq_len;
    int64_t lab_next = LMOD_IGNORE_INDEX;
    if (tpos + 1 < p.seq_len) lab_next = p.labels[orow + 1];
    const bool m_kd = p.distill_all ? true : (lab_here != LMOD_IGNORE_INDEX);
    const bool m_ce = (lab_next != LMOD_IGNORE_INDEX);   // nll is always reported (loss/lm metric); w_ce only scales its gradient
    const bool active = m_kd || m_ce;

    if (!active) {
      if (p.d != nullptr) {
        uint4 z = make_uint4(0, 0, 0, 0);
        uint4* dst = reinterpret_cast<uint4*>(p.d + row * p.ld_d + v0);
        for (int i = tid; i < nvec; i += KL_THREADS) stg_v4(dst + i, z);
      }
      if (rank == 0 && tid == 0) {
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(p.row_out + orow * 4) = o;
      }
      continue;
    }
    const uint32_t xi = it_active & 1u;                                        // exchange slot
    const uint32_t bsel = (NBUF == 2) ? (it_active & 1u) : 0u;                  // slice buffer
    const uint32_t par = (NBUF == 2) ? ((it_active >> 1) & 1u) : (it_active & 1u);
    uint64_t* bars = bars_all[bsel];
    uint4* s_buf = reinterpret_cast<uint4*>(smem_raw + bsel * buf_bytes);
    uint4* t_buf = reinterpret_cast<uint4*>(smem_raw + bsel * buf_bytes + (size_t)p.slice * 2);

    // ---- issue the slice loads (1-D TMA bulk copies), chunked so math can start early ----
    auto issue_row = [&](int64_t r, uint32_t b) {
      if (nvec <= 0) return;
      const __nv_bfloat16* srow = p.s + r * p.ld_s + v0;
      const __nv_bfloat16* trow = p.t + r * p.ld_t + v0;
      uint4* sb = reinterpret_cast<uint4*>(smem_raw + b * buf_bytes);
      uint4* tb = reinterpret_cast<uint4*>(smem_raw + b * buf_bytes + (size_t)p.slice * 2);
      for (int c = 0; c < KL_CHUNKS; ++c) {
        int cb = c * cvec, ce = min(nvec, cb + cvec);
        if (ce <= cb) { mbar_arrive(&bars_all[b][c]); continue; }
        uint32_t bytes = (uint32_t)(ce - cb) * 16u;
        mbar_expect_tx(&bars_all[b][c], 2 * bytes);
        bulk_g2s(sb + cb, srow + (size_t)cb * 8, bytes, &bars_all[b][c]);
        bulk_g2s(tb + cb, trow + (size_t)cb * 8, bytes, &bars_all[b][c]);
      }
    };
    if (NBUF == 1) {
      if (tid == 0) issue_row(row, 0);
    } else if (warp == 0) {
      // the first active row loads itself; every active row then looks ahead (32 candidate rows per ballot) for the cluster's next
      // active row and starts ITS loads into the other buffer, which the previous row released at its closing __syncthreads
      if (it_active == 0 && lane == 0) issue_row(row, 0);
      int64_t nxt = -1;
      for (int64_t base = row; base + ncl < n_rows; base += 32 * (int64_t)ncl) {
        const int64_t r = base + (int64_t)(lane + 1) * ncl;
        bool act = false;
        if (r < n_rows) {
          const int64_t ro = p.perm ? (int64_t)p.perm[r] : r;
          act = p.distill_all || (p.labels[ro] != LMOD_IGNORE_INDEX);
          if (!act && (ro % p.seq_len) + 1 < p.seq_len) act = p.labels[ro + 1] != LMOD_IGNORE_INDEX;
        }
        const unsigned m = __ballot_sync(0xffffffffu, act);
        if (m) { nxt = base + (int64_t)__ffs(m) * ncl; break; }
      }
      if (lane == 0 && nxt >= 0) issue_row(nxt, bsel ^ 1u);
    }
    ++it_active;

    // ---- pass A+B (one sweep, chunk by chunk as the bulk copies land): running maxima with rescaled partial sums -------------------
    // per thread: (m_s, zs = sum e^{s-m_s}) and (m_t, zt = sum e^{t-m_t}, acc = sum e^{t-m_t} s, zk = kept teacher mass).  The running
    // maxima settle after a few vectors, so the rescale branch is cold.  Infinite logits never enter a running maximum: -inf terms vanish
    // on their own, +inf keeps the old degenerate outcome (sum-exp = inf); vectors that hold an infinite student logit take the checked path
    // (align_trainer.py:509-510 drops those terms).
    float m_s = -INFINITY, m_t = -INFINITY, zs = 0.f, zt = 0.f, acc = 0.f, zk = 0.f;
    if (nvec > 0) {
      for (int c = 0; c < KL_CHUNKS; ++c) {
        const int b0 = c * cvec, e0 = min(nvec, b0 + cvec);
        mbar_wait(&bars[c], par);
        for (int i = b0 + tid; i < e0; i += KL_THREADS) {
          const uint4 sv = s_buf[i], tv = t_buf[i];
          const uint32_t pmx_s = hmax2_u32(hmax2_u32(sv.x, sv.y), hmax2_u32(sv.z, sv.w));
          const uint32_t pmn_s = hmin2_u32(hmin2_u32(sv.x, sv.y), hmin2_u32(sv.z, sv.w));
          const uint32_t pmx_t = hmax2_u32(hmax2_u32(tv.x, tv.y), hmax2_u32(tv.z, tv.w));
          const float vmax_s = fmaxf(bf16lo(pmx_s), bf16hi(pmx_s)), vmin_s = fminf(bf16lo(pmn_s), bf16hi(pmn_s));
          const float vmax_t = fmaxf(bf16lo(pmx_t), bf16hi(pmx_t));
          if (vmax_s > m_s && !isinf(vmax_s)) {
            zs *= ex2f((m_s - vmax_s) * LOG2E_F);                      // m_s = -inf the first time: zs = 0 * 0
            m_s = vmax_s;
          }
          if (vmax_t > m_t && !isinf(vmax_t)) {
            const float f = ex2f((m_t - vmax_t) * LOG2E_F);
            zt *= f; acc *= f; zk *= f;
            m_t = vmax_t;
          }
          const float nms = isinf(m_s) ? 0.f : -m_s * LOG2E_F, nmt = isinf(m_t) ? 0.f : -m_t * LOG2E_F;
          if (!(isinf(vmin_s) || isinf(vmax_s))) {
            float zk_unused = 0.f;
            accum_pair<false>(sv.x, tv.x, nms, nmt, zs, zt, acc, zk_unused);
            accum_pair<false>(sv.y, tv.y, nms, nmt, zs, zt, acc, zk_unused);
            accum_pair<false>(sv.z, tv.z, nms, nmt, zs, zt, acc, zk_unused);
            accum_pair<false>(sv.w, tv.w, nms, nmt, zs, zt, acc, zk_unused);
            // all terms kept: the kept teacher mass of this vector equals its share of zt (added below through dzt)
          } else {
            const float zt0 = zt;
            float zk_v = 0.f;
            accum_pair<true>(sv.x, tv.x, nms, nmt, zs, zt, acc, zk_v);
            accum_pair<true>(sv.y, tv.y, nms, nmt, zs, zt, acc, zk_v);
            accum_pair<true>(sv.z, tv.z, nms, nmt, zs, zt, acc, zk_v);
            accum_pair<true>(sv.w, tv.w, nms, nmt, zs, zt, acc, zk_v);
            zk += zk_v - (zt - zt0);                                   // zk tracks (kept - all) teacher mass; the final zk = zt + this
          }
        }
      }
    }
    zk += zt;                                                         // kept teacher mass on this thread's scale m_t
    // ---- block reduction with the (max, scaled sums) combine; one __syncthreads ----
    {
      float Ms = warp_max(m_s), Mt = warp_max(m_t);
      const float fs = isinf(m_s) ? 0.f : ex2f((m_s - Ms) * LOG2E_F);   // Ms finite whenever some lane's m_s is
      const float ft = isinf(m_t) ? 0.f : ex2f((m_t - Mt) * LOG2E_F);
      zs = warp_sum(isinf(zs) ? zs : zs * fs);                          // an infinite sum-exp (+inf logit) stays infinite
      zt = warp_sum(isinf(zt) ? zt : zt * ft);
      acc = warp_sum(acc * ft); zk = warp_sum(zk * ft);
      if (lane == 0) { red[0][warp] = Ms; red[1][warp] = Mt; red[3][warp] = zs; red[4][warp] = zt; red[5][warp] = acc; red[6][warp] = zk; }
    }
    __syncthreads();
    float ms = -INFINITY, mt = -INFINITY;
    if (warp == 0) {
      constexpr int NW = KL_THREADS / 32;
      const float wms = (lane < NW) ? red[0][lane] : -INFINITY, wmt = (lane < NW) ? red[1][lane] : -INFINITY;
      ms = warp_max(wms); mt = warp_max(wmt);
      const float fs = isinf(wms) ? 0.f : ex2f((wms - ms) * LOG2E_F);
      const float ft = isinf(wmt) ? 0.f : ex2f((wmt - mt) * LOG2E_F);
      float a = (lane < NW) ? red[3][lane] : 0.f, b = (lane < NW) ? red[4][lane] : 0.f;
      float c = (lane < NW) ? red[5][lane] : 0.f, k = (lane < NW) ? red[6][lane] : 0.f;
      a = warp_sum(isinf(a) ? a : a * fs); b = warp_sum(isinf(b) ? b : b * ft);
      c = warp_sum(c * ft); k = warp_sum(k * ft);
      if (lane == 0) {
        float slab = 0.f;
        if (m_ce) {
          int64_t off = lab_next - v0;
          if (off >= 0 && off < len)
            slab = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(s_buf)[off]);
        }
        Xchg x;
        x.ms = (nvec > 0) ? ms : -INFINITY; x.mt = (nvec > 0) ? mt : -INFINITY;
        x.zs = a; x.zt = b; x.a = c; x.slab = slab; x.pad0 = k; x.pad1 = 0.f;
        xchg[xi] = x;
      }
    }
    // ---- cluster exchange through distributed shared memory ----
    cluster_sync_all();
    float lse_s, lse_t, xrow, slab;
    {
      float r_ms = -INFINITY, r_mt = -INFINITY, r_zs = 0.f, r_zt = 0.f, r_a = 0.f, r_sl = 0.f, r_zk = 0.f;
      if ((uint32_t)lane < cs) {
        const float* base = reinterpret_cast<const float*>(&xchg[xi]);
        r_ms = dsmem_ld_f32(base + 0, lane); r_mt = dsmem_ld_f32(base + 1, lane);
        r_zs = dsmem_ld_f32(base + 2, lane); r_zt = dsmem_ld_f32(base + 3, lane);
        r_a = dsmem_ld_f32(base + 4, lane);  r_sl = dsmem_ld_f32(base + 5, lane); r_zk = dsmem_ld_f32(base + 6, lane);
      }
      float Ms = warp_max(r_ms), Mt = warp_max(r_mt);
      float Ms_u = isinf(Ms) ? 0.f : Ms, Mt_u = isinf(Mt) ? 0.f : Mt;
      float fs = isinf(r_ms) ? 0.f : ex2f((r_ms - Ms_u) * LOG2E_F);
      float ft = isinf(r_mt) ? 0.f : ex2f((r_mt - Mt_u) * LOG2E_F);
      float Zs = warp_sum(r_zs * fs), Zt = warp_sum(r_zt * ft), A = warp_sum(r_a * ft), Zk = warp_sum(r_zk * ft);
      slab = warp_sum(r_sl);
      lse_s = Ms_u + lg2f(Zs) * LN2_F;
      lse_t = Mt_u + lg2f(Zt) * LN2_F;
      xrow = (A - lse_s * Zk) / Zt;
    }
    if (rank == 0 && tid == 0) {
      float4 o = make_float4(xrow, m_ce ? (lse_s - slab) : 0.f, lse_s, lse_t);
      *reinterpret_cast<float4*>(p.row_out + orow * 4) = o;
    }

    // ---- pass C: gradient slice straight from shared memory ----
    if (p.d != nullptr) {
      const float ckd = m_kd ? (p.w_kd / n_kd) : 0.f;
      const float cce = m_ce ? (p.w_ce / n_ce) : 0.f;
      const float ca = ckd + cce, cb = ckd;
      const float es = -lse_s * LOG2E_F, et = -lse_t * LOG2E_F;
      const int lab_local = m_ce ? (int)(lab_next - v0) : -1;
      uint4* dst = reinterpret_cast<uint4*>(p.d + row * p.ld_d + v0);
      for (int i = tid; i < nvec; i += KL_THREADS) {
        uint4 sv = s_buf[i], tv = t_buf[i];
        float g[8];
        const uint32_t sw[4] = {sv.x, sv.y, sv.z, sv.w};
        const uint32_t tw[4] = {tv.x, tv.y, tv.z, tv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float q0 = ex2f(fmaf(bf16lo(sw[j]), LOG2E_F, es)), q1 = ex2f(fmaf(bf16hi(sw[j]), LOG2E_F, es));
          float p0 = ex2f(fmaf(bf16lo(tw[j]), LOG2E_F, et)), p1 = ex2f(fmaf(bf16hi(tw[j]), LOG2E_F, et));
          g[2 * j] = fmaf(ca, q0, -cb * p0);
          g[2 * j + 1] = fmaf(ca, q1, -cb * p1);
        }
        const unsigned rel = (unsigned)(lab_local - i * 8);
        if (rel < 8u) {
#pragma unroll
          for (int j = 0; j < 8; ++j) if (rel == (unsigned)j) g[j] -= cce;
        }
        uint4 o;
        o.x = pack_bf16x2(g[0], g[1]); o.y = pack_bf16x2(g[2], g[3]);
        o.z = pack_bf16x2(g[4], g[5]); o.w = pack_bf16x2(g[6], g[7]);
        stg_v4(dst + i, o);
      }
    }
    __syncthreads();   // all generic-proxy reads of the slice are done before the next bulk load lands
  }
  cluster_sync_all();  // keep this CTA's shared memory alive until every peer finished its DSMEM reads
}

// =====================================================================================================================
// Streaming form (default): ONE CTA owns a row (a cluster of 2 / 4 CTAs sharing a row through DSMEM is kept as an experiment) and STREAMS
// it through a shared-memory ring fed by a dedicated TMA-producer warp, twice:
//   pass 1  online max / sum-exp / sum p_T*s over the half row (no per-row shared-memory residency, so no 76 KB-per-row limit and no
//           load latency in front of the math: the ring always holds the next chunks);
//   pass 2  the same chunks again -- issued by the producer right behind pass 1, so they come out of L2 as long as the rows in flight
//           fit in it -- turned into the gradient and written back in place.
// On H100 (50 MB L2, 132 SMs) one CTA per row keeps 132 rows x 0.6 MB = 79 MB in flight and pass 2 partly misses; two CTAs per row
// (a cluster of 2 sharing the row through DSMEM) keep 66 rows = 40 MB in flight.  Timed on one H100 (400 W limit), 885 rows x 151936:
// 0.338 ms with two CTAs per row against 0.415 ms with one -> two is the default.
// The per-row fixed cost (block reduction + exchange between the CTAs of a row) is paid once per HALF row of 76 K logit pairs instead
// of once per 19 K-pair slice, and the exchange is a DSMEM store + remote mbarrier arrive instead of a barrier.cluster, so the producer
// warp never stops prefetching.  HBM traffic stays the algorithmic 4V read + 2V written per token as long as pass 2 hits L2
// (DRAM bytes read per launch is the check).
// =====================================================================================================================
constexpr int KS_CS = 2;                 // CTAs per row (a cluster shares a row through DSMEM; LMOD_KL_MODE=stream1 / stream4 override)
constexpr int KS_CH = 8192;              // logit pairs per ring stage (16 KB student + 16 KB teacher)
constexpr int KS_STAGES = 6;             // 192 KB ring

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
__device__ __forceinline__ void ks_wait(uint64_t* bar, uint32_t phase);
// one lane polls, the warp sleeps at the warp barrier (512 polling threads would fight the loads for the LSU)
__device__ __forceinline__ void ks_wait_warp(uint64_t* bar, uint32_t phase) {
  if ((threadIdx.x & 31) == 0) ks_wait(bar, phase);
  __syncwarp();
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


// ---- two-lane arithmetic + exp2 on the FMA / ALU pipes ----------------------------------------------------------------------------
// The kernel needs 4 exponentials per (student, teacher) logit pair and the MUFU pipe retires 16 per clock per SM: at V = 151936 that
// is about the HBM time of the row.  A share of the exponentials is therefore evaluated WITHOUT the MUFU: Cody-Waite split
// x = n + f, f in [-0.5, 0.5], 2^f by a degree-4 minimax polynomial (max relative error 3.7e-6), 2^n by an integer add into the exponent.
// Inputs are <= 0 here (logit - running max), clamped at -126.  Every operation is rounded to nearest (no contraction into other FMAs).
__device__ __forceinline__ float exp2_poly1(float x, uint32_t& t) {
  const float tf = __fadd_rn(x, 12582912.f);          // t = x + 1.5*2^23: the integer part sits in the low mantissa bits
  const float n = __fadd_rn(tf, -12582912.f);         // n = round(x)
  const float f = __fmaf_rn(n, -1.f, x);              // f = x - n
  float p = 9.676037098e-03f;
  p = __fmaf_rn(p, f, 5.592203565e-02f);
  p = __fmaf_rn(p, f, 2.402210736e-01f);
  p = __fmaf_rn(p, f, 6.931210340e-01f);
  p = __fmaf_rn(p, f, 1.000000075f);
  t = __float_as_uint(tf);
  return p;
}
__device__ __forceinline__ void exp2_poly2(float x0, float x1, float& y0, float& y1) {
  x0 = fmaxf(x0, -126.f); x1 = fmaxf(x1, -126.f);
  uint32_t t0, t1;
  const float p0 = exp2_poly1(x0, t0), p1 = exp2_poly1(x1, t1);
  y0 = __uint_as_float(__float_as_uint(p0) + (t0 << 23));
  y1 = __uint_as_float(__float_as_uint(p1) + (t1 << 23));
}
__device__ __forceinline__ void ffma2_bcast(float& d0, float& d1, float a0, float a1, float b, float c) {      // d = a * b + c
  d0 = __fmaf_rn(a0, b, c); d1 = __fmaf_rn(a1, b, c);
}
__device__ __forceinline__ void fadd2_into(float& d0, float& d1, float a0, float a1) {                         // d += a
  d0 = __fadd_rn(d0, a0); d1 = __fadd_rn(d1, a1);
}
__device__ __forceinline__ void ffma2_into(float& d0, float& d1, float a0, float a1, float b0, float b1) {     // d += a * b
  d0 = __fmaf_rn(a0, b0, d0); d1 = __fmaf_rn(a1, b1, d1);
}
// two-lane accumulators of the online pass
struct Acc2 { float zs0, zs1, zt0, zt1, a0, a1; };
// one 32-bit word of student logits + one of teacher logits (two vocabulary positions): exponentials by MUFU or by the polynomial
template <bool S_POLY, bool T_POLY>
__device__ __forceinline__ void accum_word(uint32_t sw, uint32_t tw, float nms, float nmt, Acc2& A) {
  const float s0 = bf16lo(sw), s1 = bf16hi(sw), t0 = bf16lo(tw), t1 = bf16hi(tw);
  float xs0, xs1, xt0, xt1, es0, es1, et0, et1;
  ffma2_bcast(xs0, xs1, s0, s1, LOG2E_F, nms);
  ffma2_bcast(xt0, xt1, t0, t1, LOG2E_F, nmt);
  if (S_POLY) exp2_poly2(xs0, xs1, es0, es1); else { es0 = ex2f(xs0); es1 = ex2f(xs1); }
  if (T_POLY) exp2_poly2(xt0, xt1, et0, et1); else { et0 = ex2f(xt0); et1 = ex2f(xt1); }
  fadd2_into(A.zs0, A.zs1, es0, es1);
  fadd2_into(A.zt0, A.zt1, et0, et1);
  ffma2_into(A.a0, A.a1, et0, et1, s0, s1);
}
// gradient of one word: g = ca * q_S - cb * p_T
template <bool S_POLY, bool T_POLY>
__device__ __forceinline__ uint32_t grad_word(uint32_t sw, uint32_t tw, float es, float et, float ca, float ncb, float& g0, float& g1) {
  float xs0, xs1, xt0, xt1, q0, q1, p0, p1;
  ffma2_bcast(xs0, xs1, bf16lo(sw), bf16hi(sw), LOG2E_F, es);
  ffma2_bcast(xt0, xt1, bf16lo(tw), bf16hi(tw), LOG2E_F, et);
  if (S_POLY) exp2_poly2(xs0, xs1, q0, q1); else { q0 = ex2f(xs0); q1 = ex2f(xs1); }
  if (T_POLY) exp2_poly2(xt0, xt1, p0, p1); else { p0 = ex2f(xt0); p1 = ex2f(xt1); }
  float c0, c1;
  ffma2_bcast(c0, c1, p0, p1, ncb, 0.f);                  // -cb * p
  g0 = __fmaf_rn(q0, ca, c0); g1 = __fmaf_rn(q1, ca, c1);
  return 0u;
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

// P1 / P2: how many of the 8 word-level exponential pairs of a 16-byte vector (4 words x {student, teacher}) use the polynomial in pass 1 / 2
// KS_THREADS: consumer threads (+ one producer warp)
template <int P1, int P2, int KS_THREADS>
__global__ void __launch_bounds__(KS_THREADS + 32, 1) kl_stream_kernel(const KlParams p) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ __align__(16) XchgS xchg[2][KL_MAX_CS];            // [slot][source CTA]: written by the peers through DSMEM
  __shared__ __align__(8) uint64_t full[KS_STAGES], empty[KS_STAGES], xbar[2];
  __shared__ float red[7][KS_THREADS / 32];
  __shared__ float s_lab;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank(), cs = cluster_nctarank();
  const uint32_t cid = cluster_id_x(), ncl = cluster_nclusters_x();
  const int v0 = (int)rank * p.slice;
  int len = p.vocab - v0;
  len = len < 0 ? 0 : (len > p.slice ? p.slice : len);
  const int nchunks = (len + KS_CH - 1) / KS_CH;
  const bool want_grad = p.d != nullptr;
  const int held = (want_grad && p.keep_tail) ? min(KS_STAGES, nchunks) : 0;     // pass-1 chunks kept in the ring for pass 2

  if (tid == 0) {
    for (int i = 0; i < KS_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], KS_THREADS / 32); }
    mbar_init(&xbar[0], cs); mbar_init(&xbar[1], cs);
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
            accum_word<(P1 > 0), (P1 > 1)>(sv.x, tv.x, nms, nmt, A);
            accum_word<(P1 > 2), (P1 > 3)>(sv.y, tv.y, nms, nmt, A);
            accum_word<(P1 > 4), (P1 > 5)>(sv.z, tv.z, nms, nmt, A);
            accum_word<(P1 > 6), (P1 > 7)>(sv.w, tv.w, nms, nmt, A);
          } else {
            // a vector that holds an infinite student logit: scalar path that drops those terms (align_trainer.py:509-510)
            float zs = 0.f, zt = 0.f, acc = 0.f, zk_v = 0.f;
            accum_pair<true>(sv.x, tv.x, nms, nmt, zs, zt, acc, zk_v);
            accum_pair<true>(sv.y, tv.y, nms, nmt, zs, zt, acc, zk_v);
            accum_pair<true>(sv.z, tv.z, nms, nmt, zs, zt, acc, zk_v);
            accum_pair<true>(sv.w, tv.w, nms, nmt, zs, zt, acc, zk_v);
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
        if (cs == 1) {
          // one CTA per row: the block totals go through shared memory and a named barrier (no DSMEM, no cluster-scope acquire -- ptxas
          // turns that into an L1 invalidate per poll)
          if (lane == 0) {
            XchgS x;
            x.ms = (len > 0) ? ms : -INFINITY; x.mt = (len > 0) ? mt : -INFINITY; x.zs = a; x.zt = b; x.a = c2; x.slab = sl; x.zk = k; x.pad = 0.f;
            xchg[xi][0] = x;
          }
        } else if ((uint32_t)lane < cs) {
          // publish this CTA's partials into slot [xi][rank] of EVERY CTA of the cluster (lane l -> CTA l), then arrive on its barrier
          const uint32_t base = mapa_u32(smem_u32(&xchg[xi][rank]), (uint32_t)lane);
          st_cluster_f32(base + 0, (len > 0) ? ms : -INFINITY); st_cluster_f32(base + 4, (len > 0) ? mt : -INFINITY);
          st_cluster_f32(base + 8, a); st_cluster_f32(base + 12, b); st_cluster_f32(base + 16, c2); st_cluster_f32(base + 20, sl);
          st_cluster_f32(base + 24, k);
          mbar_arrive_cluster(mapa_u32(smem_u32(&xbar[xi]), (uint32_t)lane));
        }
      }
      if (cs == 1) asm volatile("bar.sync 1, %0;" :: "n"(KS_THREADS) : "memory");
      else mbar_wait_cluster(&xbar[xi], xpar);
      float lse_s, lse_t, xrow, slab_row;
      {
        float r_ms = -INFINITY, r_mt = -INFINITY, r_zs = 0.f, r_zt = 0.f, r_a = 0.f, r_sl = 0.f, r_zk = 0.f;
        if ((uint32_t)lane < cs) {
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
            grad_word<(P2 > 0), (P2 > 1)>(sv.x, tv.x, es, et, ca, -cb, g[0], g[1]);
            grad_word<(P2 > 2), (P2 > 3)>(sv.y, tv.y, es, et, ca, -cb, g[2], g[3]);
            grad_word<(P2 > 4), (P2 > 5)>(sv.z, tv.z, es, et, ca, -cb, g[4], g[5]);
            grad_word<(P2 > 6), (P2 > 7)>(sv.w, tv.w, es, et, ca, -cb, g[6], g[7]);
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

template <int T, int NB>
int kl_launch(KlParams p, int cs, size_t smem, int64_t n_rows, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(kl_fused_kernel<T, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    attr_done = true;
  }
  smem *= NB;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(T); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cfg.gridDim = dim3(cs);
  static int cached_clusters[2] = {0, 0};        // per cluster size (1 / 8): queried once, outside any stream capture
  int& max_clusters = cached_clusters[cs == 1 ? 0 : 1];   // (one multi-CTA cluster size per process)
  if (max_clusters <= 0) {
    cudaError_t e = cudaOccupancyMaxActiveClusters(&max_clusters, kl_fused_kernel<T, NB>, &cfg);
    if (e != cudaSuccess || max_clusters <= 0) { (void)cudaGetLastError(); max_clusters = lmod_num_sms() / cs; }
    if (getenv("LMOD_KL_VERBOSE")) fprintf(stderr, "[lmod] kl_fused_kernel<%d,%d>: cluster %d, %zu B smem, %d co-resident clusters\n", T, NB, cs, smem, max_clusters);
  }
  int64_t ncl = n_rows < max_clusters ? n_rows : max_clusters;
  cfg.gridDim = dim3((unsigned)(ncl * cs));
  LMOD_CUDA_OK(cudaLaunchKernelEx(&cfg, kl_fused_kernel<T, NB>, p));
  lmod_count_launch();
  return LMOD_OK;
}

template <int P1, int P2, int KS_THREADS>
static int kl_stream_launch_t(KlParams p, int cs, int64_t n_rows, cudaStream_t stream) {
  const size_t smem = (size_t)KS_STAGES * KS_CH * 4;
  static bool attr_done = false;
  if (!attr_done) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(kl_stream_kernel<P1, P2, KS_THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(KS_THREADS + 32); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cfg.gridDim = dim3(cs);
  static int cached[KL_MAX_CS + 1] = {0};                        // co-resident clusters per cluster size: queried once, outside any capture
  int& max_clusters = cached[cs];
  if (max_clusters <= 0) {
    cudaError_t e = cudaOccupancyMaxActiveClusters(&max_clusters, kl_stream_kernel<P1, P2, KS_THREADS>, &cfg);
    if (e != cudaSuccess || max_clusters <= 0) { (void)cudaGetLastError(); max_clusters = lmod_num_sms() / cs; }
    if (getenv("LMOD_KL_VERBOSE"))
      fprintf(stderr, "[lmod] kl_stream_kernel<%d,%d,%d>: cluster %d, %zu B smem, %d co-resident clusters, keep_tail %d\n", P1, P2, KS_THREADS, cs,
              smem, max_clusters, p.keep_tail);
  }
  int64_t ncl = n_rows < max_clusters ? n_rows : max_clusters;
  cfg.gridDim = dim3((unsigned)(ncl * cs));
  LMOD_CUDA_OK(cudaLaunchKernelEx(&cfg, kl_stream_kernel<P1, P2, KS_THREADS>, p));
  lmod_count_launch();
  return LMOD_OK;
}
// the kernel is not MUFU-bound, so the extra FMA-pipe instructions of the polynomial exponentials only cost issue slots; the MUFU-only
// form is the default and <3,3> stays as the A/B arm
static int kl_stream_launch(KlParams p, int cs, int64_t n_rows, cudaStream_t stream) {
  static const char* e = getenv("LMOD_KL_POLY");       // "33": polynomial share 3/8 in both passes
  static const char* th = getenv("LMOD_KL_THREADS");   // "256" / "768": consumer threads (default 512)
  const int nt = th ? atoi(th) : 512;
  if (e && e[0] == '3') return kl_stream_launch_t<3, 3, 512>(p, cs, n_rows, stream);
  if (nt == 256) return kl_stream_launch_t<0, 0, 256>(p, cs, n_rows, stream);
  if (nt == 768) return kl_stream_launch_t<0, 0, 768>(p, cs, n_rows, stream);
  return kl_stream_launch_t<0, 0, 512>(p, cs, n_rows, stream);
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

  int cs = (vocab >= 512) ? KL_MAX_CS : 1;
  int64_t per = (vocab + cs - 1) / cs;
  int slice = (int)((per + 7) / 8 * 8);
  size_t smem = (size_t)slice * 2 * 2;
  LMOD_CHECK_ARG(smem <= 220 * 1024, "lmod_kl_fwd_bwd: vocab %lld too large for the 8-CTA cluster layout", (long long)vocab);

  KlParams p;
  p.s = (const __nv_bfloat16*)s_logits; p.t = (const __nv_bfloat16*)t_logits; p.labels = labels;
  p.counts = counts2; p.row_out = row_out; p.d = (__nv_bfloat16*)dlogits;
  p.ld_s = ld_s; p.ld_t = ld_t; p.ld_d = ld_d; p.n_rows = n_rows; p.seq_len = seq_len;
  static const int keep_env = getenv("LMOD_KL_KEEP") ? atoi(getenv("LMOD_KL_KEEP")) : 1;
  p.keep_tail = keep_env;
  p.vocab = (int)vocab; p.slice = slice; p.distill_all = distill_all; p.w_kd = w_kd; p.w_ce = w_ce;
  LMOD_CHECK_ARG((perm == nullptr) == (count == nullptr), "lmod_kl_fwd_bwd_rows: perm and count go together");
  p.perm = perm; p.count = count;

  // LMOD_KL_MODE: unset / "stream" = the streaming kernel (KS_CS CTAs per row, ring + L2 re-read); "stream1" / "stream2" / "stream4" = 1 / 2 / 4 CTAs per row;
  // "sb128" the shared-memory-resident 8-CTA kernel (kept as an A/B arm), "sb256"/"sb384"/"sb512" its
  // thread-count variants, "db256"/"db512" its double-buffered experiments
  static const char* mode_env = getenv("LMOD_KL_MODE");
  if (!mode_env || !strncmp(mode_env, "stream", 6)) {
    int scs = KS_CS;
    if (mode_env && mode_env[6] >= '1' && mode_env[6] <= '8') scs = mode_env[6] - '0';
    int64_t sper = (vocab + scs - 1) / scs;
    p.slice = (int)((sper + 7) / 8 * 8);
    return kl_stream_launch(p, scs, n_rows, (cudaStream_t)stream);
  }
  static const int mode = !mode_env ? KL_DEFAULT_MODE
                          : (!strcmp(mode_env, "sb256") ? 0 : (!strcmp(mode_env, "db256") ? 1 : (!strcmp(mode_env, "sb512") ? 3 : (!strcmp(mode_env, "sb384") ? 4 : (!strcmp(mode_env, "sb128") ? 5 : 2)))));
  const bool db_fits = smem * 2 <= 220 * 1024;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == 3) return kl_launch<512, 1>(p, cs, smem, n_rows, st);
  if (mode == 4) return kl_launch<384, 1>(p, cs, smem, n_rows, st);
  if (mode == 5) return kl_launch<128, 1>(p, cs, smem, n_rows, st);
  if (mode == 0 || !db_fits) return kl_launch<256, 1>(p, cs, smem, n_rows, st);
  return (mode == 1) ? kl_launch<256, 2>(p, cs, smem, n_rows, st) : kl_launch<512, 2>(p, cs, smem, n_rows, st);
}

extern "C" int lmod_kl_fwd_bwd(const void* s_logits, int64_t ld_s, const void* t_logits, int64_t ld_t,
                               const int64_t* labels, int64_t n_rows, int64_t seq_len, int64_t vocab,
                               int distill_all, float w_kd, float w_ce, const float* counts2,
                               float* row_out, void* dlogits, int64_t ld_d, void* stream) {
  return lmod_kl_fwd_bwd_rows(s_logits, ld_s, t_logits, ld_t, labels, n_rows, seq_len, vocab, distill_all, w_kd, w_ce, counts2, row_out,
                              dlogits, ld_d, nullptr, nullptr, stream);
}
