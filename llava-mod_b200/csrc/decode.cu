// decode.cu -- KV-cache decoding on sm_90a: the cache append and split-KV single-query attention (flash-decoding).
//
// Replaces the past_key_value branch of Qwen2SdpaAttention.forward (modeling_qwen2.py:652-728): DynamicCache.update (cache_utils.py)
// concatenating the new k / v onto the layer's cache, then SDPA of the one new query against every cached key.
//
// Cache layout: per layer one K and one V buffer [B, nkv, max_len, hd] bf16 (HF's legacy layout); sequence b holds len[b] valid rows.
//
// lmod_attn_decode: grid (split, kv head, batch), 128 threads.  A CTA serves every query head of its GQA group, so each K / V row is
// read once per step.  Its key range [split * SK, (split + 1) * SK) ∩ [0, len[b]) streams through an NST-stage shared-memory ring
// (1-D TMA bulk copies, completion on an mbarrier per stage; only rows below len[b] are copied, so rows never written are never read).
// Per 64-key block:
//   scores  : HD/8 lanes per key, 16 B of the key row each, dot with the G query heads, reduced over the lane group by shuffles
//   softmax : one warp per head: block max, exp2 with scale*log2(e) folded into the score, running (m, l) in shared memory
//   P.V     : each thread owns two output columns of every head and a quarter (hd 64) / half (hd 128) of the keys; only keys below
//             len[b] are visited (P = 0 times a NaN row would still be NaN)
// The split writes its unnormalised fp32 output and (m, l) to the workspace; lmod_attn_decode's second launch merges the splits.
// The split length depends on max_len, nkv and the SM count only -- not on len or B -- so one captured graph serves every step and a
// sequence gives the same bits whatever batch it is decoded in.
//
// lmod_attn_decode_chunk: T new query rows per sequence (the verify step of assisted decoding), row t attending to keys
// [0, len[b] - T + t + 1).  The same kernel body with CHUNK = true: a CTA serves G "virtual heads" (row t, query head g) of one KV head, and
// each virtual head has its own key limit.  A key at or past the limit scores -inf and is skipped by P.V, and a split wholly past a row's
// limit leaves (m, l) = (-inf, 0), so row t runs the single-query kernel's arithmetic at len = len[b] - T + t + 1 operation for operation:
// the same splits, 64-key blocks, lane-to-key mapping and merge.  Its out and lse are the bytes lmod_attn_decode gives for that row alone.
//
// lmod_attn_decode_shared: n sequences per prompt (num_return_sequences) that share the prompt's K / V.  Prompt b's rows
// [0, prefix_len[b]) live once in a prefix buffer [B, nkv, P_max, hd]; copy j's rows from prefix_len[b] on in its own suffix buffer
// [B*n, nkv, S_max, hd] (suffix row i - prefix_len[b] holds key i).  The same kernel body with SHARED: a CTA serves the virtual heads
// (copy j, query head g) of one KV head, min(n, 8 / G) copies per CTA, each with its own key limit len[b*n + j].  Its key range is walked
// as a list of items: a 64-key block wholly inside the prefix is one item, loaded once and scored for every virtual head of the CTA (the
// bandwidth saving); a block that reaches past the prefix is one item per copy, loaded from the prefix and the copy's suffix rows and
// applied to that copy's heads only.
// Each copy's heads see every block of its key range once, with the lmod_attn_decode splits of the max_len passed in (the bucketed length
// the expanded cache would have), the same lane-to-key mapping, per-head limits as in the chunk kernel, and the same merge, so sequence
// b*n + j's out and lse are the bytes lmod_attn_decode gives on its materialised cache (prefix rows then suffix rows) at that max_len.
//
// lmod_kv_beam_reorder: beam search's cache reorder (HF _reorder_cache), in place and for every layer's K and V in one launch.  On the
// shared cache only the beams' suffix rows move (the prompt's rows are common to all beams); on a plain cache every row below len.
#include "sm90.cuh"

namespace {

constexpr int DEC_THREADS = 128;
constexpr int DEC_BK = 64;            // keys per ring stage
constexpr int DEC_MIN_BLOCKS = 4;     // a split covers at least this many key blocks
constexpr int DEC_MAX_G = 8;          // query heads per KV head
enum DecMode { DEC_SINGLE, DEC_CHUNK, DEC_SHARED };

template <int HD> struct DecCfg {
  static constexpr int NST = HD == 128 ? 3 : 4;
  static constexpr int KV_BYTES = DEC_BK * HD * 2;
  static constexpr int LANES = HD / 8;                  // lanes per key in the score pass
  static constexpr int GROUPS = DEC_THREADS / LANES;    // keys scored at once
  static constexpr int PAIRS = HD / 2;                  // bf16x2 output columns
  static constexpr int KSUB = DEC_THREADS / PAIRS;      // key subsets of the P.V pass
  static constexpr int SMEM = 2 * NST * KV_BYTES;
};

struct DecParams {
  const __nv_bfloat16* q;   // [B, ld_q]: the query heads of row b at columns [h*HD, (h+1)*HD)
  int64_t ld_q;
  const __nv_bfloat16* k;   // [B, nkv, max_len, HD]
  const __nv_bfloat16* v;
  const int32_t* len;       // [B] valid rows per sequence (device)
  float* ws_o;              // [B, nh, nsplit, HD] unnormalised split outputs
  float* ws_ml;             // [B, nh, nsplit, 2]  (running max in log2 units, sum of exp2)
  int nh, nkv, max_len, nsplit, split_blocks;
  float scale_log2;
  int T, g, rows;           // chunk: query rows per sequence (q / ws rows are b*T + t), query heads per KV head, rows per CTA
                            // shared: T = n copies per prompt (q / ws / len rows are b*n + j), g as chunk, rows = copies per CTA
  const __nv_bfloat16* ks;  // shared only: suffix buffers [B*n, nkv, s_max, HD]; k / v above are the prefix buffers [B, nkv, max_len, HD]
  const __nv_bfloat16* vs;
  const int32_t* plen;      // shared only: [B] prefix rows per prompt (device)
  int p_max, s_max;
};

template <int HD>
__device__ __forceinline__ void dec_issue(uint8_t* sK, uint8_t* sV, uint64_t* full, const __nv_bfloat16* kg, const __nv_bfloat16* vg,
                                          int kbeg, int kend, int j) {
  using C = DecCfg<HD>;
  const int s = j % C::NST;
  const int k0 = kbeg + j * DEC_BK;
  const uint32_t bytes = (uint32_t)min(DEC_BK, kend - k0) * HD * 2;
  mbar_expect_tx(&full[s], 2 * bytes);
  bulk_g2s(sK + s * C::KV_BYTES, kg + (size_t)k0 * HD, bytes, &full[s]);
  bulk_g2s(sV + s * C::KV_BYTES, vg + (size_t)k0 * HD, bytes, &full[s]);
}

// shared: item i of a CTA's key range -> (block j, copy c of the CTA, or -1 for a block wholly in the prefix, which is the first jp blocks)
__device__ __forceinline__ void dec_item(int i, int jp, int ncopy, int& j, int& c) {
  if (i < jp) { j = i; c = -1; }
  else { j = jp + (i - jp) / ncopy; c = (i - jp) % ncopy; }
}

// shared: the keys copy c0 + c of prompt b may see, clamped so no row outside the prefix or suffix buffer is ever addressed
__device__ __forceinline__ int dec_shared_lim(const DecParams& p, int b, int c, int plen) {
  return c < p.T ? max(0, min(min(p.len[b * p.T + c], p.max_len), plen + p.s_max)) : 0;
}

// shared: stage the rows of item i.  A prefix block comes from the prefix buffer; a copy's block from the prefix rows below plen and its
// own suffix rows from plen on, only rows below the copy's limit (an item with none still arrives on the stage's barrier).
template <int HD>
__device__ __forceinline__ void dec_issue_shared(uint8_t* sK, uint8_t* sV, uint64_t* full, const DecParams& p, int b, int hk, int c0,
                                                 int plen, int kbeg, int kend, int jp, int ncopy, int i) {
  using C = DecCfg<HD>;
  const int s = i % C::NST;
  int j, c;
  dec_item(i, jp, ncopy, j, c);
  const int k0 = kbeg + j * DEC_BK;
  const int kn = min(DEC_BK, kend - k0);
  const size_t pre = ((size_t)b * p.nkv + hk) * p.p_max;
  uint8_t* dk = sK + s * C::KV_BYTES;
  uint8_t* dv = sV + s * C::KV_BYTES;
  if (c < 0) {
    const uint32_t bytes = (uint32_t)kn * HD * 2;
    mbar_expect_tx(&full[s], 2 * bytes);
    bulk_g2s(dk, p.k + (pre + k0) * HD, bytes, &full[s]);
    bulk_g2s(dv, p.v + (pre + k0) * HD, bytes, &full[s]);
    return;
  }
  const int e = min(k0 + kn, dec_shared_lim(p, b, c0 + c, plen));      // this copy's keys of the block: [k0, e)
  const int np = max(0, min(e, plen) - k0);                            // from the prefix: [k0, k0 + np)
  const int k1 = max(k0, plen);
  const int ns = max(0, e - k1);                                       // from the suffix: [k1, k1 + ns)
  mbar_expect_tx(&full[s], 2u * (uint32_t)(np + ns) * HD * 2);
  if (np > 0) {
    bulk_g2s(dk, p.k + (pre + k0) * HD, (uint32_t)np * HD * 2, &full[s]);
    bulk_g2s(dv, p.v + (pre + k0) * HD, (uint32_t)np * HD * 2, &full[s]);
  }
  if (ns > 0) {
    const size_t suf = (((size_t)b * p.T + c0 + c) * p.nkv + hk) * p.s_max + (k1 - plen);
    bulk_g2s(dk + (size_t)(k1 - k0) * HD * 2, p.ks + suf * HD, (uint32_t)ns * HD * 2, &full[s]);
    bulk_g2s(dv + (size_t)(k1 - k0) * HD * 2, p.vs + suf * HD, (uint32_t)ns * HD * 2, &full[s]);
  }
}

// SINGLE: G query heads of one row per CTA.  CHUNK: G virtual heads v = (row t0 + v / p.g, head v % p.g), the rows of blockIdx.y / nkv's
// row group; virtual heads past row T - 1 have limit 0 and write nothing.  SHARED: as CHUNK with copies for rows (t0 = the CTA's first copy,
// b = the prompt), each virtual head limited by its copy's len, the key range walked as items (dec_item).
template <int HD, int G, int MODE = DEC_SINGLE>
__global__ void __launch_bounds__(DEC_THREADS) attn_decode_kernel(const DecParams p) {
  using C = DecCfg<HD>;
  constexpr int NST = C::NST, LANES = C::LANES, GROUPS = C::GROUPS, PAIRS = C::PAIRS, KSUB = C::KSUB;
  constexpr bool VIRT = MODE != DEC_SINGLE, SHARED = MODE == DEC_SHARED;
  extern __shared__ __align__(128) uint8_t dec_smem[];
  __shared__ __align__(8) uint64_t full[NST];
  __shared__ __align__(16) float s_p[DEC_BK][DEC_MAX_G];       // scores, then probabilities: [key][head]
  __shared__ float s_m[DEC_MAX_G], s_l[DEC_MAX_G], s_alpha[DEC_MAX_G];
  __shared__ __align__(16) float s_red[KSUB][G][HD];
  uint8_t* sK = dec_smem;
  uint8_t* sV = dec_smem + NST * C::KV_BYTES;

  const int split = blockIdx.x, hk = VIRT ? blockIdx.y % p.nkv : blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int len = SHARED ? 0 : min(p.len[b], p.max_len);
  int lim[G];                                           // chunk / shared: key limit of each virtual head
  const int t0 = VIRT ? (int)(blockIdx.y / p.nkv) * p.rows : 0;
  const int plen = SHARED ? max(0, min(p.plen[b], p.p_max)) : 0;
  if constexpr (MODE == DEC_CHUNK) {
    const int base = p.len[b] - p.T;                    // cached rows before this step's T
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int t = t0 + g / p.g;
      lim[g] = t < p.T ? max(0, min(base + t + 1, p.max_len)) : 0;
    }
    len = max(0, min(base + min(t0 + p.rows, p.T), p.max_len));     // the row group's largest limit
  }
  if constexpr (SHARED) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      lim[g] = dec_shared_lim(p, b, t0 + g / p.g, plen);
      len = max(len, lim[g]);
    }
  }
  const int kbeg = split * p.split_blocks * DEC_BK;
  const int kend = min(len, kbeg + p.split_blocks * DEC_BK);
  const int nblk = kend > kbeg ? (kend - kbeg + DEC_BK - 1) / DEC_BK : 0;     // a split at or past len[b] contributes nothing
  // shared: the first jp blocks lie wholly in the prefix (one item each), every later block is one item per copy of the CTA
  const int ncopy = SHARED ? max(1, min(p.rows, p.T - t0)) : 1;
  const int jp = !SHARED || kend <= plen ? nblk : min(nblk, max(0, plen - kbeg) / DEC_BK);
  const int nitem = jp + (nblk - jp) * ncopy;
  const size_t head_row = ((size_t)b * p.nkv + hk) * p.max_len;
  const __nv_bfloat16* kg = p.k + head_row * HD;
  const __nv_bfloat16* vg = p.v + head_row * HD;

  if (tid == 0) {
    for (int s = 0; s < NST; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  if (tid < G) { s_m[tid] = -INFINITY; s_l[tid] = 0.f; }
  __syncthreads();
  if (tid == 0)
    for (int i = 0; i < min(NST, nitem); ++i) {
      if constexpr (SHARED) dec_issue_shared<HD>(sK, sV, full, p, b, hk, t0, plen, kbeg, kend, jp, ncopy, i);
      else dec_issue<HD>(sK, sV, full, kg, vg, kbeg, kend, i);
    }

  // this lane's 8 columns of every query head of the group
  const int li = tid % LANES, grp = tid / LANES;
  float qf[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    uint4 w;
    if constexpr (VIRT) {
      const int t = t0 + g / p.g;
      w = t < p.T ? *reinterpret_cast<const uint4*>(p.q + ((int64_t)b * p.T + t) * p.ld_q + (int64_t)(hk * p.g + g % p.g) * HD + li * 8)
                  : make_uint4(0u, 0u, 0u, 0u);
    } else {
      w = *reinterpret_cast<const uint4*>(p.q + (int64_t)b * p.ld_q + (int64_t)(hk * G + g) * HD + li * 8);
    }
    qf[g][0] = bf16lo(w.x); qf[g][1] = bf16hi(w.x); qf[g][2] = bf16lo(w.y); qf[g][3] = bf16hi(w.y);
    qf[g][4] = bf16lo(w.z); qf[g][5] = bf16hi(w.z); qf[g][6] = bf16lo(w.w); qf[g][7] = bf16hi(w.w);
  }
  const int pair = tid % PAIRS, ks = tid / PAIRS;
  float o[G][2];
#pragma unroll
  for (int g = 0; g < G; ++g) o[g][0] = o[g][1] = 0.f;

  for (int i = 0; i < nitem; ++i) {
    const int s = i % NST;
    int j = i, c = -1;                                   // c >= 0: an item of copy t0 + c only (shared), whose heads alone it updates
    if constexpr (SHARED) dec_item(i, jp, ncopy, j, c);
    const int kb = kbeg + j * DEC_BK;
    const int n = min(DEC_BK, kend - kb);
    mbar_wait_bounded(&full[s], (i / NST) & 1);
    // ---- scores: every lane group runs the same trip count (the shuffles need the whole warp); rows >= n are discarded ----
    const uint8_t* Ks = sK + s * C::KV_BYTES;
#pragma unroll
    for (int r0 = 0; r0 < DEC_BK; r0 += GROUPS) {
      const int t = r0 + grp;
      const uint4 w = *reinterpret_cast<const uint4*>(Ks + (t * HD + li * 8) * 2);
      const float kf[8] = {bf16lo(w.x), bf16hi(w.x), bf16lo(w.y), bf16hi(w.y), bf16lo(w.z), bf16hi(w.z), bf16lo(w.w), bf16hi(w.w)};
      float sc[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float a = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) a = fmaf(qf[g][e], kf[e], a);
        sc[g] = a;
      }
#pragma unroll
      for (int off = LANES / 2; off > 0; off >>= 1)
#pragma unroll
        for (int g = 0; g < G; ++g) sc[g] += __shfl_xor_sync(0xffffffffu, sc[g], off);
      if (li == 0)
#pragma unroll
        for (int g = 0; g < G; ++g) s_p[t][g] = t < n && (!VIRT || kb + t < lim[g]) ? sc[g] * p.scale_log2 : -INFINITY;
    }
    __syncthreads();
    // ---- online softmax, one warp per head (key 0 of the block is always valid, so the block max is finite; in a chunk a virtual head
    //      may have seen no valid key yet: m stays -inf, and exponents are taken against 0 so p = alpha = l = 0 instead of NaN) ----
    for (int g = warp; g < G; g += DEC_THREADS / 32) {
      if (SHARED && c >= 0 && g / p.g != c) continue;   // another copy's head: its rows are not in this stage
      const float a = s_p[lane][g], cc = s_p[lane + 32][g];
      const float m_old = s_m[g];
      const float m_new = fmaxf(m_old, warp_max(fmaxf(a, cc)));
      const float m_ref = VIRT && m_new == -INFINITY ? 0.f : m_new;
      const float pa = ex2f(a - m_ref), pc = ex2f(cc - m_ref);
      s_p[lane][g] = pa;
      s_p[lane + 32][g] = pc;
      const float sum = warp_sum(pa + pc);
      if (lane == 0) {
        const float alpha = ex2f(m_old - m_ref);        // m_old = -inf -> 0
        s_alpha[g] = alpha;
        s_l[g] = fmaf(s_l[g], alpha, sum);
        s_m[g] = m_new;
      }
    }
    __syncthreads();
    // ---- O = alpha * O + P V over the valid rows only ----
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (SHARED && c >= 0 && g / p.g != c) continue;
      o[g][0] *= s_alpha[g]; o[g][1] *= s_alpha[g];
    }
    const uint8_t* Vs = sV + s * C::KV_BYTES;
    for (int t = ks; t < n; t += KSUB) {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(Vs + (t * HD + 2 * pair) * 2);
      const float v0 = bf16lo(w), v1 = bf16hi(w);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        if (VIRT && kb + t >= lim[g]) continue;         // past this row's limit: not visited, as the single-query kernel does not
        if (SHARED && c >= 0 && g / p.g != c) continue;
        const float pg = s_p[t][g];
        o[g][0] = fmaf(pg, v0, o[g][0]);
        o[g][1] = fmaf(pg, v1, o[g][1]);
      }
    }
    __syncthreads();                                     // stage s and s_p are free again
    if (tid == 0 && i + NST < nitem) {
      if constexpr (SHARED) dec_issue_shared<HD>(sK, sV, full, p, b, hk, t0, plen, kbeg, kend, jp, ncopy, i + NST);
      else dec_issue<HD>(sK, sV, full, kg, vg, kbeg, kend, i + NST);
    }
  }

  // ---- reduce the key subsets, write this split's partial ----
#pragma unroll
  for (int g = 0; g < G; ++g) { s_red[ks][g][2 * pair] = o[g][0]; s_red[ks][g][2 * pair + 1] = o[g][1]; }
  __syncthreads();
  for (int i = tid; i < G * HD; i += DEC_THREADS) {
    const int g = i / HD, d = i % HD;
    float a = 0.f;
#pragma unroll
    for (int q = 0; q < KSUB; ++q) a += s_red[q][g][d];
    if constexpr (VIRT) {
      const int t = t0 + g / p.g;
      if (t < p.T) p.ws_o[((((size_t)b * p.T + t) * p.nh + hk * p.g + g % p.g) * p.nsplit + split) * HD + d] = a;
    } else {
      const int h = hk * G + g;
      p.ws_o[(((size_t)b * p.nh + h) * p.nsplit + split) * HD + d] = a;
    }
  }
  if (tid < G) {
    float* ml;
    if constexpr (VIRT) {
      const int t = t0 + tid / p.g;
      if (t >= p.T) return;
      ml = p.ws_ml + ((((size_t)b * p.T + t) * p.nh + hk * p.g + tid % p.g) * p.nsplit + split) * 2;
    } else {
      ml = p.ws_ml + (((size_t)b * p.nh + hk * G + tid) * p.nsplit + split) * 2;
    }
    ml[0] = s_m[tid];
    ml[1] = s_l[tid];
  }
}

// one CTA per (head, batch), one thread per output column: out = sum_i 2^(m_i - M) o_i / sum_i 2^(m_i - M) l_i
template <int HD>
__global__ void __launch_bounds__(HD) attn_decode_merge_kernel(const float* ws_o, const float* ws_ml, int nh, int nsplit,
                                                               __nv_bfloat16* out, int64_t ld_o, float* lse) {
  const int h = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
  const size_t base = ((size_t)b * nh + h) * nsplit;
  const float* ml = ws_ml + base * 2;
  float M = -INFINITY;
  for (int i = 0; i < nsplit; ++i) M = fmaxf(M, ml[2 * i]);
  float L = 0.f, acc = 0.f;
  if (M != -INFINITY) {
    for (int i = 0; i < nsplit; ++i) {
      const float mi = ml[2 * i];
      if (mi == -INFINITY) continue;                   // empty split (at or past len)
      const float w = ex2f(mi - M);
      L = fmaf(ml[2 * i + 1], w, L);
      acc = fmaf(ws_o[(base + i) * HD + d], w, acc);
    }
  }
  out[(int64_t)b * ld_o + (int64_t)h * HD + d] = __float2bfloat16_rn(L > 0.f ? acc / L : 0.f);
  if (lse && d == 0) lse[(size_t)b * nh + h] = L > 0.f ? (M + lg2f(L)) * LN2_F : -INFINITY;
}

// new rows of the fused qkv buffer -> cache: one thread per 16 B of a k or v head row
__global__ void kv_append_kernel(const __nv_bfloat16* qkv, int64_t ld, int n_new, int nh, int nkv, int hd, const int32_t* off,
                                 __nv_bfloat16* kc, __nv_bfloat16* vc, int max_len, int64_t chunks) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= chunks) return;
  const int per = hd / 8;
  int64_t i = c;
  const int d8 = (int)(i % per); i /= per;
  const int j = (int)(i % nkv); i /= nkv;
  const int isv = (int)(i % 2); i /= 2;
  const int64_t row = i;
  const int b = (int)(row / n_new), r = (int)(row % n_new);
  const int pos = off[b] + r;
  if (pos < 0 || pos >= max_len) return;                // the host bounds-checks every append; never write outside the cache
  const __nv_bfloat16* src = qkv + row * ld + (int64_t)(nh + isv * nkv + j) * hd + d8 * 8;
  __nv_bfloat16* dst = (isv ? vc : kc) + (((int64_t)b * nkv + j) * max_len + pos) * hd + d8 * 8;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
}

// rows [lo[b], hi[b]) of sequence b's n_rows rows of the fused qkv buffer -> cache rows off[b] + (r - lo[b]): the padded prefill's real
// rows, packed at the front of each sequence's cache.  One thread per 16 B of a k or v head row; rows outside the range return at once.
__global__ void kv_append_rows_kernel(const __nv_bfloat16* qkv, int64_t ld, int n_rows, int nh, int nkv, int hd, const int32_t* lo,
                                      const int32_t* hi, const int32_t* off, __nv_bfloat16* kc, __nv_bfloat16* vc, int max_len,
                                      int64_t chunks) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= chunks) return;
  const int per = hd / 8;
  int64_t i = c;
  const int d8 = (int)(i % per); i /= per;
  const int j = (int)(i % nkv); i /= nkv;
  const int isv = (int)(i % 2); i /= 2;
  const int64_t row = i;
  const int b = (int)(row / n_rows), r = (int)(row % n_rows);
  const int r0 = lo[b];
  if (r < r0 || r >= hi[b]) return;
  const int pos = off[b] + (r - r0);
  if (pos < 0 || pos >= max_len) return;                // the host bounds-checks every append; never write outside the cache
  const __nv_bfloat16* src = qkv + row * ld + (int64_t)(nh + isv * nkv + j) * hd + d8 * 8;
  __nv_bfloat16* dst = (isv ? vc : kc) + (((int64_t)b * nkv + j) * max_len + pos) * hd + d8 * 8;
  *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
}

constexpr int BEAM_THREADS = 256;
constexpr int BEAM_CHUNK = 512;         // rows per CTA, walked in blocks of R rows
constexpr int BEAM_STAGE = 32768;       // staged bytes per CTA: R = BEAM_STAGE / (n * hd * 2) rows of every beam fit
constexpr int BEAM_MAX_N = 128;         // beams per prompt (R >= 1 at hd 128)

// Beam reorder, in place: new[b*n + j, h, r] = old[b*n + parent[b*n + j], h, r] for r < rows[b], columns [0, hd) of each hp-wide row.
// CTA = (buffer, prompt, KV head) x chunk of BEAM_CHUNK rows.  Thread 0 lists the beams that change (parent != self) and the beams some
// changed beam reads (sources, each staged once); per row block every source tile is loaded to shared memory before any changed beam is
// written, so cycles and many-from-one maps need no second buffer.  A prompt whose map is the identity moves nothing.
__global__ void __launch_bounds__(BEAM_THREADS) kv_beam_reorder_kernel(__nv_bfloat16* const* bufs, int64_t prompts, int n, int nkv,
                                                                      int64_t cap, int hd, int hp, int R, const int32_t* rows,
                                                                      const int32_t* parent) {
  extern __shared__ __align__(16) uint4 stage[];
  __shared__ int par[BEAM_MAX_N], slot[BEAM_MAX_N], src[BEAM_MAX_N], dst[BEAM_MAX_N];
  __shared__ int n_src, n_dst;
  const int64_t t = blockIdx.x;
  const int h = (int)(t % nkv);
  const int64_t b = (t / nkv) % prompts;
  const int64_t buf = t / nkv / prompts;
  const int64_t r_lo = (int64_t)blockIdx.y * BEAM_CHUNK;
  const int64_t r_end = min(min((int64_t)rows[b], cap), r_lo + BEAM_CHUNK);
  if (r_lo >= r_end) return;
  if (threadIdx.x == 0) {
    int ns = 0, nd = 0;
    for (int j = 0; j < n; ++j) {
      par[j] = parent[b * n + j];
      slot[j] = -1;
    }
    for (int j = 0; j < n; ++j) {
      const int p = par[j];
      if (p == j || p < 0 || p >= n) continue;          // the host checks the range; an out-of-range parent leaves its beam alone
      dst[nd++] = j;
      if (slot[p] < 0) {
        slot[p] = ns;
        src[ns++] = p;
      }
    }
    n_src = ns;
    n_dst = nd;
  }
  __syncthreads();
  const int ns = n_src, nd = n_dst;
  if (nd == 0) return;
  const int cpr = hd / 8;                               // 16-byte chunks per row
  __nv_bfloat16* base = bufs[buf];
  const int64_t beam_stride = (int64_t)nkv * cap * hp;
  __nv_bfloat16* head = base + (b * n * nkv + h) * cap * hp;   // beam 0 of prompt b, head h, row 0
  for (int64_t r0 = r_lo; r0 < r_end; r0 += R) {
    const int per = (int)min((int64_t)R, r_end - r0) * cpr;
    for (int i = threadIdx.x; i < ns * per; i += BEAM_THREADS) {
      const int s = i / per, w = i - s * per, r = w / cpr, c = w - r * cpr;
      stage[(s * R + r) * cpr + c] = reinterpret_cast<const uint4*>(head + src[s] * beam_stride + (r0 + r) * hp)[c];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nd * per; i += BEAM_THREADS) {
      const int d = i / per, w = i - d * per, r = w / cpr, c = w - r * cpr;
      const int j = dst[d];
      reinterpret_cast<uint4*>(head + j * beam_stride + (r0 + r) * hp)[c] = stage[(slot[par[j]] * R + r) * cpr + c];
    }
    __syncthreads();
  }
}

// split count and length (in key blocks) from max_len, nkv and the SM count: about two waves of CTAs at B = 1, at least
// DEC_MIN_BLOCKS blocks per split
int decode_splits(int64_t max_len, int nkv, int* split_blocks) {
  const int blocks = (int)((max_len + DEC_BK - 1) / DEC_BK);
  int ns = (2 * lmod_num_sms() + nkv - 1) / nkv;
  ns = max(1, min(ns, (blocks + DEC_MIN_BLOCKS - 1) / DEC_MIN_BLOCKS));
  const int sb = (blocks + ns - 1) / ns;
  *split_blocks = sb;
  return (blocks + sb - 1) / sb;
}

template <int HD, int G>
int launch_decode(const DecParams& p, int64_t batch, cudaStream_t st) {
  constexpr int SMEM = DecCfg<HD>::SMEM;
  static bool attr = false;
  if (!attr) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(attn_decode_kernel<HD, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr = true;
  }
  attn_decode_kernel<HD, G><<<dim3(p.nsplit, p.nkv, (unsigned)batch), DEC_THREADS, SMEM, st>>>(p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

template <int HD>
int launch_decode_g(const DecParams& p, int64_t batch, int G, cudaStream_t st) {
  switch (G) {
    case 1: return launch_decode<HD, 1>(p, batch, st);
    case 2: return launch_decode<HD, 2>(p, batch, st);
    case 3: return launch_decode<HD, 3>(p, batch, st);
    case 4: return launch_decode<HD, 4>(p, batch, st);
    case 5: return launch_decode<HD, 5>(p, batch, st);
    case 6: return launch_decode<HD, 6>(p, batch, st);
    case 7: return launch_decode<HD, 7>(p, batch, st);
    default: return launch_decode<HD, 8>(p, batch, st);
  }
}

// chunk / shared: G = virtual heads per CTA (rows or copies per CTA * query heads per KV head); grid y = KV head + nkv * row group
template <int HD, int G, int MODE>
int launch_decode_virt(const DecParams& p, int64_t batch, cudaStream_t st) {
  constexpr int SMEM = DecCfg<HD>::SMEM;
  static bool attr = false;
  if (!attr) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(attn_decode_kernel<HD, G, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr = true;
  }
  const unsigned groups = (unsigned)((p.T + p.rows - 1) / p.rows);
  attn_decode_kernel<HD, G, MODE><<<dim3(p.nsplit, p.nkv * groups, (unsigned)batch), DEC_THREADS, SMEM, st>>>(p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

template <int HD, int MODE>
int launch_decode_virt_g(const DecParams& p, int64_t batch, int VG, cudaStream_t st) {
  switch (VG) {
    case 1: return launch_decode_virt<HD, 1, MODE>(p, batch, st);
    case 2: return launch_decode_virt<HD, 2, MODE>(p, batch, st);
    case 3: return launch_decode_virt<HD, 3, MODE>(p, batch, st);
    case 4: return launch_decode_virt<HD, 4, MODE>(p, batch, st);
    case 5: return launch_decode_virt<HD, 5, MODE>(p, batch, st);
    case 6: return launch_decode_virt<HD, 6, MODE>(p, batch, st);
    case 7: return launch_decode_virt<HD, 7, MODE>(p, batch, st);
    default: return launch_decode_virt<HD, 8, MODE>(p, batch, st);
  }
}

}  // namespace

extern "C" int lmod_kv_append(const void* qkv, int64_t ld_qkv, int64_t batch, int64_t n_new, int nh, int nkv, int hd,
                              const int32_t* offsets, void* k_cache, void* v_cache, int64_t max_len, void* stream) {
  LMOD_CHECK_ARG(qkv && offsets && k_cache && v_cache && batch > 0 && n_new > 0 && nh > 0 && nkv > 0 && max_len > 0,
                 "lmod_kv_append: bad arguments");
  LMOD_CHECK_ARG(hd % 8 == 0 && ld_qkv % 8 == 0 && ld_qkv >= (int64_t)(nh + 2 * nkv) * hd, "lmod_kv_append: hd / ld_qkv");
  LMOD_CHECK_ARG((uintptr_t)qkv % 16 == 0 && (uintptr_t)k_cache % 16 == 0 && (uintptr_t)v_cache % 16 == 0, "lmod_kv_append: alignment");
  const int64_t chunks = batch * n_new * 2 * nkv * (hd / 8);
  kv_append_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)qkv, ld_qkv, (int)n_new, nh, nkv, hd, offsets, (__nv_bfloat16*)k_cache, (__nv_bfloat16*)v_cache, (int)max_len,
      chunks);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_kv_append_rows(const void* qkv, int64_t ld_qkv, int64_t batch, int64_t n_rows, int nh, int nkv, int hd,
                                   const int32_t* src_lo, const int32_t* src_hi, const int32_t* offsets, void* k_cache, void* v_cache,
                                   int64_t max_len, void* stream) {
  LMOD_CHECK_ARG(qkv && src_lo && src_hi && offsets && k_cache && v_cache && batch > 0 && n_rows > 0 && nh > 0 && nkv > 0 && max_len > 0,
                 "lmod_kv_append_rows: bad arguments");
  LMOD_CHECK_ARG(hd % 8 == 0 && ld_qkv % 8 == 0 && ld_qkv >= (int64_t)(nh + 2 * nkv) * hd, "lmod_kv_append_rows: hd / ld_qkv");
  LMOD_CHECK_ARG((uintptr_t)qkv % 16 == 0 && (uintptr_t)k_cache % 16 == 0 && (uintptr_t)v_cache % 16 == 0,
                 "lmod_kv_append_rows: alignment");
  const int64_t chunks = batch * n_rows * 2 * nkv * (hd / 8);
  kv_append_rows_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)qkv, ld_qkv, (int)n_rows, nh, nkv, hd, src_lo, src_hi, offsets, (__nv_bfloat16*)k_cache,
      (__nv_bfloat16*)v_cache, (int)max_len, chunks);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_kv_beam_reorder(void* const* bufs, int n_bufs, int64_t prompts, int64_t n, int nkv, int64_t cap, int hd, int hp,
                                    const int32_t* rows, const int32_t* parent, void* stream) {
  LMOD_CHECK_ARG(bufs && rows && parent && n_bufs > 0 && prompts > 0 && n >= 1 && nkv > 0 && cap > 0, "lmod_kv_beam_reorder: bad arguments");
  LMOD_CHECK_ARG(n <= BEAM_MAX_N, "lmod_kv_beam_reorder: %lld beams per prompt (at most %d are built)", (long long)n, BEAM_MAX_N);
  LMOD_CHECK_ARG(hd > 0 && hd % 8 == 0 && hp % 8 == 0 && hd <= hp && hp <= 128, "lmod_kv_beam_reorder: hd %d / hp %d", hd, hp);
  const int64_t tiles = (int64_t)n_bufs * prompts * nkv, chunks = (cap + BEAM_CHUNK - 1) / BEAM_CHUNK;
  LMOD_CHECK_ARG(tiles < (1ll << 31) && chunks < 65536, "lmod_kv_beam_reorder: grid too large");
  if (n == 1) return LMOD_OK;                           // a single beam's map is the identity
  const int R = (int)max(1ll, min((long long)BEAM_CHUNK, (long long)(BEAM_STAGE / (n * hd * 2))));
  kv_beam_reorder_kernel<<<dim3((unsigned)tiles, (unsigned)chunks), BEAM_THREADS, (size_t)n * R * hd * 2, (cudaStream_t)stream>>>(
      (__nv_bfloat16* const*)bufs, prompts, (int)n, nkv, cap, hd, hp, R, rows, parent);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int64_t lmod_attn_decode_ws_elems(int64_t batch, int nh, int nkv, int hd, int64_t max_len) {
  if (batch <= 0 || nh <= 0 || nkv <= 0 || max_len <= 0) return 0;
  int sb;
  const int ns = decode_splits(max_len, nkv, &sb);
  return batch * nh * (int64_t)ns * (hd + 2);
}

extern "C" int lmod_attn_decode(const void* q, int64_t ld_q, const void* k_cache, const void* v_cache, const int32_t* len,
                                int64_t batch, int nh, int nkv, int hd, int64_t max_len, float softmax_scale, void* out, int64_t ld_o,
                                float* lse, float* ws, int64_t ws_elems, void* stream) {
  LMOD_CHECK_ARG(q && k_cache && v_cache && len && out && ws && batch > 0 && nh > 0 && nkv > 0 && nh % nkv == 0 && max_len > 0 &&
                 max_len < (1 << 30), "lmod_attn_decode: bad arguments");
  LMOD_CHECK_ARG(hd == 64 || hd == 128, "lmod_attn_decode: head_dim %d not built (64 and 128 are)", hd);
  LMOD_CHECK_ARG(nh / nkv <= DEC_MAX_G, "lmod_attn_decode: %d query heads per KV head (at most %d are built)", nh / nkv, DEC_MAX_G);
  LMOD_CHECK_ARG(ld_q % 8 == 0 && (uintptr_t)q % 16 == 0 && (uintptr_t)k_cache % 16 == 0 && (uintptr_t)v_cache % 16 == 0,
                 "lmod_attn_decode: alignment");
  LMOD_CHECK_ARG(ws_elems >= lmod_attn_decode_ws_elems(batch, nh, nkv, hd, max_len), "lmod_attn_decode: workspace too small");
  DecParams p;
  p.q = (const __nv_bfloat16*)q; p.ld_q = ld_q;
  p.k = (const __nv_bfloat16*)k_cache; p.v = (const __nv_bfloat16*)v_cache; p.len = len;
  p.nh = nh; p.nkv = nkv; p.max_len = (int)max_len;
  p.nsplit = decode_splits(max_len, nkv, &p.split_blocks);
  p.ws_o = ws;
  p.ws_ml = ws + batch * nh * (int64_t)p.nsplit * hd;
  p.scale_log2 = softmax_scale * LOG2E_F;
  cudaStream_t st = (cudaStream_t)stream;
  const int G = nh / nkv;
  int rc = hd == 128 ? launch_decode_g<128>(p, batch, G, st) : launch_decode_g<64>(p, batch, G, st);
  if (rc) return rc;
  const dim3 grid(nh, (unsigned)batch);
  if (hd == 128) attn_decode_merge_kernel<128><<<grid, 128, 0, st>>>(p.ws_o, p.ws_ml, nh, p.nsplit, (__nv_bfloat16*)out, ld_o, lse);
  else attn_decode_merge_kernel<64><<<grid, 64, 0, st>>>(p.ws_o, p.ws_ml, nh, p.nsplit, (__nv_bfloat16*)out, ld_o, lse);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int64_t lmod_attn_decode_chunk_ws_elems(int64_t batch, int64_t T, int nh, int nkv, int hd, int64_t max_len) {
  if (T <= 0) return 0;
  return lmod_attn_decode_ws_elems(batch * T, nh, nkv, hd, max_len);
}

extern "C" int lmod_attn_decode_chunk(const void* q, int64_t ld_q, const void* k_cache, const void* v_cache, const int32_t* len,
                                      int64_t batch, int64_t T, int nh, int nkv, int hd, int64_t max_len, float softmax_scale, void* out,
                                      int64_t ld_o, float* lse, float* ws, int64_t ws_elems, void* stream) {
  LMOD_CHECK_ARG(q && k_cache && v_cache && len && out && ws && batch > 0 && T > 0 && T <= 4096 && nh > 0 && nkv > 0 && nh % nkv == 0 &&
                 max_len > 0 && max_len < (1 << 30), "lmod_attn_decode_chunk: bad arguments");
  LMOD_CHECK_ARG(hd == 64 || hd == 128, "lmod_attn_decode_chunk: head_dim %d not built (64 and 128 are)", hd);
  LMOD_CHECK_ARG(nh / nkv <= DEC_MAX_G, "lmod_attn_decode_chunk: %d query heads per KV head (at most %d are built)", nh / nkv, DEC_MAX_G);
  LMOD_CHECK_ARG(ld_q % 8 == 0 && (uintptr_t)q % 16 == 0 && (uintptr_t)k_cache % 16 == 0 && (uintptr_t)v_cache % 16 == 0,
                 "lmod_attn_decode_chunk: alignment");
  LMOD_CHECK_ARG(ws_elems >= lmod_attn_decode_chunk_ws_elems(batch, T, nh, nkv, hd, max_len), "lmod_attn_decode_chunk: workspace too small");
  DecParams p;
  p.q = (const __nv_bfloat16*)q; p.ld_q = ld_q;
  p.k = (const __nv_bfloat16*)k_cache; p.v = (const __nv_bfloat16*)v_cache; p.len = len;
  p.nh = nh; p.nkv = nkv; p.max_len = (int)max_len;
  p.nsplit = decode_splits(max_len, nkv, &p.split_blocks);
  p.ws_o = ws;
  p.ws_ml = ws + batch * T * nh * (int64_t)p.nsplit * hd;
  p.scale_log2 = softmax_scale * LOG2E_F;
  p.T = (int)T;
  p.g = nh / nkv;
  p.rows = (int)std::min<int64_t>(T, DEC_MAX_G / p.g);
  cudaStream_t st = (cudaStream_t)stream;
  const int VG = p.rows * p.g;
  int rc = hd == 128 ? launch_decode_virt_g<128, DEC_CHUNK>(p, batch, VG, st) : launch_decode_virt_g<64, DEC_CHUNK>(p, batch, VG, st);
  if (rc) return rc;
  // the merge is lmod_attn_decode's, over batch * T rows
  const dim3 grid(nh, (unsigned)(batch * T));
  if (hd == 128) attn_decode_merge_kernel<128><<<grid, 128, 0, st>>>(p.ws_o, p.ws_ml, nh, p.nsplit, (__nv_bfloat16*)out, ld_o, lse);
  else attn_decode_merge_kernel<64><<<grid, 64, 0, st>>>(p.ws_o, p.ws_ml, nh, p.nsplit, (__nv_bfloat16*)out, ld_o, lse);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int64_t lmod_attn_decode_shared_ws_elems(int64_t batch, int64_t n, int nh, int nkv, int hd, int64_t max_len) {
  if (n <= 0) return 0;
  return lmod_attn_decode_ws_elems(batch * n, nh, nkv, hd, max_len);
}

extern "C" int lmod_attn_decode_shared(const void* q, int64_t ld_q, const void* k_prefix, const void* v_prefix, const int32_t* prefix_len,
                                       int64_t p_max, const void* k_suffix, const void* v_suffix, int64_t s_max, const int32_t* len,
                                       int64_t batch, int64_t n, int nh, int nkv, int hd, int64_t max_len, float softmax_scale, void* out,
                                       int64_t ld_o, float* lse, float* ws, int64_t ws_elems, void* stream) {
  LMOD_CHECK_ARG(q && k_prefix && v_prefix && prefix_len && k_suffix && v_suffix && len && out && ws && batch > 0 && n > 0 && n <= 4096 &&
                 nh > 0 && nkv > 0 && nh % nkv == 0 && p_max > 0 && s_max > 0 && max_len > 0 && max_len < (1 << 30) &&
                 p_max < (1 << 30) && s_max < (1 << 30), "lmod_attn_decode_shared: bad arguments");
  LMOD_CHECK_ARG(hd == 64 || hd == 128, "lmod_attn_decode_shared: head_dim %d not built (64 and 128 are)", hd);
  LMOD_CHECK_ARG(nh / nkv <= DEC_MAX_G, "lmod_attn_decode_shared: %d query heads per KV head (at most %d are built)", nh / nkv, DEC_MAX_G);
  LMOD_CHECK_ARG(ld_q % 8 == 0 && (uintptr_t)q % 16 == 0 && (uintptr_t)k_prefix % 16 == 0 && (uintptr_t)v_prefix % 16 == 0 &&
                 (uintptr_t)k_suffix % 16 == 0 && (uintptr_t)v_suffix % 16 == 0, "lmod_attn_decode_shared: alignment");
  LMOD_CHECK_ARG(ws_elems >= lmod_attn_decode_shared_ws_elems(batch, n, nh, nkv, hd, max_len), "lmod_attn_decode_shared: workspace too small");
  DecParams p;
  p.q = (const __nv_bfloat16*)q; p.ld_q = ld_q;
  p.k = (const __nv_bfloat16*)k_prefix; p.v = (const __nv_bfloat16*)v_prefix; p.len = len;
  p.ks = (const __nv_bfloat16*)k_suffix; p.vs = (const __nv_bfloat16*)v_suffix; p.plen = prefix_len;
  p.p_max = (int)p_max; p.s_max = (int)s_max;
  p.nh = nh; p.nkv = nkv; p.max_len = (int)max_len;
  p.nsplit = decode_splits(max_len, nkv, &p.split_blocks);      // lmod_attn_decode's splits at the expanded cache's max_len
  p.ws_o = ws;
  p.ws_ml = ws + batch * n * nh * (int64_t)p.nsplit * hd;
  p.scale_log2 = softmax_scale * LOG2E_F;
  p.T = (int)n;
  p.g = nh / nkv;
  p.rows = (int)std::min<int64_t>(n, DEC_MAX_G / p.g);
  cudaStream_t st = (cudaStream_t)stream;
  const int VG = p.rows * p.g;
  int rc = hd == 128 ? launch_decode_virt_g<128, DEC_SHARED>(p, batch, VG, st) : launch_decode_virt_g<64, DEC_SHARED>(p, batch, VG, st);
  if (rc) return rc;
  // the merge is lmod_attn_decode's, over batch * n rows
  const dim3 grid(nh, (unsigned)(batch * n));
  if (hd == 128) attn_decode_merge_kernel<128><<<grid, 128, 0, st>>>(p.ws_o, p.ws_ml, nh, p.nsplit, (__nv_bfloat16*)out, ld_o, lse);
  else attn_decode_merge_kernel<64><<<grid, 64, 0, st>>>(p.ws_o, p.ws_ml, nh, p.nsplit, (__nv_bfloat16*)out, ld_o, lse);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
