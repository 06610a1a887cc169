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
#include "sm90.cuh"

namespace {

constexpr int DEC_THREADS = 128;
constexpr int DEC_BK = 64;            // keys per ring stage
constexpr int DEC_MIN_BLOCKS = 4;     // a split covers at least this many key blocks
constexpr int DEC_MAX_G = 8;          // query heads per KV head

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

template <int HD, int G>
__global__ void __launch_bounds__(DEC_THREADS) attn_decode_kernel(const DecParams p) {
  using C = DecCfg<HD>;
  constexpr int NST = C::NST, LANES = C::LANES, GROUPS = C::GROUPS, PAIRS = C::PAIRS, KSUB = C::KSUB;
  extern __shared__ __align__(128) uint8_t dec_smem[];
  __shared__ __align__(8) uint64_t full[NST];
  __shared__ __align__(16) float s_p[DEC_BK][DEC_MAX_G];       // scores, then probabilities: [key][head]
  __shared__ float s_m[DEC_MAX_G], s_l[DEC_MAX_G], s_alpha[DEC_MAX_G];
  __shared__ __align__(16) float s_red[KSUB][G][HD];
  uint8_t* sK = dec_smem;
  uint8_t* sV = dec_smem + NST * C::KV_BYTES;

  const int split = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int len = min(p.len[b], p.max_len);
  const int kbeg = split * p.split_blocks * DEC_BK;
  const int kend = min(len, kbeg + p.split_blocks * DEC_BK);
  const int nblk = kend > kbeg ? (kend - kbeg + DEC_BK - 1) / DEC_BK : 0;     // a split at or past len[b] contributes nothing
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
    for (int j = 0; j < min(NST, nblk); ++j) dec_issue<HD>(sK, sV, full, kg, vg, kbeg, kend, j);

  // this lane's 8 columns of every query head of the group
  const int li = tid % LANES, grp = tid / LANES;
  float qf[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4 w = *reinterpret_cast<const uint4*>(p.q + (int64_t)b * p.ld_q + (int64_t)(hk * G + g) * HD + li * 8);
    qf[g][0] = bf16lo(w.x); qf[g][1] = bf16hi(w.x); qf[g][2] = bf16lo(w.y); qf[g][3] = bf16hi(w.y);
    qf[g][4] = bf16lo(w.z); qf[g][5] = bf16hi(w.z); qf[g][6] = bf16lo(w.w); qf[g][7] = bf16hi(w.w);
  }
  const int pair = tid % PAIRS, ks = tid / PAIRS;
  float o[G][2];
#pragma unroll
  for (int g = 0; g < G; ++g) o[g][0] = o[g][1] = 0.f;

  for (int j = 0; j < nblk; ++j) {
    const int s = j % NST;
    const int n = min(DEC_BK, kend - (kbeg + j * DEC_BK));
    mbar_wait_bounded(&full[s], (j / NST) & 1);
    // ---- scores: every lane group runs the same trip count (the shuffles need the whole warp); rows >= n are discarded ----
    const uint8_t* Ks = sK + s * C::KV_BYTES;
#pragma unroll
    for (int t0 = 0; t0 < DEC_BK; t0 += GROUPS) {
      const int t = t0 + grp;
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
        for (int g = 0; g < G; ++g) s_p[t][g] = t < n ? sc[g] * p.scale_log2 : -INFINITY;
    }
    __syncthreads();
    // ---- online softmax, one warp per head (key 0 of the block is always valid, so the block max is finite) ----
    for (int g = warp; g < G; g += DEC_THREADS / 32) {
      const float a = s_p[lane][g], c = s_p[lane + 32][g];
      const float m_old = s_m[g];
      const float m_new = fmaxf(m_old, warp_max(fmaxf(a, c)));
      const float pa = ex2f(a - m_new), pc = ex2f(c - m_new);
      s_p[lane][g] = pa;
      s_p[lane + 32][g] = pc;
      const float sum = warp_sum(pa + pc);
      if (lane == 0) {
        const float alpha = ex2f(m_old - m_new);        // m_old = -inf -> 0
        s_alpha[g] = alpha;
        s_l[g] = fmaf(s_l[g], alpha, sum);
        s_m[g] = m_new;
      }
    }
    __syncthreads();
    // ---- O = alpha * O + P V over the valid rows only ----
#pragma unroll
    for (int g = 0; g < G; ++g) { o[g][0] *= s_alpha[g]; o[g][1] *= s_alpha[g]; }
    const uint8_t* Vs = sV + s * C::KV_BYTES;
    for (int t = ks; t < n; t += KSUB) {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(Vs + (t * HD + 2 * pair) * 2);
      const float v0 = bf16lo(w), v1 = bf16hi(w);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float pg = s_p[t][g];
        o[g][0] = fmaf(pg, v0, o[g][0]);
        o[g][1] = fmaf(pg, v1, o[g][1]);
      }
    }
    __syncthreads();                                     // stage s and s_p are free again
    if (tid == 0 && j + NST < nblk) dec_issue<HD>(sK, sV, full, kg, vg, kbeg, kend, j + NST);
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
    const int h = hk * G + g;
    p.ws_o[(((size_t)b * p.nh + h) * p.nsplit + split) * HD + d] = a;
  }
  if (tid < G) {
    float* ml = p.ws_ml + (((size_t)b * p.nh + hk * G + tid) * p.nsplit + split) * 2;
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
