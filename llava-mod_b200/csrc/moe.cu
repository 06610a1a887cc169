// moe.cu -- DeepSpeed-0.9.5 top-2 MoE routing on H100: gate (GEMV + softmax + top-2) and seat+scatter (stable capacity positions by
// warp ballots, token copy) as two ordinary launches of small CTAs; weighted gather/combine; and their backward kernels.
// Top-1 (top1gating with random token selection) reuses the gate and seat+scatter kernels through a template flag, with a selection
// launch between them that finds, per expert, which routed tokens keep a seat (the C largest uniforms).
//
// Replaces (third-party, call site llavamod/model/language_model/llava_qwen1_5_moe.py:536-546)
// deepspeed.moe.sharded_moe.TopKGate / top2gating / MOELayer dispatch+combine einsums
// (SURVEY.md Appendix A): ~40 small ATen kernels, a D2H sync (exp_counts.to('cpu')) and two one-hot
// einsums per MoE layer become: route_scatter (2 launches) + expert GEMMs + gather_combine (1 launch).
//
// Semantics kept bit-exact for the integer record (idx1, idx2, slot, kept) given the same fp32 logits
// and the same Gumbel noise tensor: first choices are seated before any second choice, positions are
// a STABLE prefix count over the flattened [B*T] token order (warp-ballot + popc, no atomics races),
// capacity C = ceil(S/E * cf * 2), drops by position >= C.
#include <float.h>
#include "common.cuh"

namespace {

constexpr int RT_THREADS = 256;
constexpr int RT_WARPS = RT_THREADS / 32;
constexpr int MAXE = 8;
constexpr int TOK_PER_WARP = 2;                       // a warp gates two tokens at a time (both rows in flight, one pass over wg)
constexpr int TILE_MIN = RT_WARPS * TOK_PER_WARP;     // 16 tokens per CTA
constexpr int MAX_TILES = 1024;

struct RouteParams {
  const __nv_bfloat16* x;
  const float* wg;
  const float* noise;
  int S, H, E;
  int capacity;
  int layout;            // 0: compact rows ; 1: offsets[e] = e*capacity (capacity-padded slabs) ; 2: compact, groups aligned to 128 rows
  int tpb, ntiles;       // tokens per CTA (multiple of 16), number of CTAs
  float* logits; float* gates; int32_t* idx; int32_t* row; float* w;
  int32_t* offsets; float* meta; __nv_bfloat16* xp;
  int32_t* tile_cnt;     // [ntiles][2*MAXE]: first-choice counts per expert, then second-choice counts (top-1: kept counts)
  float* tile_gsum;      // [ntiles][MAXE]: sum of gates per expert over the tile's tokens (token order)
  int32_t* sel;          // top-1 only, [2*MAXE]: per expert the threshold key's bits, then the last token index kept at the threshold
};

// ---- kernel 1 of 2: gate.  fp32 GEMV against wg (staged in shared memory), softmax, top-1, Gumbel top-2; per-tile expert counts ----
// An ordinary launch of ceil(S/16) small CTAs (no cooperative launch, no grid barrier): it shares the machine with whatever else is
// running (the frozen teacher's GEMMs on the side stream).  K = 1: no second choice (idx[:,1] = -1, second-choice counts 0).
template <int K>
__global__ void __launch_bounds__(RT_THREADS) moe_gate_kernel(const RouteParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  float* s_wg = reinterpret_cast<float*>(smem);                           // [E,H] fp32
  float* s_gates = s_wg + (size_t)p.E * p.H;                              // [tpb][MAXE]
  __shared__ int s_cnt[2 * MAXE];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int E = p.E, H = p.H, hv = H >> 3;
  const int b0 = min(p.S, (int)blockIdx.x * p.tpb), b1 = min(p.S, b0 + p.tpb);

  for (int i = tid; i < E * H / 4; i += RT_THREADS)
    reinterpret_cast<float4*>(s_wg)[i] = __ldg(reinterpret_cast<const float4*>(p.wg) + i);
  if (tid < 2 * MAXE) s_cnt[tid] = 0;
  __syncthreads();

  for (int t0 = b0 + warp * TOK_PER_WARP; t0 < b1; t0 += RT_WARPS * TOK_PER_WARP) {
    const bool has1 = t0 + 1 < b1;
    const uint4* xr0 = reinterpret_cast<const uint4*>(p.x + (size_t)t0 * H);
    const uint4* xr1 = reinterpret_cast<const uint4*>(p.x + (size_t)(has1 ? t0 + 1 : t0) * H);
    float acc0[MAXE], acc1[MAXE];
#pragma unroll
    for (int e = 0; e < MAXE; ++e) { acc0[e] = 0.f; acc1[e] = 0.f; }
    for (int v = lane; v < hv; v += 32) {
      const uint4 u0 = ldg_nc_v4(xr0 + v), u1 = ldg_nc_v4(xr1 + v);
      const float xf[8] = {bf16lo(u0.x), bf16hi(u0.x), bf16lo(u0.y), bf16hi(u0.y), bf16lo(u0.z), bf16hi(u0.z), bf16lo(u0.w), bf16hi(u0.w)};
      const float yf[8] = {bf16lo(u1.x), bf16hi(u1.x), bf16lo(u1.y), bf16hi(u1.y), bf16lo(u1.z), bf16hi(u1.z), bf16lo(u1.w), bf16hi(u1.w)};
#pragma unroll
      for (int e = 0; e < MAXE; ++e) {
        if (e < E) {
          const float4 w0 = *reinterpret_cast<const float4*>(s_wg + (size_t)e * H + v * 8);
          const float4 w1 = *reinterpret_cast<const float4*>(s_wg + (size_t)e * H + v * 8 + 4);
          acc0[e] = fmaf(xf[0], w0.x, acc0[e]); acc0[e] = fmaf(xf[1], w0.y, acc0[e]);
          acc0[e] = fmaf(xf[2], w0.z, acc0[e]); acc0[e] = fmaf(xf[3], w0.w, acc0[e]);
          acc0[e] = fmaf(xf[4], w1.x, acc0[e]); acc0[e] = fmaf(xf[5], w1.y, acc0[e]);
          acc0[e] = fmaf(xf[6], w1.z, acc0[e]); acc0[e] = fmaf(xf[7], w1.w, acc0[e]);
          acc1[e] = fmaf(yf[0], w0.x, acc1[e]); acc1[e] = fmaf(yf[1], w0.y, acc1[e]);
          acc1[e] = fmaf(yf[2], w0.z, acc1[e]); acc1[e] = fmaf(yf[3], w0.w, acc1[e]);
          acc1[e] = fmaf(yf[4], w1.x, acc1[e]); acc1[e] = fmaf(yf[5], w1.y, acc1[e]);
          acc1[e] = fmaf(yf[6], w1.z, acc1[e]); acc1[e] = fmaf(yf[7], w1.w, acc1[e]);
        }
      }
    }
#pragma unroll
    for (int e = 0; e < MAXE; ++e) { acc0[e] = warp_sum(acc0[e]); acc1[e] = warp_sum(acc1[e]); }
    if (lane == 1) {
#pragma unroll
      for (int e = 0; e < MAXE; ++e) acc0[e] = acc1[e];
    }
    if (lane == 0 || (lane == 1 && has1)) {          // lane 0 finishes token t0, lane 1 token t0+1
      const int tok = t0 + lane;
      float mx = -INFINITY;
#pragma unroll
      for (int e = 0; e < MAXE; ++e) if (e < E) mx = fmaxf(mx, acc0[e]);
      float ex[MAXE], g[MAXE], den = 0.f;
#pragma unroll
      for (int e = 0; e < MAXE; ++e) { ex[e] = (e < E) ? expf(acc0[e] - mx) : 0.f; den += ex[e]; }
      // top2gating takes argmax(softmax(logits)): the first choice is the first maximal GATE.  Logits closer than exp can resolve
      // (about 2^-25 apart) give equal gates, and then the lower expert wins even if its logit is the smaller one.
      int i1 = 0;
      float gmx = -1.f;
#pragma unroll
      for (int e = 0; e < MAXE; ++e) {
        g[e] = ex[e] / den;
        if (e < E && g[e] > gmx) { gmx = g[e]; i1 = e; }
      }
      int i2 = -1;
      if (K == 2) {
        float best = -INFINITY;
        i2 = (i1 == 0) ? 1 : 0;
#pragma unroll
        for (int e = 0; e < MAXE; ++e) {
          if (e < E && e != i1) {
            const float v = acc0[e] + p.noise[(size_t)tok * E + e];
            if (v > best) { best = v; i2 = e; }
          }
        }
      }
#pragma unroll
      for (int e = 0; e < MAXE; ++e) {
        if (e < E) { p.logits[(size_t)tok * E + e] = acc0[e]; p.gates[(size_t)tok * E + e] = g[e]; }
        s_gates[(tok - b0) * MAXE + e] = (e < E) ? g[e] : 0.f;
      }
      p.idx[2 * tok] = i1; p.idx[2 * tok + 1] = i2;
      atomicAdd(&s_cnt[i1], 1);
      if (K == 2) atomicAdd(&s_cnt[MAXE + i2], 1);
    }
  }
  __syncthreads();
  if (tid < 2 * MAXE) p.tile_cnt[(size_t)blockIdx.x * 2 * MAXE + tid] = s_cnt[tid];
  if (tid >= 32 && tid < 32 + MAXE) {                 // per-expert gate mass of the tile, summed in token order (deterministic l_aux)
    const int e = tid - 32;
    float a = 0.f;
    for (int t = 0; t < b1 - b0; ++t) a += s_gates[t * MAXE + e];
    p.tile_gsum[(size_t)blockIdx.x * MAXE + e] = a;
  }
}

// ---- top-1 only, between the gate and seat+scatter: random token selection.  One CTA per expert.  top1gating keeps, per expert, the
// routed tokens with the C largest uniforms u[s, idx1[s]] (topk over mask1 * u along the tokens).  A uniform in [0, 1) is a non-negative
// float, so its bit pattern orders like its value: an MSB-first radix select over the 32 key bits (four 8-bit digits) finds the C-th
// largest key T.  Keys above T are kept; among keys equal to T the lowest token indices are kept, up to the count still missing
// (torch.topk leaves that order unspecified; this is the build's rule).  An expert with n_e <= C keeps every routed token (T = 0, every
// index).  Writes sel = {T bits, last kept index at T} and each tile's kept count into tile_cnt[tile][MAXE + e]. ----
constexpr int SEL_THREADS = 1024;
constexpr int SEL_WARPS = SEL_THREADS / 32;
__global__ void __launch_bounds__(SEL_THREADS) moe_top1_select_kernel(const RouteParams p) {
  __shared__ int s_hist[256];
  __shared__ int s_wt[SEL_WARPS];
  __shared__ int s_n, s_need, s_lim;
  __shared__ unsigned s_prefix;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int e = blockIdx.x, E = p.E, S = p.S;
  if (tid == 0) { s_n = 0; s_lim = S - 1; s_prefix = 0u; s_need = 0; }
  __syncthreads();
  {
    int n = 0;
    for (int t = tid; t < p.ntiles; t += SEL_THREADS) n += __ldg(p.tile_cnt + (size_t)t * 2 * MAXE + e);
    n = warp_sum(n);
    if (lane == 0) atomicAdd(&s_n, n);
  }
  __syncthreads();
  if (s_n > p.capacity) {                         // block-uniform
    unsigned mask = 0u;
    if (tid == 0) s_need = p.capacity;            // rank of the threshold from the top, 1-based
    for (int shift = 24; shift >= 0; shift -= 8) {
      if (tid < 256) s_hist[tid] = 0;
      __syncthreads();
      const unsigned prefix = s_prefix;
      for (int t = tid; t < S; t += SEL_THREADS) {
        if (__ldg(p.idx + 2 * t) != e) continue;
        const unsigned key = __float_as_uint(__ldg(p.noise + (size_t)t * E + e));
        if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int above = 0, d = 255;
        for (; d > 0; --d) {
          if (above + s_hist[d] >= s_need) break;
          above += s_hist[d];
        }
        s_need -= above;
        s_prefix = prefix | ((unsigned)d << shift);
      }
      mask |= 255u << shift;
      __syncthreads();
    }
    // the s_need-th token (in token order) of this expert whose key equals the threshold is the last one kept at the threshold
    const unsigned thr = s_prefix;
    const int need = s_need;
    const unsigned lt = (1u << lane) - 1u;
    int run = 0;
    for (int base = 0; base < S; base += SEL_THREADS) {
      const int t = base + tid;
      const bool tie = t < S && __ldg(p.idx + 2 * t) == e && __float_as_uint(__ldg(p.noise + (size_t)t * E + e)) == thr;
      const unsigned b = __ballot_sync(0xffffffffu, tie);
      if (lane == 0) s_wt[warp] = __popc(b);
      __syncthreads();
      int pre = run, tot = run;
      for (int w = 0; w < SEL_WARPS; ++w) { const int c = s_wt[w]; tot += c; if (w < warp) pre += c; }
      if (tie && pre + __popc(b & lt) + 1 == need) s_lim = t;
      run = tot;
      __syncthreads();
      if (run >= need) break;                     // block-uniform
    }
  }
  __syncthreads();
  const unsigned thr = s_prefix;
  const int lim = s_lim;
  if (tid == 0) { p.sel[e] = (int)thr; p.sel[MAXE + e] = lim; }
  // kept tokens per tile, for the seat kernel's token-order prefix
  for (int t = warp; t < p.ntiles; t += SEL_WARPS) {
    const int b0 = t * p.tpb, b1 = min(S, b0 + p.tpb);
    int c = 0;
    for (int s = b0 + lane; s < b1; s += 32) {
      if (__ldg(p.idx + 2 * s) != e) continue;
      const unsigned key = __float_as_uint(__ldg(p.noise + (size_t)s * E + e));
      c += (key > thr || (key == thr && s <= lim)) ? 1 : 0;
    }
    c = warp_sum(c);
    if (lane == 0) p.tile_cnt[(size_t)t * 2 * MAXE + MAXE + e] = c;
  }
}

// ---- kernel 2 of 2: seat + scatter.  Every CTA rebuilds the global per-expert totals and its own exclusive prefix from the tile
// counts (a few KB, L2 resident), seats its tokens in token order with warp ballots + popc (all first choices before any second
// choice, drop at position >= capacity), renormalises the two gate weights, and copies its token rows to their expert rows.
// K = 1: the tokens the selection kept are seated in token order from the per-tile kept counts; w[:,0] is the raw gate of a kept token
// (top1gating does not renormalise), row[:,1] = -1 and w[:,1] = 0. ----
template <int K>
__global__ void __launch_bounds__(RT_THREADS) moe_seat_scatter_kernel(const RouteParams p) {
  __shared__ int s_tot[2 * MAXE], s_pre[2 * MAXE], s_off[MAXE + 1], s_used[MAXE];
  __shared__ int s_row[2 * 32 * 64];                  // rows of this CTA's tokens (tpb <= 1024... see launch: tpb*2 <= 4096)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int E = p.E, H = p.H, hv = H >> 3;
  const int tile = blockIdx.x;
  const int b0 = min(p.S, tile * p.tpb), b1 = min(p.S, b0 + p.tpb);
  if (tid < 2 * MAXE) { s_tot[tid] = 0; s_pre[tid] = 0; }
  __syncthreads();
  {
    // lanes 0..15 / 16..31 read the 16 counters of two consecutive tiles per step
    const int c = lane & 15;
    int tot = 0, pre = 0;
    for (int t = 2 * warp + (lane >> 4); t < p.ntiles; t += 2 * RT_WARPS) {
      const int v = __ldg(p.tile_cnt + (size_t)t * 2 * MAXE + c);
      tot += v;
      if (t < tile) pre += v;
    }
    tot += __shfl_xor_sync(0xffffffffu, tot, 16);
    pre += __shfl_xor_sync(0xffffffffu, pre, 16);
    if (lane < 16) { atomicAdd(&s_tot[c], tot); atomicAdd(&s_pre[c], pre); }
  }
  __syncthreads();
  if (tid == 0) {
    int o = 0, used = 0;
    for (int e = 0; e < E; ++e) {
      s_off[e] = (p.layout == 1) ? e * p.capacity : o;
      const int rows_e = (K == 2) ? min(s_tot[e] + s_tot[MAXE + e], p.capacity) : s_tot[MAXE + e];    // top-1: kept = min(n_e, C)
      s_used[e] = rows_e;
      used += rows_e;
      o += (p.layout == 2) ? ((rows_e + 127) & ~127) : rows_e;
    }
    s_off[E] = (p.layout == 1) ? E * p.capacity : o;
    if (tile == 0) {
      for (int e = 0; e <= E; ++e) p.offsets[e] = s_off[e];
      p.meta[1] = (float)p.capacity; p.meta[2] = (float)used; p.meta[3] = (float)s_off[E];
      for (int e = 0; e < E; ++e) p.meta[4 + e] = (float)s_tot[e];
    }
  }
  __syncthreads();
  // l_aux = E * sum_e mean_s(gates[:,e]) * mean_s(mask1[:,e])   (before capacity drops); tile sums added in a fixed order
  if (tile == 0 && warp < E) {
    float a = 0.f;
    for (int t = lane; t < p.ntiles; t += 32) a += __ldg(p.tile_gsum + (size_t)t * MAXE + warp);
    a = warp_sum(a);
    if (lane == 0) s_row[warp] = __float_as_int((a / (float)p.S) * ((float)s_tot[warp] / (float)p.S));
  }
  __syncthreads();
  if (tile == 0 && tid == 0) {
    float laux = 0.f;
    for (int e = 0; e < E; ++e) laux += __int_as_float(s_row[e]);
    p.meta[0] = laux * (float)E;
  }
  __syncthreads();
  // warp 0 seats this CTA's tokens in order (32 at a time, ballot + popc prefix)
  if (K == 1 && warp == 0) {
    int c[MAXE];
    unsigned thr[MAXE];
    int lim[MAXE];
#pragma unroll
    for (int e = 0; e < MAXE; ++e) {
      c[e] = s_pre[MAXE + e];
      thr[e] = (e < E) ? (unsigned)__ldg(p.sel + e) : 0u;
      lim[e] = (e < E) ? __ldg(p.sel + MAXE + e) : 0;
    }
    const unsigned lt = (1u << lane) - 1u;
    for (int base = b0; base < b1; base += 32) {
      const int tok = base + lane;
      const bool valid = tok < b1;
      int e1 = -1;
      bool kept = false;
      if (valid) {
        e1 = __ldg(p.idx + 2 * tok);
        unsigned t_e = 0u; int l_e = 0;
#pragma unroll
        for (int e = 0; e < MAXE; ++e) if (e == e1) { t_e = thr[e]; l_e = lim[e]; }
        const unsigned key = __float_as_uint(__ldg(p.noise + (size_t)tok * E + e1));
        kept = key > t_e || (key == t_e && tok <= l_e);
      }
      int loc = 0;
#pragma unroll
      for (int e = 0; e < MAXE; ++e) {
        if (e < E) {
          const unsigned a = __ballot_sync(0xffffffffu, kept && e1 == e);
          if (kept && e1 == e) loc = c[e] + __popc(a & lt);
          c[e] += __popc(a);
        }
      }
      if (valid) {
        const int r1 = kept ? s_off[e1] + loc : -1;
        p.row[2 * tok] = r1; p.row[2 * tok + 1] = -1;
        p.w[2 * tok] = kept ? __ldg(p.gates + (size_t)tok * E + e1) : 0.f; p.w[2 * tok + 1] = 0.f;
        s_row[2 * (tok - b0)] = r1; s_row[2 * (tok - b0) + 1] = -1;
      }
    }
  }
  if (K == 2 && warp == 0) {
    int c1[MAXE], c2[MAXE];
#pragma unroll
    for (int e = 0; e < MAXE; ++e) { c1[e] = s_pre[e]; c2[e] = s_pre[MAXE + e]; }
    const unsigned lt = (1u << lane) - 1u;
    for (int base = b0; base < b1; base += 32) {
      const int tok = base + lane;
      const bool valid = tok < b1;
      int e1 = -1, e2 = -1;
      if (valid) { const int2 v = __ldg(reinterpret_cast<const int2*>(p.idx) + tok); e1 = v.x; e2 = v.y; }
      int loc1 = 0, loc2 = 0;
#pragma unroll
      for (int e = 0; e < MAXE; ++e) {
        if (e < E) {
          const unsigned a = __ballot_sync(0xffffffffu, e1 == e), b = __ballot_sync(0xffffffffu, e2 == e);
          if (e1 == e) loc1 = c1[e] + __popc(a & lt);
          if (e2 == e) loc2 = s_tot[e] + c2[e] + __popc(b & lt);
          c1[e] += __popc(a); c2[e] += __popc(b);
        }
      }
      if (valid) {
        const bool k1 = loc1 < p.capacity, k2 = loc2 < p.capacity;
        const float g1 = k1 ? __ldg(p.gates + (size_t)tok * E + e1) : 0.f;
        const float g2 = k2 ? __ldg(p.gates + (size_t)tok * E + e2) : 0.f;
        const float den = fmaxf(g1 + g2, FLT_EPSILON);
        const int r1 = k1 ? s_off[e1] + loc1 : -1, r2 = k2 ? s_off[e2] + loc2 : -1;
        p.row[2 * tok] = r1; p.row[2 * tok + 1] = r2;
        p.w[2 * tok] = g1 / den; p.w[2 * tok + 1] = g2 / den;
        s_row[2 * (tok - b0)] = r1; s_row[2 * (tok - b0) + 1] = r2;
      }
    }
  }
  __syncthreads();
  // scatter the token rows to their expert rows (two tokens per warp in flight; the rows were just read by the gate kernel: L2 hits)
  for (int t0 = b0 + warp * TOK_PER_WARP; t0 < b1; t0 += RT_WARPS * TOK_PER_WARP) {
    const bool has1 = t0 + 1 < b1;
    const int ra1 = s_row[2 * (t0 - b0)], ra2 = s_row[2 * (t0 - b0) + 1];
    const int rb1 = has1 ? s_row[2 * (t0 + 1 - b0)] : -1, rb2 = has1 ? s_row[2 * (t0 + 1 - b0) + 1] : -1;
    const uint4* xa = reinterpret_cast<const uint4*>(p.x + (size_t)t0 * H);
    const uint4* xb = reinterpret_cast<const uint4*>(p.x + (size_t)(has1 ? t0 + 1 : t0) * H);
    for (int v = lane; v < hv; v += 32) {
      const uint4 ua = ldg_nc_v4(xa + v), ub = ldg_nc_v4(xb + v);
      if (ra1 >= 0) stg_v4(reinterpret_cast<uint4*>(p.xp + (size_t)ra1 * H) + v, ua);
      if (ra2 >= 0) stg_v4(reinterpret_cast<uint4*>(p.xp + (size_t)ra2 * H) + v, ua);
      if (rb1 >= 0) stg_v4(reinterpret_cast<uint4*>(p.xp + (size_t)rb1 * H) + v, ub);
      if (rb2 >= 0) stg_v4(reinterpret_cast<uint4*>(p.xp + (size_t)rb2 * H) + v, ub);
    }
  }
  // zero the padding rows [offsets[e] + used[e], offsets[e+1]) (128-row alignment / capacity slabs): they are operands of the grouped
  // wgrad reduction and must be inert.  Pad row q (global numbering over the experts) belongs to CTA q mod gridDim, one warp per row.
  {
    int q0 = 0;
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (int e = 0; e < E; ++e) {
      const int first = s_off[e] + s_used[e], npad = s_off[e + 1] - first;
      for (int q = (int)blockIdx.x * RT_WARPS + warp; q < q0 + npad; q += (int)gridDim.x * RT_WARPS) {
        if (q < q0) continue;
        uint4* dst = reinterpret_cast<uint4*>(p.xp + (size_t)(first + q - q0) * H);
        for (int v = lane; v < hv; v += 32) stg_v4(dst + v, z);
      }
      q0 += npad;
    }
  }
}

// out[s] = bf16( bf16(w1)*y[row1] + bf16(w2)*y[row2] ) (+ residual, rounded again like the reference's bf16 add)
__global__ void __launch_bounds__(256) moe_gather_combine_kernel(const __nv_bfloat16* __restrict__ y, const int32_t* __restrict__ row,
                                                                const float* __restrict__ w, const __nv_bfloat16* __restrict__ res,
                                                                int S, int H, __nv_bfloat16* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= S) return;
  const int r1 = row[2 * warp], r2 = row[2 * warp + 1];
  const float w1 = bf16_round(w[2 * warp]), w2 = bf16_round(w[2 * warp + 1]);
  const int hv = H >> 3;
  for (int v = lane; v < hv; v += 32) {
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = 0.f;
    if (r1 >= 0) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(y + (size_t)r1 * H) + v);
      a[0] = w1 * bf16lo(u.x); a[1] = w1 * bf16hi(u.x); a[2] = w1 * bf16lo(u.y); a[3] = w1 * bf16hi(u.y);
      a[4] = w1 * bf16lo(u.z); a[5] = w1 * bf16hi(u.z); a[6] = w1 * bf16lo(u.w); a[7] = w1 * bf16hi(u.w);
    }
    if (r2 >= 0) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(y + (size_t)r2 * H) + v);
      a[0] = fmaf(w2, bf16lo(u.x), a[0]); a[1] = fmaf(w2, bf16hi(u.x), a[1]); a[2] = fmaf(w2, bf16lo(u.y), a[2]);
      a[3] = fmaf(w2, bf16hi(u.y), a[3]); a[4] = fmaf(w2, bf16lo(u.z), a[4]); a[5] = fmaf(w2, bf16hi(u.z), a[5]);
      a[6] = fmaf(w2, bf16lo(u.w), a[6]); a[7] = fmaf(w2, bf16hi(u.w), a[7]);
    }
    if (res) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(res + (size_t)warp * H) + v);
      float rr[8] = {bf16lo(u.x), bf16hi(u.x), bf16lo(u.y), bf16hi(u.y), bf16lo(u.z), bf16hi(u.z), bf16lo(u.w), bf16hi(u.w)};
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = rr[j] + bf16_round(a[j]);
    }
    uint4 o;
    o.x = pack_bf16x2(a[0], a[1]); o.y = pack_bf16x2(a[2], a[3]); o.z = pack_bf16x2(a[4], a[5]); o.w = pack_bf16x2(a[6], a[7]);
    stg_v4(reinterpret_cast<uint4*>(out + (size_t)warp * H) + v, o);
  }
}

// dY[row_k] = bf16(w_k) * dout[s] ; dw_k = <dout[s], y[row_k]>
__global__ void __launch_bounds__(256) moe_combine_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ y,
                                                             const int32_t* __restrict__ row, const float* __restrict__ w, int S, int H,
                                                             __nv_bfloat16* __restrict__ dy, float* __restrict__ dw) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= S) return;
  const int r1 = row[2 * warp], r2 = row[2 * warp + 1];
  const float w1 = bf16_round(w[2 * warp]), w2 = bf16_round(w[2 * warp + 1]);
  const int hv = H >> 3;
  float d1 = 0.f, d2 = 0.f;
  for (int v = lane; v < hv; v += 32) {
    uint4 g = ldg_nc_v4(reinterpret_cast<const uint4*>(dout + (size_t)warp * H) + v);
    float gf[8] = {bf16lo(g.x), bf16hi(g.x), bf16lo(g.y), bf16hi(g.y), bf16lo(g.z), bf16hi(g.z), bf16lo(g.w), bf16hi(g.w)};
    if (r1 >= 0) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(y + (size_t)r1 * H) + v);
      float yf[8] = {bf16lo(u.x), bf16hi(u.x), bf16lo(u.y), bf16hi(u.y), bf16lo(u.z), bf16hi(u.z), bf16lo(u.w), bf16hi(u.w)};
      uint4 o;
#pragma unroll
      for (int j = 0; j < 8; ++j) d1 = fmaf(gf[j], yf[j], d1);
      o.x = pack_bf16x2(w1 * gf[0], w1 * gf[1]); o.y = pack_bf16x2(w1 * gf[2], w1 * gf[3]);
      o.z = pack_bf16x2(w1 * gf[4], w1 * gf[5]); o.w = pack_bf16x2(w1 * gf[6], w1 * gf[7]);
      stg_v4(reinterpret_cast<uint4*>(dy + (size_t)r1 * H) + v, o);
    }
    if (r2 >= 0) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(y + (size_t)r2 * H) + v);
      float yf[8] = {bf16lo(u.x), bf16hi(u.x), bf16lo(u.y), bf16hi(u.y), bf16lo(u.z), bf16hi(u.z), bf16lo(u.w), bf16hi(u.w)};
      uint4 o;
#pragma unroll
      for (int j = 0; j < 8; ++j) d2 = fmaf(gf[j], yf[j], d2);
      o.x = pack_bf16x2(w2 * gf[0], w2 * gf[1]); o.y = pack_bf16x2(w2 * gf[2], w2 * gf[3]);
      o.z = pack_bf16x2(w2 * gf[4], w2 * gf[5]); o.w = pack_bf16x2(w2 * gf[6], w2 * gf[7]);
      stg_v4(reinterpret_cast<uint4*>(dy + (size_t)r2 * H) + v, o);
    }
  }
  d1 = warp_sum(d1); d2 = warp_sum(d2);
  if (lane == 0) { dw[2 * warp] = (r1 >= 0) ? d1 : 0.f; dw[2 * warp + 1] = (r2 >= 0) ? d2 : 0.f; }
}

// gate backward: (dw1, dw2, d l_aux) -> dlogits through renormalisation + softmax.  K = 1: w1 is the raw gate, dgates[s, e1] += dw1
template <int K>
__global__ void moe_gate_bwd_kernel(const float* __restrict__ gates, const int32_t* __restrict__ idx, const int32_t* __restrict__ row,
                                    const float* __restrict__ dw, const float* __restrict__ meta, const float* __restrict__ g_laux,
                                    int S, int E, float* __restrict__ dlogits) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  float g[MAXE], dg[MAXE];
  const float gl = g_laux ? g_laux[0] : 0.f;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) {
    g[e] = (e < E) ? gates[(size_t)s * E + e] : 0.f;
    // d l_aux / d gates[s,e] = E * ce[e] / S , ce[e] = exp_counts[e] / S
    dg[e] = (e < E) ? gl * (float)E * (meta[4 + e] / (float)S) / (float)S : 0.f;
  }
  const int e1 = idx[2 * s], e2 = idx[2 * s + 1];
  const bool k1 = row[2 * s] >= 0, k2 = row[2 * s + 1] >= 0;
  if (K == 1) {
    const float d1 = dw[2 * s];
#pragma unroll
    for (int e = 0; e < MAXE; ++e) if (e == e1 && k1) dg[e] += d1;
  } else {
  float a = 0.f, b = 0.f;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) { if (e == e1 && k1) a = g[e]; if (e == e2 && k2) b = g[e]; }
  const float sum = a + b;
  if (sum > FLT_EPSILON) {      // clamp(min=eps) inactive -> w1 = a/(a+b), w2 = b/(a+b)
    const float inv2 = 1.f / (sum * sum);
    const float da = (dw[2 * s] - dw[2 * s + 1]) * b * inv2, db = (dw[2 * s + 1] - dw[2 * s]) * a * inv2;
#pragma unroll
    for (int e = 0; e < MAXE; ++e) { if (e == e1 && k1) dg[e] += da; if (e == e2 && k2) dg[e] += db; }
  } else {                      // clamped: w = g / eps
#pragma unroll
    for (int e = 0; e < MAXE; ++e) {
      if (e == e1 && k1) dg[e] += dw[2 * s] / FLT_EPSILON;
      if (e == e2 && k2) dg[e] += dw[2 * s + 1] / FLT_EPSILON;
    }
  }
  }
  float dot = 0.f;
#pragma unroll
  for (int e = 0; e < MAXE; ++e) dot = fmaf(g[e], dg[e], dot);
#pragma unroll
  for (int e = 0; e < MAXE; ++e) if (e < E) dlogits[(size_t)s * E + e] = g[e] * (dg[e] - dot);
}

// dx[s] = dxp[row1] + dxp[row2] + sum_e dlogits[s,e] * wg[e,:] (+ dres[s])
__global__ void __launch_bounds__(256) moe_scatter_bwd_kernel(const __nv_bfloat16* __restrict__ dxp, const int32_t* __restrict__ row,
                                                             const float* __restrict__ dlogits, const float* __restrict__ wg,
                                                             const __nv_bfloat16* __restrict__ dres, int S, int H, int E,
                                                             __nv_bfloat16* __restrict__ dx) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= S) return;
  const int r1 = row[2 * warp], r2 = row[2 * warp + 1];
  float dl[MAXE];
#pragma unroll
  for (int e = 0; e < MAXE; ++e) dl[e] = (dlogits && e < E) ? dlogits[(size_t)warp * E + e] : 0.f;
  const int hv = H >> 3;
  for (int v = lane; v < hv; v += 32) {
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = 0.f;
    if (r1 >= 0) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(dxp + (size_t)r1 * H) + v);
      a[0] += bf16lo(u.x); a[1] += bf16hi(u.x); a[2] += bf16lo(u.y); a[3] += bf16hi(u.y);
      a[4] += bf16lo(u.z); a[5] += bf16hi(u.z); a[6] += bf16lo(u.w); a[7] += bf16hi(u.w);
    }
    if (r2 >= 0) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(dxp + (size_t)r2 * H) + v);
      a[0] += bf16lo(u.x); a[1] += bf16hi(u.x); a[2] += bf16lo(u.y); a[3] += bf16hi(u.y);
      a[4] += bf16lo(u.z); a[5] += bf16hi(u.z); a[6] += bf16lo(u.w); a[7] += bf16hi(u.w);
    }
    if (dres) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(dres + (size_t)warp * H) + v);
      a[0] += bf16lo(u.x); a[1] += bf16hi(u.x); a[2] += bf16lo(u.y); a[3] += bf16hi(u.y);
      a[4] += bf16lo(u.z); a[5] += bf16hi(u.z); a[6] += bf16lo(u.w); a[7] += bf16hi(u.w);
    }
    if (dlogits) {
#pragma unroll
      for (int e = 0; e < MAXE; ++e) {
        if (e < E) {
          const float4 w0 = __ldg(reinterpret_cast<const float4*>(wg + (size_t)e * H + v * 8));
          const float4 w1 = __ldg(reinterpret_cast<const float4*>(wg + (size_t)e * H + v * 8 + 4));
          a[0] = fmaf(dl[e], w0.x, a[0]); a[1] = fmaf(dl[e], w0.y, a[1]); a[2] = fmaf(dl[e], w0.z, a[2]); a[3] = fmaf(dl[e], w0.w, a[3]);
          a[4] = fmaf(dl[e], w1.x, a[4]); a[5] = fmaf(dl[e], w1.y, a[5]); a[6] = fmaf(dl[e], w1.z, a[6]); a[7] = fmaf(dl[e], w1.w, a[7]);
        }
      }
    }
    uint4 o;
    o.x = pack_bf16x2(a[0], a[1]); o.y = pack_bf16x2(a[2], a[3]); o.z = pack_bf16x2(a[4], a[5]); o.w = pack_bf16x2(a[6], a[7]);
    stg_v4(reinterpret_cast<uint4*>(dx + (size_t)warp * H) + v, o);
  }
}

constexpr int WG_SPLITS = 32;
// ws[split,e,h] = sum_{s in split} dlogits[s,e] * x[s,h]
__global__ void __launch_bounds__(256) moe_wg_grad_partial_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ dlogits,
                                                                 int S, int H, int E, float* __restrict__ ws) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  const int split = blockIdx.y;
  const int per = (S + WG_SPLITS - 1) / WG_SPLITS;
  const int s0 = split * per, s1 = min(S, s0 + per);
  if (h >= H) return;
  float acc[MAXE];
#pragma unroll
  for (int e = 0; e < MAXE; ++e) acc[e] = 0.f;
  for (int s = s0; s < s1; ++s) {
    const float xv = __bfloat162float(x[(size_t)s * H + h]);
#pragma unroll
    for (int e = 0; e < MAXE; ++e) if (e < E) acc[e] = fmaf(__ldg(dlogits + (size_t)s * E + e), xv, acc[e]);
  }
#pragma unroll
  for (int e = 0; e < MAXE; ++e) if (e < E) ws[((size_t)split * E + e) * H + h] = acc[e];
}
__global__ void moe_wg_grad_reduce_kernel(const float* __restrict__ ws, int H, int E, float* __restrict__ dwg) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= E * H) return;
  float a = 0.f;
  for (int sp = 0; sp < WG_SPLITS; ++sp) a += ws[(size_t)sp * E * H + i];
  dwg[i] += a;
}

// ---- Residual-MoE (DeepSpeed MoE(use_residual=True)): the routed output and a dense MLP mixed per token by softmax(coefficient(x)).
// One warp per token.  Forward, all bf16 tensors as the reference rounds them:
//   z = bf16(x Wc^T + b) (fp32 accumulate), c = bf16(softmax_fp32(z)), out = bf16(bf16(moe*c0) + bf16(mlp*c1)), stream = bf16(res + out)
__global__ void __launch_bounds__(256) moe_residual_mix_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ moe,
                                                              const __nv_bfloat16* __restrict__ mlp, const __nv_bfloat16* __restrict__ res,
                                                              const __nv_bfloat16* __restrict__ wc, const __nv_bfloat16* __restrict__ bc,
                                                              int S, int H, __nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ coef) {
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= S) return;
  const int hv = H >> 3;
  const size_t o = (size_t)s * H;
  float z0 = 0.f, z1 = 0.f;
  for (int v = lane; v < hv; v += 32) {
    const uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(x + o) + v);
    const uint4 a = ldg_nc_v4(reinterpret_cast<const uint4*>(wc) + v), b = ldg_nc_v4(reinterpret_cast<const uint4*>(wc + H) + v);
    const float xf[8] = {bf16lo(u.x), bf16hi(u.x), bf16lo(u.y), bf16hi(u.y), bf16lo(u.z), bf16hi(u.z), bf16lo(u.w), bf16hi(u.w)};
    const float af[8] = {bf16lo(a.x), bf16hi(a.x), bf16lo(a.y), bf16hi(a.y), bf16lo(a.z), bf16hi(a.z), bf16lo(a.w), bf16hi(a.w)};
    const float bf[8] = {bf16lo(b.x), bf16hi(b.x), bf16lo(b.y), bf16hi(b.y), bf16lo(b.z), bf16hi(b.z), bf16lo(b.w), bf16hi(b.w)};
#pragma unroll
    for (int j = 0; j < 8; ++j) { z0 = fmaf(xf[j], af[j], z0); z1 = fmaf(xf[j], bf[j], z1); }
  }
  z0 = warp_sum(z0); z1 = warp_sum(z1);
  if (bc) { z0 += __bfloat162float(bc[0]); z1 += __bfloat162float(bc[1]); }
  z0 = bf16_round(z0); z1 = bf16_round(z1);
  const float m = fmaxf(z0, z1), e0 = expf(z0 - m), e1 = expf(z1 - m), den = e0 + e1;
  const float c0 = bf16_round(e0 / den), c1 = bf16_round(e1 / den);
  if (lane == 0) *reinterpret_cast<uint32_t*>(coef + 2 * (size_t)s) = pack_bf16x2(c0, c1);
  for (int v = lane; v < hv; v += 32) {
    const uint4 a = ldg_nc_v4(reinterpret_cast<const uint4*>(moe + o) + v), b = ldg_nc_v4(reinterpret_cast<const uint4*>(mlp + o) + v);
    const uint4 r = ldg_nc_v4(reinterpret_cast<const uint4*>(res + o) + v);
    const float af[8] = {bf16lo(a.x), bf16hi(a.x), bf16lo(a.y), bf16hi(a.y), bf16lo(a.z), bf16hi(a.z), bf16lo(a.w), bf16hi(a.w)};
    const float bf[8] = {bf16lo(b.x), bf16hi(b.x), bf16lo(b.y), bf16hi(b.y), bf16lo(b.z), bf16hi(b.z), bf16lo(b.w), bf16hi(b.w)};
    const float rf[8] = {bf16lo(r.x), bf16hi(r.x), bf16lo(r.y), bf16hi(r.y), bf16lo(r.z), bf16hi(r.z), bf16lo(r.w), bf16hi(r.w)};
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = rf[j] + bf16_round(bf16_round(af[j] * c0) + bf16_round(bf[j] * c1));
    uint4 w;
    w.x = pack_bf16x2(y[0], y[1]); w.y = pack_bf16x2(y[2], y[3]); w.z = pack_bf16x2(y[4], y[5]); w.w = pack_bf16x2(y[6], y[7]);
    stg_v4(reinterpret_cast<uint4*>(out + o) + v, w);
  }
}

// Backward of the mix for upstream g (the residual's own gradient is g itself and is not touched here).  One warp per token:
//   d_moe = bf16(g*c0), d_mlp = bf16(g*c1), dc_j = sum_h g*{moe,mlp}_j (fp32), dz = c (dc - <c, dc>),
//   dx_coef = bf16(dz0*Wc[0] + dz1*Wc[1]) (the coefficient's input-gradient term).  dz [S,2] fp32 feeds the Wc / b reduction.
__global__ void __launch_bounds__(256) moe_residual_mix_bwd_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ moe,
                                                                  const __nv_bfloat16* __restrict__ mlp, const __nv_bfloat16* __restrict__ coef,
                                                                  const __nv_bfloat16* __restrict__ wc, int S, int H,
                                                                  __nv_bfloat16* __restrict__ d_moe, __nv_bfloat16* __restrict__ d_mlp,
                                                                  float* __restrict__ dz, __nv_bfloat16* __restrict__ dx) {
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= S) return;
  const int hv = H >> 3;
  const size_t o = (size_t)s * H;
  const uint32_t cw = __ldg(reinterpret_cast<const unsigned int*>(coef) + s);
  const float c0 = bf16lo(cw), c1 = bf16hi(cw);
  float d0 = 0.f, d1 = 0.f;
  for (int v = lane; v < hv; v += 32) {
    const uint4 q = ldg_nc_v4(reinterpret_cast<const uint4*>(g + o) + v);
    const uint4 a = ldg_nc_v4(reinterpret_cast<const uint4*>(moe + o) + v), b = ldg_nc_v4(reinterpret_cast<const uint4*>(mlp + o) + v);
    const float gf[8] = {bf16lo(q.x), bf16hi(q.x), bf16lo(q.y), bf16hi(q.y), bf16lo(q.z), bf16hi(q.z), bf16lo(q.w), bf16hi(q.w)};
    const float af[8] = {bf16lo(a.x), bf16hi(a.x), bf16lo(a.y), bf16hi(a.y), bf16lo(a.z), bf16hi(a.z), bf16lo(a.w), bf16hi(a.w)};
    const float bf[8] = {bf16lo(b.x), bf16hi(b.x), bf16lo(b.y), bf16hi(b.y), bf16lo(b.z), bf16hi(b.z), bf16lo(b.w), bf16hi(b.w)};
#pragma unroll
    for (int j = 0; j < 8; ++j) { d0 = fmaf(gf[j], af[j], d0); d1 = fmaf(gf[j], bf[j], d1); }
    uint4 w;
    w.x = pack_bf16x2(gf[0] * c0, gf[1] * c0); w.y = pack_bf16x2(gf[2] * c0, gf[3] * c0);
    w.z = pack_bf16x2(gf[4] * c0, gf[5] * c0); w.w = pack_bf16x2(gf[6] * c0, gf[7] * c0);
    stg_v4(reinterpret_cast<uint4*>(d_moe + o) + v, w);
    w.x = pack_bf16x2(gf[0] * c1, gf[1] * c1); w.y = pack_bf16x2(gf[2] * c1, gf[3] * c1);
    w.z = pack_bf16x2(gf[4] * c1, gf[5] * c1); w.w = pack_bf16x2(gf[6] * c1, gf[7] * c1);
    stg_v4(reinterpret_cast<uint4*>(d_mlp + o) + v, w);
  }
  d0 = warp_sum(d0); d1 = warp_sum(d1);
  const float dot = c0 * d0 + c1 * d1;
  const float z0 = c0 * (d0 - dot), z1 = c1 * (d1 - dot);
  if (lane == 0) { dz[2 * (size_t)s] = z0; dz[2 * (size_t)s + 1] = z1; }
  for (int v = lane; v < hv; v += 32) {
    const uint4 a = ldg_nc_v4(reinterpret_cast<const uint4*>(wc) + v), b = ldg_nc_v4(reinterpret_cast<const uint4*>(wc + H) + v);
    const float af[8] = {bf16lo(a.x), bf16hi(a.x), bf16lo(a.y), bf16hi(a.y), bf16lo(a.z), bf16hi(a.z), bf16lo(a.w), bf16hi(a.w)};
    const float bf[8] = {bf16lo(b.x), bf16hi(b.x), bf16lo(b.y), bf16hi(b.y), bf16lo(b.z), bf16hi(b.z), bf16lo(b.w), bf16hi(b.w)};
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = fmaf(z1, bf[j], z0 * af[j]);
    uint4 w;
    w.x = pack_bf16x2(y[0], y[1]); w.y = pack_bf16x2(y[2], y[3]); w.z = pack_bf16x2(y[4], y[5]); w.w = pack_bf16x2(y[6], y[7]);
    stg_v4(reinterpret_cast<uint4*>(dx + o) + v, w);
  }
}

// dWc / db of the coefficient, deterministic: a fixed partition of the tokens into RM_SPLITS contiguous ranges (a function of S only),
// per-range partial sums in token order, then one pass adding the ranges in range order into the bf16 gradient.
constexpr int RM_SPLITS = 128;
constexpr int RM_COLS = 1024;                         // columns per CTA of the partial kernel: 128 threads x 8
// ws[(split*2 + j)*H + h] = sum_{s in split} dz[s,j] * x[s,h] ; ws[RM_SPLITS*2*H + split*2 + j] = sum_{s in split} dz[s,j]
__global__ void __launch_bounds__(128) moe_residual_coef_grad_partial_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ dz,
                                                                            int S, int H, float* __restrict__ ws) {
  const int split = blockIdx.y;
  const int per = (S + RM_SPLITS - 1) / RM_SPLITS;
  const int s0 = min(S, split * per), s1 = min(S, s0 + per);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float b0 = 0.f, b1 = 0.f;
    for (int s = s0; s < s1; ++s) { b0 += __ldg(dz + 2 * s); b1 += __ldg(dz + 2 * s + 1); }
    ws[(size_t)RM_SPLITS * 2 * H + 2 * split] = b0;
    ws[(size_t)RM_SPLITS * 2 * H + 2 * split + 1] = b1;
  }
  const int h0 = (blockIdx.x * RM_COLS) + threadIdx.x * 8;
  if (h0 >= H) return;
  float a0[8], a1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { a0[j] = 0.f; a1[j] = 0.f; }
  for (int s = s0; s < s1; ++s) {
    const float z0 = __ldg(dz + 2 * s), z1 = __ldg(dz + 2 * s + 1);
    const uint4 u = ldg_nc_v4(x + (size_t)s * H + h0);
    const float xf[8] = {bf16lo(u.x), bf16hi(u.x), bf16lo(u.y), bf16hi(u.y), bf16lo(u.z), bf16hi(u.z), bf16lo(u.w), bf16hi(u.w)};
#pragma unroll
    for (int j = 0; j < 8; ++j) { a0[j] = fmaf(z0, xf[j], a0[j]); a1[j] = fmaf(z1, xf[j], a1[j]); }
  }
  float* w0 = ws + (size_t)(split * 2) * H + h0;
  float* w1 = w0 + H;
#pragma unroll
  for (int j = 0; j < 8; j += 4) {
    *reinterpret_cast<float4*>(w0 + j) = make_float4(a0[j], a0[j + 1], a0[j + 2], a0[j + 3]);
    *reinterpret_cast<float4*>(w1 + j) = make_float4(a1[j], a1[j + 1], a1[j + 2], a1[j + 3]);
  }
}
// dwc[i] = bf16(dwc[i] + sum_split ws[split][i]) for i < 2H, dbc[j] likewise (either pointer null: that parameter is frozen)
__global__ void moe_residual_coef_grad_reduce_kernel(const float* __restrict__ ws, int H, __nv_bfloat16* __restrict__ dwc,
                                                     __nv_bfloat16* __restrict__ dbc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * H + 2) return;
  const bool bias = i >= 2 * H;
  __nv_bfloat16* dst = bias ? (dbc ? dbc + (i - 2 * H) : nullptr) : (dwc ? dwc + i : nullptr);
  if (!dst) return;
  const size_t stride = bias ? 2 : (size_t)2 * H;
  const float* src = bias ? ws + (size_t)RM_SPLITS * 2 * H + (i - 2 * H) : ws + i;
  float a = 0.f;
  for (int sp = 0; sp < RM_SPLITS; ++sp) a += src[(size_t)sp * stride];
  *dst = __float2bfloat16_rn(__bfloat162float(*dst) + a);
}

}  // namespace

extern "C" int lmod_moe_capacity(int64_t S, int E, double capacity_factor, int64_t min_capacity) {
  // deepspeed _capacity: ceil(S/E * (cf*2)) ; computed in double like Python, raised to min_capacity.  The factor is taken as a double:
  // a user-set factor such as 0.3 rounded to float first moves the product across an integer (S=320, E=4: C=49 instead of 48).
  double c = ceil(((double)S / (double)E) * (capacity_factor * 2.0));
  int64_t ci = (int64_t)c;
  if (ci < min_capacity) ci = min_capacity;
  return (int)ci;
}

// top1gating's _capacity: ceil(S/E * cf) (no factor 2), in double like lmod_moe_capacity, raised to min_capacity
extern "C" int lmod_moe_capacity_top1(int64_t S, int E, double capacity_factor, int64_t min_capacity) {
  double c = ceil(((double)S / (double)E) * capacity_factor);
  int64_t ci = (int64_t)c;
  if (ci < min_capacity) ci = min_capacity;
  return (int)ci;
}

static int route_tpb(int64_t S) {
  int64_t tpb = TILE_MIN;
  while ((S + tpb - 1) / tpb > MAX_TILES) tpb += TILE_MIN;
  return (int)tpb;
}

// int32 elements of scratch lmod_moe_route_scatter needs (per call; no initialisation required): tile counts + tile gate sums
extern "C" int64_t lmod_moe_route_ws_elems(int64_t S, int E) {
  (void)E;
  const int tpb = route_tpb(S);
  const int64_t ntiles = (S + tpb - 1) / tpb;
  return ntiles * (2 * MAXE + MAXE);
}

extern "C" int64_t lmod_moe_route_top1_ws_elems(int64_t S, int E) {
  return lmod_moe_route_ws_elems(S, E) + 2 * MAXE;
}

// the checks and the launch plan both routers share; the capacity is the caller's (top-2 or top-1 rule)
static int route_params(RouteParams& p, const char* fn, const void* x, const float* wg, const float* noise, int64_t S, int64_t H, int E,
                        int capacity, int layout, float* logits, float* gates, int32_t* idx, int32_t* row, float* w, int32_t* offsets,
                        float* meta, void* xp, int32_t* ws) {
  LMOD_CHECK_ARG(x && wg && noise && logits && gates && idx && row && w && offsets && meta && xp && ws, "%s: null pointer", fn);
  LMOD_CHECK_ARG(E >= 2 && E <= MAXE, "%s: 2 <= E <= %d required (got %d)", fn, MAXE, E);
  LMOD_CHECK_ARG(S > 0 && H > 0 && H % 8 == 0, "%s: H must be a multiple of 8", fn);
  LMOD_CHECK_ARG(layout >= 0 && layout <= 2, "%s: layout must be 0 (compact), 1 (capacity slabs) or 2 (compact, 128-aligned)", fn);
  p.x = (const __nv_bfloat16*)x; p.wg = wg; p.noise = noise; p.S = (int)S; p.H = (int)H; p.E = E;
  p.capacity = capacity;
  p.layout = layout;
  p.logits = logits; p.gates = gates; p.idx = idx; p.row = row; p.w = w; p.offsets = offsets; p.meta = meta;
  p.xp = (__nv_bfloat16*)xp;
  p.tpb = route_tpb(S);
  p.ntiles = (int)((S + p.tpb - 1) / p.tpb);
  LMOD_CHECK_ARG(p.tpb <= 2048, "%s: S = %lld is beyond the tile plan", fn, (long long)S);
  p.tile_cnt = ws;
  p.tile_gsum = reinterpret_cast<float*>(ws + (size_t)p.ntiles * 2 * MAXE);
  p.sel = ws + (size_t)p.ntiles * 3 * MAXE;
  const size_t smem = (size_t)E * H * 4 + (size_t)p.tpb * MAXE * 4;
  LMOD_CHECK_ARG(smem <= 200 * 1024, "%s: E*H*4 exceeds the shared-memory budget", fn);
  return LMOD_OK;
}

template <int K>
static int launch_gate(const RouteParams& p, cudaStream_t stream) {
  const size_t smem = (size_t)p.E * p.H * 4 + (size_t)p.tpb * MAXE * 4;
  static size_t smem_set = 0;
  if (smem > 48 * 1024 && smem > smem_set) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(moe_gate_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    smem_set = smem;
  }
  moe_gate_kernel<K><<<p.ntiles, RT_THREADS, smem, stream>>>(p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_route_scatter(const void* x, const float* wg, const float* noise, int64_t S, int64_t H, int E,
                                      double capacity_factor, int64_t min_capacity, int layout, float* logits, float* gates,
                                      int32_t* idx, int32_t* row, float* w, int32_t* offsets, float* meta, void* xp,
                                      int32_t* ws, void* stream) {
  RouteParams p;
  const int rc = route_params(p, "lmod_moe_route_scatter", x, wg, noise, S, H, E, lmod_moe_capacity(S, E, capacity_factor, min_capacity),
                              layout, logits, gates, idx, row, w, offsets, meta, xp, ws);
  if (rc != LMOD_OK) return rc;
  p.sel = nullptr;
  const int rg = launch_gate<2>(p, (cudaStream_t)stream);
  if (rg != LMOD_OK) return rg;
  moe_seat_scatter_kernel<2><<<p.ntiles, RT_THREADS, 0, (cudaStream_t)stream>>>(p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_route_scatter_top1(const void* x, const float* wg, const float* uniform, int64_t S, int64_t H, int E,
                                           double capacity_factor, int64_t min_capacity, int layout, float* logits, float* gates,
                                           int32_t* idx, int32_t* row, float* w, int32_t* offsets, float* meta, void* xp,
                                           int32_t* ws, void* stream) {
  // top1gating fails in these two cases (an assert on the batch size, torch.topk with k > S); say so before any launch
  LMOD_CHECK_ARG(S >= min_capacity, "lmod_moe_route_scatter_top1: %lld tokens < min_capacity %lld (top1gating requires S >= min_capacity)",
                 (long long)S, (long long)min_capacity);
  const int C = lmod_moe_capacity_top1(S, E, capacity_factor, min_capacity);
  LMOD_CHECK_ARG(C <= S, "lmod_moe_route_scatter_top1: capacity %d > %lld tokens (top1gating's topk over the tokens needs C <= S)",
                 C, (long long)S);
  RouteParams p;
  const int rc = route_params(p, "lmod_moe_route_scatter_top1", x, wg, uniform, S, H, E, C, layout, logits, gates, idx, row, w, offsets,
                              meta, xp, ws);
  if (rc != LMOD_OK) return rc;
  const int rg = launch_gate<1>(p, (cudaStream_t)stream);
  if (rg != LMOD_OK) return rg;
  moe_top1_select_kernel<<<E, SEL_THREADS, 0, (cudaStream_t)stream>>>(p);
  LMOD_LAUNCH_OK();
  moe_seat_scatter_kernel<1><<<p.ntiles, RT_THREADS, 0, (cudaStream_t)stream>>>(p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_gather_combine(const void* y, const int32_t* row, const float* w, const void* residual, int64_t S,
                                       int64_t H, void* out, void* stream) {
  LMOD_CHECK_ARG(y && row && w && out && S > 0 && H % 8 == 0, "lmod_moe_gather_combine: bad arguments");
  unsigned blocks = (unsigned)((S * 32 + 255) / 256);
  moe_gather_combine_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)y, row, w, (const __nv_bfloat16*)residual,
                                                                      (int)S, (int)H, (__nv_bfloat16*)out);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_combine_bwd(const void* dout, const void* y, const int32_t* row, const float* w, int64_t S, int64_t H,
                                    void* dy, float* dw, void* stream) {
  LMOD_CHECK_ARG(dout && y && row && w && dy && dw && S > 0 && H % 8 == 0, "lmod_moe_combine_bwd: bad arguments");
  unsigned blocks = (unsigned)((S * 32 + 255) / 256);
  moe_combine_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)y, row, w, (int)S,
                                                                   (int)H, (__nv_bfloat16*)dy, dw);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_gate_bwd(const float* gates, const int32_t* idx, const int32_t* row, const float* dw, const float* meta,
                                 const float* g_laux, int64_t S, int E, float* dlogits, void* stream) {
  LMOD_CHECK_ARG(gates && idx && row && dw && meta && dlogits && S > 0 && E >= 2 && E <= MAXE, "lmod_moe_gate_bwd: bad arguments");
  moe_gate_bwd_kernel<2><<<(unsigned)((S + 127) / 128), 128, 0, (cudaStream_t)stream>>>(gates, idx, row, dw, meta, g_laux, (int)S, E,
                                                                                        dlogits);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_gate_bwd_top1(const float* gates, const int32_t* idx, const int32_t* row, const float* dw, const float* meta,
                                      const float* g_laux, int64_t S, int E, float* dlogits, void* stream) {
  LMOD_CHECK_ARG(gates && idx && row && dw && meta && dlogits && S > 0 && E >= 2 && E <= MAXE, "lmod_moe_gate_bwd_top1: bad arguments");
  moe_gate_bwd_kernel<1><<<(unsigned)((S + 127) / 128), 128, 0, (cudaStream_t)stream>>>(gates, idx, row, dw, meta, g_laux, (int)S, E,
                                                                                        dlogits);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_scatter_bwd(const void* dxp, const int32_t* row, const float* dlogits, const float* wg, const void* dres,
                                    int64_t S, int64_t H, int E, void* dx, void* stream) {
  LMOD_CHECK_ARG(dxp && row && dx && S > 0 && H % 8 == 0 && E <= MAXE, "lmod_moe_scatter_bwd: bad arguments");
  LMOD_CHECK_ARG(!dlogits || wg, "lmod_moe_scatter_bwd: wg required with dlogits");
  unsigned blocks = (unsigned)((S * 32 + 255) / 256);
  moe_scatter_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dxp, row, dlogits, wg, (const __nv_bfloat16*)dres,
                                                                   (int)S, (int)H, E, (__nv_bfloat16*)dx);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_moe_wg_grad(const void* x, const float* dlogits, int64_t S, int64_t H, int E, float* ws, float* dwg, void* stream) {
  LMOD_CHECK_ARG(x && dlogits && ws && dwg && S > 0 && H > 0 && E <= MAXE, "lmod_moe_wg_grad: bad arguments");
  dim3 grid((unsigned)((H + 255) / 256), WG_SPLITS);
  moe_wg_grad_partial_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, dlogits, (int)S, (int)H, E, ws);
  LMOD_LAUNCH_OK();
  moe_wg_grad_reduce_kernel<<<(unsigned)((E * H + 255) / 256), 256, 0, (cudaStream_t)stream>>>(ws, (int)H, E, dwg);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

extern "C" int lmod_moe_residual_mix(const void* x, const void* moe, const void* mlp, const void* res, const void* wc, const void* bc,
                                     int64_t S, int64_t H, void* out, void* coef, void* stream) {
  LMOD_CHECK_ARG(x && moe && mlp && res && wc && out && coef && S > 0 && H > 0 && H % 8 == 0,
                 "lmod_moe_residual_mix: bad arguments (H must be a multiple of 8)");
  LMOD_CHECK_ARG(aligned16(x) && aligned16(moe) && aligned16(mlp) && aligned16(res) && aligned16(wc) && aligned16(out) && aligned16(coef),
                 "lmod_moe_residual_mix: every tensor must be 16-byte aligned");
  const unsigned blocks = (unsigned)((S * 32 + 255) / 256);
  moe_residual_mix_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x, (const __nv_bfloat16*)moe, (const __nv_bfloat16*)mlp, (const __nv_bfloat16*)res, (const __nv_bfloat16*)wc,
      (const __nv_bfloat16*)bc, (int)S, (int)H, (__nv_bfloat16*)out, (__nv_bfloat16*)coef);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int64_t lmod_moe_residual_ws_elems(int64_t H) { return (int64_t)RM_SPLITS * (2 * H + 2); }

extern "C" int lmod_moe_residual_mix_bwd(const void* g, const void* x, const void* moe, const void* mlp, const void* coef, const void* wc,
                                         int64_t S, int64_t H, void* d_moe, void* d_mlp, float* dz, void* dx_coef, float* ws, void* dwc,
                                         void* dbc, void* stream) {
  LMOD_CHECK_ARG(g && moe && mlp && coef && wc && d_moe && d_mlp && dz && dx_coef && S > 0 && H > 0 && H % 8 == 0,
                 "lmod_moe_residual_mix_bwd: bad arguments (H must be a multiple of 8)");
  LMOD_CHECK_ARG(!(dwc || dbc) || (x && ws), "lmod_moe_residual_mix_bwd: x and ws are required for the coefficient's gradient");
  LMOD_CHECK_ARG(aligned16(g) && aligned16(moe) && aligned16(mlp) && aligned16(wc) && aligned16(d_moe) && aligned16(d_mlp) &&
                 aligned16(dx_coef) && (!x || aligned16(x)) && (!ws || aligned16(ws)) && ((uintptr_t)coef & 3u) == 0,
                 "lmod_moe_residual_mix_bwd: every [S,H] tensor must be 16-byte aligned");
  const unsigned blocks = (unsigned)((S * 32 + 255) / 256);
  moe_residual_mix_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)g, (const __nv_bfloat16*)moe, (const __nv_bfloat16*)mlp, (const __nv_bfloat16*)coef, (const __nv_bfloat16*)wc,
      (int)S, (int)H, (__nv_bfloat16*)d_moe, (__nv_bfloat16*)d_mlp, dz, (__nv_bfloat16*)dx_coef);
  LMOD_LAUNCH_OK();
  if (dwc || dbc) {
    dim3 grid((unsigned)((H + RM_COLS - 1) / RM_COLS), RM_SPLITS);
    moe_residual_coef_grad_partial_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, dz, (int)S, (int)H, ws);
    LMOD_LAUNCH_OK();
    moe_residual_coef_grad_reduce_kernel<<<(unsigned)((2 * H + 2 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        ws, (int)H, (__nv_bfloat16*)dwc, (__nv_bfloat16*)dbc);
    LMOD_LAUNCH_OK();
  }
  return LMOD_OK;
}
