// gemm.cu -- hand-written wgmma + TMA GEMM for sm_90a:  D[M,N] (+)= A[M,K] * B[N,K]^T  (bf16 in, fp32 register accumulate)
//
// Replaces the nn.Linear call sites of the path (modeling_qwen2.py:199-200 gate/up/down, :678-680 q/k/v, :726 o_proj, :1176
// lm_head; CLIP / projector linears) and, in its grouped form, DeepSpeed's per-expert loop (Experts.forward) on COMPACT
// expert rows -- no capacity padding.
//
// Structure (one persistent CTA per SM, 384 threads = three warpgroups, warp-specialised):
//   warpgroup 0, thread 0 : TMA producer -- cp.async.bulk.tensor.2d into a 128B-swizzled shared-memory ring (A 128x64, B BNx64;
//                           4 stages for BN = 256, 6 for BN = 128); gives its registers to the math warpgroups (setmaxnreg)
//   warpgroups 1, 2       : math -- each owns 64 rows of the 128 x BN tile: wgmma.mma_async m64nBNk16 (both operands from shared
//                           memory), fp32 accumulators in registers; one k-block of MMAs stays in flight while the previous
//                           stage is handed back; then the epilogue (+bias) (+D_old) ... -> bf16 -> global from the registers
//   mbarriers             : full[stage] (TMA complete_tx) / empty[stage] (one arrive per math warpgroup)
// Operand "major-ness" is a template parameter, so dgrad (B = W as stored, MN-major) and wgrad (A = dY^T, B = X^T, both MN-major)
// run without transposes: the wgmma transpose bits and descriptors and the TMA boxes change, the pipeline does not.
#include <stdlib.h>
#include "sm90.cuh"

namespace {

constexpr int BM = 128, BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;            // 16 KB
// two tile widths: BN = 256 (4-stage ring) for the big GEMMs, BN = 128 (6-stage ring) when a 256-wide tiling would leave SMs idle
template <int BN> struct Cfg {
  static constexpr int STAGES = (BN == 256) ? 4 : 6;
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024;   // + alignment slack
};
constexpr int GEMM_THREADS = 384;
constexpr int MAX_GROUPS = 8;

struct GemmParams {
  __nv_bfloat16* D;
  const __nv_bfloat16* bias;       // [N] or null
  float* D32;                      // optional fp32 output (accumulated: D32 += acc) instead of D
  int64_t ldd;
  int M, N, K;                     // dense problem (per group for grouped: M is the slab bound)
  int bn;                          // tile width (256 or 128)
  int beta;                        // 1: D = bf16(D + acc)
  int splits;                      // split-K factor (>1: fp32 atomic accumulation into D32)
  // fused SwiGLU forward (Qwen2MLP act_fn(gate_proj(x)) * up_proj(x), modeling_qwen2.py:199-200): B is the fused gate|up weight [2I, K]
  // as stored (gate rows, then up rows); N = I; an output tile = 128 act columns whose accumulator holds [128 gate | 128 up] columns (the
  // two halves of the B stage are loaded from rows n0 and I + n0).  D[:, I] = bf16(bf16(silu(g)) * u); H1 (optional) keeps the bf16
  // pre-activations [M, 2I] for the backward.
  int swiglu;
  int swiglu_I;
  __nv_bfloat16* H1;
  int64_t ld_h1;
  // fused SwiGLU backward in the epilogue of the down_proj dgrad (dact = dY W_dn, N = I): reads the saved pre-activations GU [M, 2I],
  // writes d(gate) | d(up) into D [M, 2I] (columns col and I + col) -- the [M, I] dact tensor never exists
  int silu_bwd;
  const __nv_bfloat16* GU;
  int64_t ld_gu;
  // fused rotary embedding in the epilogue of the q|k|v projection (apply_rotary_pos_emb, modeling_qwen2.py:159-184): columns below
  // rope_cols (the q and k heads) are rotated per head of rope_hd columns with cos / sin [max_pos, rope_hd] rows picked by rope_pos[row];
  // the v columns pass through.  Same bf16 roundings as GEMM(+bias) followed by lmod_rope (bit-identical).
  const __nv_bfloat16* rope_cos;
  const __nv_bfloat16* rope_sin;
  const int64_t* rope_pos;
  int rope_hd, rope_cols;
  // fused residual add (Qwen2DecoderLayer `hidden_states = residual + hidden_states`, modeling_qwen2.py:796,808; CLIP encoder layers):
  // D = bf16( bf16(acc + bias) + R ) -- the GEMM output is rounded to bf16 first, exactly as the reference materialises it before its add
  const __nv_bfloat16* R;
  int64_t ld_r;
  int dbg_nostore;                 // timing experiments only (LMOD_GEMM_NOSTORE=1): the epilogue does not write D
  // grouped (experts): row ranges from `offsets` (device), B / D32 advance per group
  const int32_t* offsets;          // [groups+1] or null
  int groups;
  int64_t b_group_rows;            // rows of B per group (N for K-major B) -- B coordinate offset
  int64_t d_group_stride;          // wgrad grouped: element stride of D per group
  int wgrad_grouped;               // 1: groups split the REDUCTION (K) range via offsets; M,N dense per group
  // dense only: extents read from DEVICE memory at kernel start (the loss head works on the batch's supervised rows, whose count is
  // data-dependent, inside a CUDA graph): M_eff = min(M, *m_dev), K_eff = min(K, round_up(*k_dev, BK)); null = static
  const int32_t* m_dev;
  const int32_t* k_dev;
};

__device__ __forceinline__ GemmParams effective_extents(const GemmParams& in) {
  GemmParams p = in;
  if (in.m_dev) p.M = min(in.M, max(0, *in.m_dev));
  if (in.k_dev) p.K = min(in.K, (max(0, *in.k_dev) + BK - 1) / BK * BK);
  return p;
}

struct Tile { int m0, n0, kb0, kb1, group, m_end; };

// The epilogue works on what one thread holds of a wgmma accumulator: two adjacent columns (col, col + 1) of one row.
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ void bias2(const __nv_bfloat16* b, float& f0, float& f1) {
  const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(b));
  f0 += bf16lo(w); f1 += bf16hi(w);
}
// rotate one (x1, x2) pair of columns of a head: x = bf16(acc + bias); o1 = bf16(bf16(x1 c) + bf16(-x2 s)), o2 = bf16(bf16(x2 c) + bf16(x1 s))
// (the expression of rope_vec_kernel).  a1 / a2: fp32 accumulators of the first-half / second-half columns, b1 / b2: their bias (or null).
__device__ __forceinline__ void rope_store2(float a10, float a11, float a20, float a21, const __nv_bfloat16* b1, const __nv_bfloat16* b2,
                                            const __nv_bfloat16* cs, const __nv_bfloat16* sn, __nv_bfloat16* d1, __nv_bfloat16* d2) {
  float x1[2] = {a10, a11}, x2[2] = {a20, a21};
  if (b1) { bias2(b1, x1[0], x1[1]); bias2(b2, x2[0], x2[1]); }
  const uint32_t cw = __ldg(reinterpret_cast<const uint32_t*>(cs)), sw = __ldg(reinterpret_cast<const uint32_t*>(sn));
  const float c[2] = {bf16lo(cw), bf16hi(cw)}, s[2] = {bf16lo(sw), bf16hi(sw)};
  float o1[2], o2[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float y1 = bf16_round(x1[j]), y2 = bf16_round(x2[j]);
    o1[j] = bf16_round(y1 * c[j]) + bf16_round(-y2 * s[j]);
    o2[j] = bf16_round(y2 * c[j]) + bf16_round(y1 * s[j]);
  }
  *reinterpret_cast<uint32_t*>(d1) = pack_bf16x2(o1[0], o1[1]);
  *reinterpret_cast<uint32_t*>(d2) = pack_bf16x2(o2[0], o2[1]);
}
// act = bf16(bf16(silu(g)) * u) on bf16-rounded GEMM outputs: the expression of silu_mul_fwd_kernel (bit-identical to GEMM + that kernel)
__device__ __forceinline__ void swiglu_store2(float g0, float g1, float u0, float u1, __nv_bfloat16* act, __nv_bfloat16* h1g, __nv_bfloat16* h1u) {
  const float gb[2] = {bf16_round(g0), bf16_round(g1)}, ub[2] = {bf16_round(u0), bf16_round(u1)};
  float f[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) f[j] = bf16_round(gb[j] * sigmoid_f(gb[j])) * ub[j];
  *reinterpret_cast<uint32_t*>(act) = pack_bf16x2(f[0], f[1]);
  if (h1g) {
    *reinterpret_cast<uint32_t*>(h1g) = pack_bf16x2(gb[0], gb[1]);
    *reinterpret_cast<uint32_t*>(h1u) = pack_bf16x2(ub[0], ub[1]);
  }
}
// d(gate), d(up) from dact (the fp32 accumulator rounded to bf16, as the unfused path materialises it) and the saved pre-activations:
// the expression of silu_mul_bwd_kernel
__device__ __forceinline__ void silu_bwd_store2(float a0, float a1, const __nv_bfloat16* gp, const __nv_bfloat16* up, __nv_bfloat16* dgp, __nv_bfloat16* dup) {
  const uint32_t gv = __ldg(reinterpret_cast<const uint32_t*>(gp)), uv = __ldg(reinterpret_cast<const uint32_t*>(up));
  const float g[2] = {bf16lo(gv), bf16hi(gv)}, u[2] = {bf16lo(uv), bf16hi(uv)}, dacc[2] = {a0, a1};
  float dg[2], du[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float d = bf16_round(dacc[j]);
    const float sg = sigmoid_f(g[j]);
    du[j] = d * g[j] * sg;
    dg[j] = d * u[j] * sg * (1.f + g[j] * (1.f - sg));
  }
  *reinterpret_cast<uint32_t*>(dgp) = pack_bf16x2(dg[0], dg[1]);
  *reinterpret_cast<uint32_t*>(dup) = pack_bf16x2(du[0], du[1]);
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

// tile index -> coordinates.  Dense: M fastest (consecutive CTAs share the B tile in L2).  Grouped forward/dgrad: per-group row
// ranges [offsets[g], offsets[g+1]) (128-row aligned by the router), B rows offset by g*b_group_rows.  Grouped wgrad: each group owns
// the reduction range [offsets[g], offsets[g+1]) and its own D.
__device__ __forceinline__ bool get_tile(const GemmParams& p, int t, Tile& o) {
  const int BN = p.bn;
  const int num_n = (p.N + BN - 1) / BN;
  if (p.offsets == nullptr) {
    const int num_m = (p.M + BM - 1) / BM;
    const int mn = num_m * num_n, nk = (p.K + BK - 1) / BK;
    if (t >= mn * p.splits) return false;
    const int ks = t / mn, r = t % mn;                       // output tiles fastest: concurrent CTAs hit different D tiles
    const int per = (nk + p.splits - 1) / p.splits;
    o.m0 = (r % num_m) * BM; o.n0 = (r / num_m) * BN; o.kb0 = ks * per; o.kb1 = min(nk, o.kb0 + per); o.group = 0; o.m_end = p.M;
    return true;
  }
  if (p.wgrad_grouped) {
    const int num_m = (p.M + BM - 1) / BM;
    const int per = num_m * num_n;
    const int g = t / per;
    if (g >= p.groups) return false;
    const int r = t % per;
    o.m0 = (r % num_m) * BM; o.n0 = (r / num_m) * BN; o.group = g; o.m_end = p.M;
    o.kb0 = p.offsets[g] / BK; o.kb1 = (p.offsets[g + 1] + BK - 1) / BK;
    return true;
  }
  int base = 0;
  for (int g = 0; g < p.groups; ++g) {
    const int r0 = p.offsets[g], r1 = p.offsets[g + 1];
    const int nm = (r1 - r0 + BM - 1) / BM;
    const int cnt = nm * num_n;
    if (t < base + cnt) {
      const int r = t - base;
      o.m0 = r0 + (r % nm) * BM; o.n0 = (r / nm) * BN; o.kb0 = 0; o.kb1 = (p.K + BK - 1) / BK; o.group = g; o.m_end = r1;
      return true;
    }
    base += cnt;
  }
  return false;
}

template <int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void mma_kblock(float* acc, uint32_t sa, uint32_t sb, uint32_t accumulate) {
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint64_t da = A_MN ? gmma_desc(sa + k * 2048, BK * 128, 1024) : gmma_desc(sa + k * 32, 16, 1024);
    const uint64_t db = B_MN ? gmma_desc(sb + k * 2048, BK * 128, 1024) : gmma_desc(sb + k * 32, 16, 1024);
    const uint32_t acc_in = (k > 0) ? 1u : accumulate;
    if constexpr (BN == 256) wgmma_ss_n256<A_MN, B_MN>(acc, da, db, acc_in);
    else wgmma_ss_n128<A_MN, B_MN>(acc, da, db, acc_in);
  }
}

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const GemmParams p_in) {
  const GemmParams p = effective_extents(p_in);
  constexpr int STAGES = Cfg<BN>::STAGES, STAGE_BYTES = Cfg<BN>::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);   // SW128 needs 1024 B
  const int wg = threadIdx.x >> 7;

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
      Tile t;
      for (int ti = blockIdx.x; get_tile(p, ti, t); ti += gridDim.x) {
        const int b_row0 = (int)(t.group * p.b_group_rows);
        for (int kb = t.kb0; kb < t.kb1; ++kb) {
          mbar_wait_bounded(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          if (!A_MN) {
            tma_load_2d(sa, &tma_a, kb * BK, t.m0, &full_bar[stage]);                      // box (64 k, 128 rows)
          } else {
#pragma unroll
            for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * (BK * 128), &tma_a, t.m0 + 64 * j, kb * BK, &full_bar[stage]);   // box (64 mn, 64 k)
          }
          if (!B_MN && p.swiglu) {                                                         // box (64 k, 128 rows): gate rows, then the matching up rows
            tma_load_2d(sb, &tma_b, kb * BK, b_row0 + t.n0, &full_bar[stage]);
            tma_load_2d(sb + 128 * 128, &tma_b, kb * BK, b_row0 + p.swiglu_I + t.n0, &full_bar[stage]);
          } else if (!B_MN) {
            tma_load_2d(sb, &tma_b, kb * BK, b_row0 + t.n0, &full_bar[stage]);             // box (64 k, BN rows)
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * (BK * 128), &tma_b, t.n0 + 64 * j, b_row0 + kb * BK, &full_bar[stage]);
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
  float acc[BN / 2];
  uint32_t stage = 0, phase = 0;
  Tile t;
  for (int ti = blockIdx.x; get_tile(p, ti, t); ti += gridDim.x) {
    uint32_t prev = 0;
    for (int kb = t.kb0; kb < t.kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + c * (64 * 128), sb = smem_u32(smem + stage * STAGE_BYTES + A_STAGE_BYTES);
      wgmma_fence();
      mma_kblock<BN, A_MN, B_MN>(acc, sa, sb, kb > t.kb0 ? 1u : 0u);
      wgmma_commit();
      if (kb > t.kb0) {                                    // the previous k-block's MMAs are done: hand its stage back
        wgmma_wait<1>();
        if (wg_leader) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    const bool empty_k = t.kb1 <= t.kb0;                   // grouped wgrad of an expert with no rows / empty dynamic reduction: zero
    wgmma_wait<0>();                                       // on every path: a conditional wait makes ptxas drain after each MMA (C7517)
    if (!empty_k && wg_leader) mbar_arrive(&empty_bar[prev]);
    reg_fence<BN / 2>(acc);

    // accumulator fragment: register 4i + 2h + e holds row 16w + lane/4 + 8h, column 8i + 2(lane%4) + e of this warpgroup's 64 x BN block
    const int row0 = t.m0 + c * 64 + w * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const int64_t goff = p.wgrad_grouped ? t.group * p.d_group_stride : 0;
    if (BN == 256 && p.swiglu) {
      // accumulator columns [0,128) = gate, [128,256) = up of the same 128 act columns
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int col = t.n0 + 8 * i + cq;
        if (col >= p.N) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          if (row >= t.m_end) continue;
          __nv_bfloat16* drow = p.D + (int64_t)row * p.ldd;
          __nv_bfloat16* h1row = p.H1 ? p.H1 + (int64_t)row * p.ld_h1 : nullptr;
          swiglu_store2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], acc[4 * (i + 16) + 2 * h], acc[4 * (i + 16) + 2 * h + 1], drow + col,
                        h1row ? h1row + col : nullptr, h1row ? h1row + p.swiglu_I + col : nullptr);
        }
      }
      continue;
    }
    if (!p.rope_cos && !p.silu_bwd && !p.D32 && !p.beta && !p.R && !p.dbg_nostore && (reinterpret_cast<uintptr_t>(p.D) & 15) == 0) {
      // plain bf16 output (+bias): the four lanes of a quad trade their packed column pairs so that each stores one 16-byte block of
      // 8 columns -- a quad writes 64 contiguous bytes of a row per instruction instead of 16, with a quarter of the store instructions
      const int q = lane & 3;
#pragma unroll
      for (int k = 0; k < BN / 32; ++k) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t wd[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int col = t.n0 + 8 * (4 * k + j) + cq;
            float f0 = empty_k ? 0.f : acc[4 * (4 * k + j) + 2 * h], f1 = empty_k ? 0.f : acc[4 * (4 * k + j) + 2 * h + 1];
            if (p.bias && col < p.N) bias2(p.bias + col, f0, f1);
            wd[j] = pack_bf16x2(f0, f1);
          }
          quad_transpose(wd, q);
          const int row = row0 + 8 * h, col8 = t.n0 + 8 * (4 * k + q);
          if (row < t.m_end && col8 < p.N)                 // N % 8 == 0: a block of 8 columns is in or out as a whole
            *reinterpret_cast<uint4*>(p.D + goff + (int64_t)row * p.ldd + col8) = make_uint4(wd[0], wd[1], wd[2], wd[3]);
        }
      }
      continue;
    }
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int col8 = t.n0 + 8 * i, col = col8 + cq;
      if (p.rope_cos && col8 < p.rope_cols) {
        // q / k head columns: the first half of a head is processed together with its partner half a head further on (same thread)
        const int hoff = col8 % p.rope_hd, half = p.rope_hd >> 1;
        if (hoff >= half) continue;                                     // done with its partner
        const int ip = (half == 32) ? i + 4 : i + 8;
        if (ip >= BN / 8) continue;                                     // (a head never straddles a tile: tiles start at multiples of 128)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          if (row >= t.m_end) continue;
          float x20, x21;
          if (half == 32) { x20 = acc[4 * ((i + 4) % (BN / 8)) + 2 * h]; x21 = acc[4 * ((i + 4) % (BN / 8)) + 2 * h + 1]; }
          else { x20 = acc[4 * ((i + 8) % (BN / 8)) + 2 * h]; x21 = acc[4 * ((i + 8) % (BN / 8)) + 2 * h + 1]; }
          const int64_t pp = __ldg(p.rope_pos + row);
          __nv_bfloat16* drow = p.D + (int64_t)row * p.ldd;
          rope_store2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1], x20, x21, p.bias ? p.bias + col : nullptr, p.bias ? p.bias + col + half : nullptr,
                      p.rope_cos + pp * p.rope_hd + hoff + cq, p.rope_sin + pp * p.rope_hd + hoff + cq, drow + col, drow + col + half);
        }
        continue;
      }
      if (col >= p.N || p.dbg_nostore) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        if (row >= t.m_end) continue;
        float f0 = empty_k ? 0.f : acc[4 * i + 2 * h], f1 = empty_k ? 0.f : acc[4 * i + 2 * h + 1];
        if (p.bias) bias2(p.bias + col, f0, f1);
        if (p.silu_bwd) {
          const __nv_bfloat16* gurow = p.GU + (int64_t)row * p.ld_gu;
          __nv_bfloat16* drow = p.D + (int64_t)row * p.ldd;
          silu_bwd_store2(f0, f1, gurow + col, gurow + p.N + col, drow + col, drow + p.N + col);
        } else if (p.D32) {
          float* d32 = p.D32 + goff + (int64_t)row * p.ldd + col;
          if (p.splits > 1) { atomicAdd(d32, f0); atomicAdd(d32 + 1, f1); }
          else { float2 o = *reinterpret_cast<float2*>(d32); o.x += f0; o.y += f1; *reinterpret_cast<float2*>(d32) = o; }
        } else {
          uint32_t* o = reinterpret_cast<uint32_t*>(p.D + goff + (int64_t)row * p.ldd + col);
          if (p.beta) { const uint32_t old = *o; f0 += bf16lo(old); f1 += bf16hi(old); }
          if (p.R) {
            const uint32_t rr = __ldg(reinterpret_cast<const uint32_t*>(p.R + (int64_t)row * p.ld_r + col));
            f0 = bf16_round(f0) + bf16lo(rr); f1 = bf16_round(f1) + bf16hi(rr);
          }
          *o = pack_bf16x2(f0, f1);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
template <int BN, bool A_MN, bool B_MN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int tiles_upper, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    LMOD_CUDA_OK(cudaFuncSetAttribute(gemm_wgmma_kernel<BN, A_MN, B_MN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM));
    attr = true;
  }
  int grid = lmod_num_sms();
  if (tiles_upper < grid) grid = tiles_upper;
  if (grid < 1) grid = 1;
  gemm_wgmma_kernel<BN, A_MN, B_MN><<<grid, GEMM_THREADS, Cfg<BN>::SMEM, st>>>(ta, tb, p);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

template <int BN>
int dispatch_bn(bool a_mn, bool b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int tiles, cudaStream_t st) {
  if (!a_mn && !b_mn) return launch<BN, false, false>(ta, tb, p, tiles, st);
  if (!a_mn && b_mn) return launch<BN, false, true>(ta, tb, p, tiles, st);
  if (a_mn && b_mn) return launch<BN, true, true>(ta, tb, p, tiles, st);
  return launch<BN, true, false>(ta, tb, p, tiles, st);
}
int dispatch(bool a_mn, bool b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int tiles, cudaStream_t st) {
  return p.bn == 256 ? dispatch_bn<256>(a_mn, b_mn, ta, tb, p, tiles, st) : dispatch_bn<128>(a_mn, b_mn, ta, tb, p, tiles, st);
}
// 256-wide tiles unless that tiling cannot fill the machine ~1.5 times over
int pick_bn(int64_t m_tiles, int64_t N) {
  const int64_t t256 = m_tiles * ((N + 255) / 256);
  return (t256 >= (int64_t)lmod_num_sms() * 3 / 2 || N <= 128) ? 256 : 128;
}

}  // namespace

// D[M,N] = A * B^T.  a_mn_major = 0: A stored [M,K] (row stride lda) ; 1: A stored [K,M].  b_mn_major = 0: B stored [N,K] ; 1: B stored [K,N].
// epilogue bit 0: D = bf16(D + acc) ;  d_f32_accum != null: fp32 D32 += acc (ldd applies to it) instead of the bf16 output;
// epilogue bit 1: retired (the fused SwiGLU forward is lmod_gemm_swiglu);
// epilogue bits 8..: split-K factor (fp32 atomic accumulation into D32, which the caller zero-initialises).
struct RopeArgs { const void* cos; const void* sin; const int64_t* pos; int hd; int cols; };
struct ResidArgs { const void* R; int64_t ld_r; };

static int gemm_dense(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major, void* D, int64_t ldd,
                      int64_t M, int64_t N, int64_t K, const void* bias, int epilogue, float* d_f32_accum,
                      const int32_t* m_rows_dev, const int32_t* k_rows_dev, void* stream, const RopeArgs* rope, const ResidArgs* resid = nullptr) {
  LMOD_CHECK_ARG(A && B && (D || d_f32_accum) && M > 0 && N > 0 && K > 0, "lmod_gemm_bf16: null pointer or empty problem");
  LMOD_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ldd % 8 == 0 && N % 8 == 0 && ((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0) &&
                 (!D || (uintptr_t)D % 16 == 0), "lmod_gemm_bf16: strides / N must be multiples of 8 elements and pointers 16-byte aligned (TMA)");
  CUtensorMap ta, tb;
  int rc;
  const int splits_req = (epilogue >> 8) > 1 ? (epilogue >> 8) : 1;
  LMOD_CHECK_ARG(!(epilogue & 2), "lmod_gemm_bf16: epilogue bit 1 is retired -- the fused SwiGLU forward is lmod_gemm_swiglu");
  const int BN = pick_bn(((M + BM - 1) / BM) * splits_req, N);
  if (!a_mn_major) rc = make_map(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
  else rc = make_map(&ta, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, BK);
  if (rc) return rc;
  if (!b_mn_major) rc = make_map(&tb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, BN);
  else rc = make_map(&tb, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, BK);
  if (rc) return rc;
  GemmParams p = {};
  p.D = (__nv_bfloat16*)D; p.bias = (const __nv_bfloat16*)bias; p.D32 = d_f32_accum; p.ldd = ldd;
  p.M = (int)M; p.N = (int)N; p.K = (int)K; p.beta = epilogue & 1; p.offsets = nullptr; p.groups = 1; p.bn = BN;
  p.dbg_nostore = getenv("LMOD_GEMM_NOSTORE") ? 1 : 0;
  p.splits = (epilogue >> 8) > 1 ? (epilogue >> 8) : 1;
  p.m_dev = m_rows_dev; p.k_dev = k_rows_dev;
  if (resid) { p.R = (const __nv_bfloat16*)resid->R; p.ld_r = resid->ld_r; }
  if (rope) { p.rope_cos = (const __nv_bfloat16*)rope->cos; p.rope_sin = (const __nv_bfloat16*)rope->sin; p.rope_pos = rope->pos; p.rope_hd = rope->hd; p.rope_cols = rope->cols; }
  LMOD_CHECK_ARG(p.splits == 1 || d_f32_accum, "lmod_gemm_bf16: split-K needs the fp32 accumulate output");
  const int tiles = (int)(((M + BM - 1) / BM) * ((N + BN - 1) / BN)) * p.splits;
  return dispatch(a_mn_major != 0, b_mn_major != 0, ta, tb, p, tiles, (cudaStream_t)stream);
}

extern "C" int lmod_gemm_bf16_dyn(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major, void* D, int64_t ldd,
                                  int64_t M, int64_t N, int64_t K, const void* bias, int epilogue, float* d_f32_accum,
                                  const int32_t* m_rows_dev, const int32_t* k_rows_dev, void* stream) {
  return gemm_dense(A, lda, a_mn_major, B, ldb, b_mn_major, D, ldd, M, N, K, bias, epilogue, d_f32_accum, m_rows_dev, k_rows_dev, stream, nullptr);
}

// q|k|v projection with the rotary embedding applied in the GEMM epilogue (Qwen2Attention: q/k/v_proj + apply_rotary_pos_emb,
// modeling_qwen2.py:678-691,159-184): D[M, (nh+2nkv)*hd] = A W^T + bias, then every q and k head rotated with cos / sin [max_pos, hd]
// (bf16) at position_ids[row]; v columns untouched.  Bit-identical to lmod_gemm_bf16 + lmod_rope.  hd in {64, 128}.
extern "C" int lmod_gemm_qkv_rope(const void* A, int64_t lda, const void* W, int64_t ldb, const void* bias, void* D, int64_t ldd, int64_t M,
                                  int64_t K, int nh, int nkv, int hd, const void* cos_table, const void* sin_table,
                                  const int64_t* position_ids, void* stream) {
  LMOD_CHECK_ARG(cos_table && sin_table && position_ids && nh > 0 && nkv > 0, "lmod_gemm_qkv_rope: null pointer");
  LMOD_CHECK_ARG(hd == 64 || hd == 128, "lmod_gemm_qkv_rope: head_dim %d not fused (64 and 128 are; use lmod_gemm_bf16 + lmod_rope)", hd);
  RopeArgs r = {cos_table, sin_table, position_ids, hd, (nh + nkv) * hd};
  return gemm_dense(A, lda, 0, W, ldb, 0, D, ldd, M, (int64_t)(nh + 2 * nkv) * hd, K, bias, 0, nullptr, nullptr, nullptr, stream, &r);
}

// D[M,N] = bf16( bf16(A W^T + bias) + R ): a projection whose output goes straight into the residual stream (o_proj / down_proj of
// Qwen2DecoderLayer, modeling_qwen2.py:796,808; out_proj / fc2 of the CLIP encoder layers).  Bit-identical to lmod_gemm_bf16 followed by
// lmod_add.  D may alias R (in-place update of the stream: every element is read and written by the same thread).
extern "C" int lmod_gemm_residual(const void* A, int64_t lda, const void* W, int64_t ldb, const void* bias, const void* R, int64_t ld_r,
                                  void* D, int64_t ldd, int64_t M, int64_t N, int64_t K, void* stream) {
  LMOD_CHECK_ARG(R && D && ld_r % 8 == 0 && ((uintptr_t)R % 16 == 0), "lmod_gemm_residual: residual pointer / stride (16-byte rows)");
  ResidArgs r = {R, ld_r};
  return gemm_dense(A, lda, 0, W, ldb, 0, D, ldd, M, N, K, bias, 0, nullptr, nullptr, nullptr, stream, nullptr, &r);
}

extern "C" int lmod_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major, void* D, int64_t ldd,
                              int64_t M, int64_t N, int64_t K, const void* bias, int epilogue, float* d_f32_accum, void* stream) {
  return lmod_gemm_bf16_dyn(A, lda, a_mn_major, B, ldb, b_mn_major, D, ldd, M, N, K, bias, epilogue, d_f32_accum, nullptr, nullptr, stream);
}

// ---- fused SwiGLU forward / backward (Qwen2MLP, modeling_qwen2.py:199-200; DeepSpeed Experts of the sparse layers) ----------------------
// act[M, I] = bf16(bf16(silu(A W_g^T)) * (A W_u^T)) with W_gu = [W_g ; W_u] stored [2I, K] exactly as the checkpoint holds it; h1 (optional,
// [M, 2I]) receives the bf16 pre-activations for the backward.  I % 128 == 0.
static int swiglu_common(const void* A, int64_t lda, const void* W, int64_t ldb, void* act, int64_t ld_act, void* h1, int64_t ld_h1,
                         const int32_t* offsets, int G, int64_t M, int64_t I, int64_t K, cudaStream_t st) {
  LMOD_CHECK_ARG(A && W && act && M > 0 && I > 0 && K > 0, "lmod_gemm_swiglu: null pointer or empty problem");
  LMOD_CHECK_ARG(I % 128 == 0, "lmod_gemm_swiglu: intermediate size %lld is not a multiple of 128 (use GEMM + lmod_silu_mul_fwd)", (long long)I);
  LMOD_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ld_act % 8 == 0 && (!h1 || ld_h1 % 8 == 0) && ((uintptr_t)A % 16 == 0) && ((uintptr_t)W % 16 == 0) &&
                 ((uintptr_t)act % 16 == 0) && (!h1 || (uintptr_t)h1 % 16 == 0), "lmod_gemm_swiglu: strides must be multiples of 8 elements, pointers 16-byte aligned");
  CUtensorMap ta, tb;
  int rc;
  GemmParams p = {};
  p.D = (__nv_bfloat16*)act; p.ldd = ld_act; p.M = (int)M; p.N = (int)I; p.K = (int)K; p.splits = 1; p.groups = G > 0 ? G : 1;
  p.swiglu = 1; p.swiglu_I = (int)I; p.H1 = (__nv_bfloat16*)h1; p.ld_h1 = ld_h1; p.bn = 128;     // tile enumeration: 128 act columns per tile
  rc = make_map(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
  if (rc) return rc;
  rc = make_map(&tb, W, (uint64_t)K, (uint64_t)((offsets ? G : 1) * 2 * I), (uint64_t)ldb, BK, 128);
  if (rc) return rc;
  int tiles;
  if (offsets) {
    p.offsets = offsets; p.b_group_rows = 2 * I;
    tiles = (int)(((M + BM - 1) / BM + G) * (I / 128));
  } else {
    tiles = (int)(((M + BM - 1) / BM) * (I / 128));
  }
  return launch<256, false, false>(ta, tb, p, tiles, st);
}

extern "C" int lmod_gemm_swiglu(const void* A, int64_t lda, const void* W_gu, int64_t ldb, void* act, int64_t ld_act, void* h1, int64_t ld_h1,
                                int64_t M, int64_t I, int64_t K, void* stream) {
  return swiglu_common(A, lda, W_gu, ldb, act, ld_act, h1, ld_h1, nullptr, 0, M, I, K, (cudaStream_t)stream);
}

// grouped form on compact expert rows: A [max_rows, K], W_gu [G, 2I, K], rows of group g = [offsets[g], offsets[g+1]) (128-aligned)
extern "C" int lmod_grouped_gemm_swiglu(const void* A, int64_t lda, const void* W_gu, int64_t ldb, void* act, int64_t ld_act, void* h1,
                                        int64_t ld_h1, const int32_t* offsets, int G, int64_t max_rows, int64_t I, int64_t K, void* stream) {
  LMOD_CHECK_ARG(offsets && G >= 1 && G <= MAX_GROUPS, "lmod_grouped_gemm_swiglu: bad group arguments");
  return swiglu_common(A, lda, W_gu, ldb, act, ld_act, h1, ld_h1, offsets, G, max_rows, I, K, (cudaStream_t)stream);
}

// backward of the fused MLP input: dh1[M, 2I] = silu_mul_bwd(dY W_dn, h1) computed in the epilogue of the dgrad GEMM dY [M, K=H] x W_dn [K, I]
// (W_dn as stored: [H, I] = MN-major B).  Grouped form: W_dn [G, K, I].
static int silu_bwd_common(const void* dY, int64_t lda, const void* W, int64_t ldb, const void* h1, int64_t ld_h1, void* dh1, int64_t ld_dh1,
                           const int32_t* offsets, int G, int64_t M, int64_t I, int64_t K, cudaStream_t st) {
  LMOD_CHECK_ARG(dY && W && h1 && dh1 && M > 0 && I > 0 && K > 0 && I % 8 == 0, "lmod_gemm_silu_bwd: bad arguments");
  LMOD_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ld_h1 % 8 == 0 && ld_dh1 % 8 == 0 && ((uintptr_t)dY % 16 == 0) && ((uintptr_t)W % 16 == 0) &&
                 ((uintptr_t)h1 % 16 == 0) && ((uintptr_t)dh1 % 16 == 0), "lmod_gemm_silu_bwd: strides must be multiples of 8 elements, pointers 16-byte aligned");
  CUtensorMap ta, tb;
  int rc;
  GemmParams p = {};
  p.D = (__nv_bfloat16*)dh1; p.ldd = ld_dh1; p.M = (int)M; p.N = (int)I; p.K = (int)K; p.splits = 1; p.groups = G > 0 ? G : 1;
  p.silu_bwd = 1; p.GU = (const __nv_bfloat16*)h1; p.ld_gu = ld_h1;
  const int BN = pick_bn((M + BM - 1) / BM, I);
  p.bn = BN;
  rc = make_map(&ta, dY, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
  if (rc) return rc;
  rc = make_map(&tb, W, (uint64_t)I, (uint64_t)((offsets ? G : 1) * K), (uint64_t)ldb, 64, BK);
  if (rc) return rc;
  int tiles;
  if (offsets) {
    p.offsets = offsets; p.b_group_rows = K;
    tiles = (int)(((M + BM - 1) / BM + G) * ((I + BN - 1) / BN));
  } else {
    tiles = (int)(((M + BM - 1) / BM) * ((I + BN - 1) / BN));
  }
  return dispatch(false, true, ta, tb, p, tiles, st);
}

extern "C" int lmod_gemm_silu_bwd(const void* dY, int64_t lda, const void* W_dn, int64_t ldb, const void* h1, int64_t ld_h1, void* dh1,
                                  int64_t ld_dh1, int64_t M, int64_t I, int64_t K, void* stream) {
  return silu_bwd_common(dY, lda, W_dn, ldb, h1, ld_h1, dh1, ld_dh1, nullptr, 0, M, I, K, (cudaStream_t)stream);
}

extern "C" int lmod_grouped_gemm_silu_bwd(const void* dY, int64_t lda, const void* W_dn, int64_t ldb, const void* h1, int64_t ld_h1, void* dh1,
                                          int64_t ld_dh1, const int32_t* offsets, int G, int64_t max_rows, int64_t I, int64_t K, void* stream) {
  LMOD_CHECK_ARG(offsets && G >= 1 && G <= MAX_GROUPS, "lmod_grouped_gemm_silu_bwd: bad group arguments");
  return silu_bwd_common(dY, lda, W_dn, ldb, h1, ld_h1, dh1, ld_dh1, offsets, G, max_rows, I, K, (cudaStream_t)stream);
}

// Grouped (per-expert) GEMM on rows [offsets[g], offsets[g+1]) (device array; boundaries must be multiples of 128 for mode 0/1, of 64 for
// mode 2).   mode 0 (forward):  D[rows_g, N] = A[rows_g, K] * B[g][N,K]^T            (A,D [R,*] ; B [G,N,K])
//            mode 1 (dgrad)  :  D[rows_g, N] = A[rows_g, K] * B[g][K,N]              (B stored [G,K,N], MN-major)
//            mode 2 (wgrad)  :  D[g][M,N] (+)= A[rows_g, M]^T * B[rows_g, N]         (A stored [R,M], B stored [R,N], both MN-major; reduction
//                                                                                      over the group's rows)
extern "C" int lmod_grouped_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, void* D, int64_t ldd, const int32_t* offsets, int G,
                                      int64_t max_rows, int64_t M, int64_t N, int64_t K, int mode, int epilogue, void* stream) {
  LMOD_CHECK_ARG(A && B && D && offsets && G >= 1 && G <= MAX_GROUPS && max_rows > 0, "lmod_grouped_gemm_bf16: bad arguments");
  LMOD_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ldd % 8 == 0 && N % 8 == 0, "lmod_grouped_gemm_bf16: strides / N must be multiples of 8");
  CUtensorMap ta, tb;
  GemmParams p = {};
  p.D = (__nv_bfloat16*)D; p.ldd = ldd; p.beta = epilogue & 1; p.offsets = offsets; p.groups = G; p.splits = 1;
  int rc, tiles;
  const int BN = (mode == 2) ? pick_bn(G * ((M + BM - 1) / BM), N) : pick_bn((max_rows + BM - 1) / BM, N);
  p.bn = BN;
  if (mode == 0 || mode == 1) {
    rc = make_map(&ta, A, (uint64_t)K, (uint64_t)max_rows, (uint64_t)lda, BK, BM);
    if (rc) return rc;
    if (mode == 0) { rc = make_map(&tb, B, (uint64_t)K, (uint64_t)(G * N), (uint64_t)ldb, BK, BN); p.b_group_rows = N; }
    else { rc = make_map(&tb, B, (uint64_t)N, (uint64_t)(G * K), (uint64_t)ldb, 64, BK); p.b_group_rows = K; }
    if (rc) return rc;
    p.M = (int)max_rows; p.N = (int)N; p.K = (int)K;
    tiles = (int)(((max_rows + BM - 1) / BM + G) * ((N + BN - 1) / BN));
    return dispatch(false, mode == 1, ta, tb, p, tiles, (cudaStream_t)stream);
  }
  LMOD_CHECK_ARG(mode == 2, "lmod_grouped_gemm_bf16: mode must be 0, 1 or 2");
  rc = make_map(&ta, A, (uint64_t)M, (uint64_t)max_rows, (uint64_t)lda, 64, BK);
  if (rc) return rc;
  rc = make_map(&tb, B, (uint64_t)N, (uint64_t)max_rows, (uint64_t)ldb, 64, BK);
  if (rc) return rc;
  p.M = (int)M; p.N = (int)N; p.K = (int)max_rows; p.wgrad_grouped = 1; p.d_group_stride = M * ldd; p.b_group_rows = 0;
  tiles = (int)(G * ((M + BM - 1) / BM) * ((N + BN - 1) / BN));
  return dispatch(true, true, ta, tb, p, tiles, (cudaStream_t)stream);
}
