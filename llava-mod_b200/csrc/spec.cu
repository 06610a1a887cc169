// spec.cu -- the acceptance step of assisted (speculative) decoding on sm_90a.
//
// Replaces HF's assisted-generation acceptance (generation/utils.py: _assisted_decoding's greedy match of the candidate tokens against
// the target's argmax, and _speculative_sampling for do_sample): the verify logits of k + 1 positions per sequence are read once on the
// device, the accepted count and the next token are written there, and both KV caches are rolled back there, so a round needs one
// device-to-host read.
//
// One CTA per sequence, rows processed in order, each row streamed by the whole CTA:
//   greedy  : a_j = argmax of target row j (first index on ties, as torch.argmax); accept d_{j+1} while d_{j+1} == a_j; next = a_{n_acc}
//   sampling: p_j, q_j fp32 softmaxes of target row j and draft row j; accept d_{j+1} while u_j * q_j(d_{j+1}) <= p_j(d_{j+1}); on the
//             first rejection sample normalize(max(0, p_j - q_j)), after k acceptances sample p_k, both by inverse CDF with u_k
// Inverse CDF: the weights are summed in a fixed order (tiles of SA_THREADS * SA_ITEMS ids, a block scan per tile, tile totals added in
// order), the token is the first id whose running sum exceeds u * total, so the result is a function of the logits and u only.
// Ids at or past V_d have draft probability 0; ids at or past V_t have target probability 0.
#include <climits>
#include "common.cuh"

namespace {

constexpr int SA_THREADS = 1024;
constexpr int SA_ITEMS = 4;                             // consecutive ids per thread per tile
constexpr int SA_TILE = SA_THREADS * SA_ITEMS;
constexpr int SA_WARPS = SA_THREADS / 32;

struct SaShared {
  float red[SA_WARPS];
  float red2[SA_WARPS];
  int ired[SA_WARPS];
};

// (max, sum of exp) of a row, in one pass: per-thread online softmax, then a fixed-order block combine
__device__ void row_stats(const float* x, int V, SaShared& sh, float& m_out, float& z_out) {
  float m = -INFINITY, z = 0.f;
  for (int i = threadIdx.x; i < V; i += SA_THREADS) {
    const float v = x[i];
    if (v > m) {
      z = z * ex2f((m - v) * LOG2E_F);                  // m = -inf -> 0
      m = v;
    }
    if (v != -INFINITY) z += ex2f((v - m) * LOG2E_F);
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), z2 = __shfl_xor_sync(0xffffffffu, z, o);
    const float mn = fmaxf(m, m2);
    z = mn == -INFINITY ? 0.f : z * ex2f((m - mn) * LOG2E_F) + z2 * ex2f((m2 - mn) * LOG2E_F);
    m = mn;
  }
  __syncthreads();
  if (lane == 0) { sh.red[w] = m; sh.red2[w] = z; }
  __syncthreads();
  m = lane < SA_WARPS ? sh.red[lane] : -INFINITY;
  z = lane < SA_WARPS ? sh.red2[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), z2 = __shfl_xor_sync(0xffffffffu, z, o);
    const float mn = fmaxf(m, m2);
    z = mn == -INFINITY ? 0.f : z * ex2f((m - mn) * LOG2E_F) + z2 * ex2f((m2 - mn) * LOG2E_F);
    m = mn;
  }
  m_out = m;
  z_out = z;
}

// probability of id x under the softmax of row x_row (max m, sum z); 0 past the row's vocabulary or for an all -inf row
__device__ __forceinline__ float prob(const float* row, int V, float m, float z, int x) {
  if (x >= V || !(z > 0.f)) return 0.f;
  return ex2f((row[x] - m) * LOG2E_F) / z;
}

// first index of the row's maximum
__device__ int row_argmax(const float* x, int V, SaShared& sh) {
  float bv = -INFINITY;
  int bi = -1;
  for (int i = threadIdx.x; i < V; i += SA_THREADS) {
    const float v = x[i];
    if (bi < 0 || v > bv) { bv = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, bv, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    if (i2 >= 0 && (bi < 0 || v2 > bv || (v2 == bv && i2 < bi))) { bv = v2; bi = i2; }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) { sh.red[w] = bv; sh.ired[w] = bi; }
  __syncthreads();
  bv = lane < SA_WARPS ? sh.red[lane] : -INFINITY;
  bi = lane < SA_WARPS ? sh.ired[lane] : -1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, bv, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    if (i2 >= 0 && (bi < 0 || v2 > bv || (v2 == bv && i2 < bi))) { bv = v2; bi = i2; }
  }
  return bi;
}

// exclusive block scan of one float per thread; *total gets the tile's sum (the last thread's exclusive + own value)
__device__ float block_exclusive_scan(float v, SaShared& sh, float* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  __syncthreads();
  if (lane == 31) sh.red[w] = incl;
  __syncthreads();
  if (w == 0) {
    float s = sh.red[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    sh.red2[lane] = s;                                  // inclusive over warps
  }
  __syncthreads();
  const float excl = (w > 0 ? sh.red2[w - 1] : 0.f) + (incl - v);
  *total = sh.red2[SA_WARPS - 1];
  return excl;
}

// block minimum / maximum of an int (result broadcast)
__device__ int block_min_int(int v, SaShared& sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) sh.ired[w] = v;
  __syncthreads();
  v = lane < SA_WARPS ? sh.ired[lane] : INT_MAX;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ int block_max_int(int v, SaShared& sh) { return -block_min_int(-v, sh); }

// inverse-CDF sample over ids [0, V) of the weights w(x) >= 0 with uniform u in [0, 1): the first id whose running sum exceeds u * total.
// If rounding leaves no such id, the last id of positive weight; if every weight is 0, -1.
template <class W>
__device__ int sample_inverse_cdf(W w, int V, float u, SaShared& sh) {
  float total = 0.f;
  int last_pos = -1;
  for (int t0 = 0; t0 < V; t0 += SA_TILE) {
    const int x0 = t0 + threadIdx.x * SA_ITEMS;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < SA_ITEMS; ++i)
      if (x0 + i < V) {
        const float wi = w(x0 + i);
        s += wi;
        if (wi > 0.f) last_pos = x0 + i;
      }
    float tile;
    block_exclusive_scan(s, sh, &tile);
    total += tile;
  }
  last_pos = block_max_int(last_pos, sh);
  if (last_pos < 0) return -1;
  const float target = u * total;
  float run = 0.f;
  for (int t0 = 0; t0 < V; t0 += SA_TILE) {
    const int x0 = t0 + threadIdx.x * SA_ITEMS;
    float wl[SA_ITEMS], s = 0.f;
#pragma unroll
    for (int i = 0; i < SA_ITEMS; ++i) {
      wl[i] = x0 + i < V ? w(x0 + i) : 0.f;
      s += wl[i];
    }
    float tile;
    const float excl = block_exclusive_scan(s, sh, &tile);
    if (run + tile > target) {
      int cand = INT_MAX, lastp = -1;
      float c = 0.f;
#pragma unroll
      for (int i = 0; i < SA_ITEMS; ++i) {
        c += wl[i];
        if (wl[i] > 0.f) {
          lastp = x0 + i;
          if (cand == INT_MAX && run + (excl + c) > target) cand = x0 + i;
        }
      }
      cand = block_min_int(cand, sh);
      if (cand != INT_MAX) return cand;
      return block_max_int(lastp, sh);                   // the scan's rounding put the crossing past this tile's last id
    }
    run += tile;
  }
  return last_pos;
}

__global__ void __launch_bounds__(SA_THREADS) spec_accept_kernel(const float* __restrict__ tl, int V_t, const float* __restrict__ dl,
                                                                 int V_d, const int64_t* __restrict__ draft, const float* __restrict__ u,
                                                                 int k, int32_t* n_acc, int64_t* next, int32_t* len_t, int32_t* len_d) {
  __shared__ SaShared sh;
  const int b = blockIdx.x;
  const float* P = tl + (size_t)b * (k + 1) * V_t;
  const int64_t* d = draft + (size_t)b * k;
  int n = 0;
  int64_t tok = -1;
  if (u == nullptr) {                                   // greedy
    for (int j = 0; j <= k; ++j) {
      const int a = row_argmax(P + (size_t)j * V_t, V_t, sh);
      if (j < k && d[j] == a) { ++n; continue; }
      tok = a;
      break;
    }
  } else {
    const float* Q = dl + (size_t)b * k * V_d;
    const float* ub = u + (size_t)b * (k + 1);
    const float uk = ub[k];
    for (int j = 0; j < k; ++j) {
      const float* pr = P + (size_t)j * V_t;
      const float* qr = Q + (size_t)j * V_d;
      float mp, zp, mq, zq;
      row_stats(pr, V_t, sh, mp, zp);
      row_stats(qr, V_d, sh, mq, zq);
      const int64_t x = d[j];
      const float pd = x >= 0 && x < V_t ? prob(pr, V_t, mp, zp, (int)x) : 0.f;
      const float qd = x >= 0 && x < V_d ? prob(qr, V_d, mq, zq, (int)x) : 0.f;
      if (ub[j] * qd <= pd) { ++n; continue; }
      tok = sample_inverse_cdf([&](int y) { return fmaxf(0.f, prob(pr, V_t, mp, zp, y) - prob(qr, V_d, mq, zq, y)); }, V_t, uk, sh);
      if (tok < 0) tok = sample_inverse_cdf([&](int y) { return prob(pr, V_t, mp, zp, y); }, V_t, uk, sh);   // p == q in fp32
      break;
    }
    if (n == k) {                                       // every draft accepted: the bonus token from p_k
      const float* pr = P + (size_t)k * V_t;
      float mp, zp;
      row_stats(pr, V_t, sh, mp, zp);
      tok = sample_inverse_cdf([&](int y) { return prob(pr, V_t, mp, zp, y); }, V_t, uk, sh);
    }
  }
  if (threadIdx.x == 0) {
    n_acc[b] = n;
    next[b] = tok < 0 ? 0 : tok;
    if (len_t) len_t[b] -= k - n;
    if (len_d) len_d[b] -= k - n;
  }
}

}  // namespace

extern "C" int lmod_spec_accept(const float* target_logits, int64_t V_t, const float* draft_logits, int64_t V_d, const int64_t* draft_tokens,
                                const float* u, int64_t batch, int k, int32_t* n_acc, int64_t* next, int32_t* len_target,
                                int32_t* len_draft, void* stream) {
  LMOD_CHECK_ARG(target_logits && draft_tokens && n_acc && next && batch > 0 && batch < 65536 && k >= 1 && k <= 64 && V_t > 0 &&
                 V_t < (1 << 30), "lmod_spec_accept: bad arguments");
  LMOD_CHECK_ARG(!u || (draft_logits && V_d > 0 && V_d < (1 << 30)), "lmod_spec_accept: sampling needs the draft logits and V_d");
  spec_accept_kernel<<<(unsigned)batch, SA_THREADS, 0, (cudaStream_t)stream>>>(target_logits, (int)V_t, draft_logits, (int)V_d,
                                                                                draft_tokens, u, k, n_acc, next, len_target, len_draft);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
