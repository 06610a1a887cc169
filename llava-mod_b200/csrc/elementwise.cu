// elementwise.cu -- HBM-bound norm / rotary / activation / splice kernels of the Qwen2 + CLIP path.
//
// Reference call sites: Qwen2RMSNorm modeling_qwen2.py:105-110; apply_rotary_pos_emb :159-184;
// Qwen2MLP :199-200; projector GELU multimodal_projector/builder.py:57-61; CLIP LayerNorm / quick_gelu
// (transformers CLIPVisionModel via multimodal_encoder/clip_encoder.py:54); multimodal splice
// llava_arch.py:228-320.  All kernels use 16-byte vector accesses, fp32 math, bf16 I/O and reproduce the
// reference's intermediate bf16 roundings where the reference materialises a bf16 tensor.
#include "common.cuh"

namespace {

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  f[0] = bf16lo(u.x); f[1] = bf16hi(u.x); f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
  f[4] = bf16lo(u.z); f[5] = bf16hi(u.z); f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]); o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
  return o;
}

constexpr int NORM_THREADS = 128;

// y = w * bf16(x' * rstd),  x' = bf16(x + res) if res  (Qwen2RMSNorm; residual add of the decoder layer fused in)
__global__ void __launch_bounds__(NORM_THREADS) rmsnorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                                                                  const __nv_bfloat16* __restrict__ w, int H, float eps,
                                                                  __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ x_out,
                                                                  float* __restrict__ rstd_out) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int hv = H >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
  const uint4* rr = res ? reinterpret_cast<const uint4*>(res + row * H) : nullptr;
  uint4* xo = x_out ? reinterpret_cast<uint4*>(x_out + row * H) : nullptr;
  float ss = 0.f;
  for (int v = threadIdx.x; v < hv; v += NORM_THREADS) {
    float f[8];
    unpack8(xr[v], f);
    if (rr) {
      float g[8];
      unpack8(rr[v], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = bf16_round(f[j] + g[j]);
      if (xo) xo[v] = pack8(f);
    } else if (xo) {
      xo[v] = xr[v];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)H + eps);
  if (threadIdx.x == 0 && rstd_out) rstd_out[row] = rstd;
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  uint4* yr = reinterpret_cast<uint4*>(y + row * H);
  for (int v = threadIdx.x; v < hv; v += NORM_THREADS) {
    float f[8], wf[8];
    unpack8(xr[v], f);
    if (rr) {
      float g[8];
      unpack8(rr[v], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = bf16_round(f[j] + g[j]);
    }
    unpack8(wr[v], wf);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = wf[j] * bf16_round(f[j] * rstd);
    yr[v] = pack8(f);
  }
}

// Same, for rows that fit the CTA's registers (H <= 128 * 8 * VPT): x (+res) is read from HBM exactly once, kept packed in registers
// across the block reduction, and all loads of a thread are in flight together.
template <int VPT>
__global__ void __launch_bounds__(NORM_THREADS) rmsnorm_fwd_reg_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                                                                      const __nv_bfloat16* __restrict__ w, int H, float eps,
                                                                      __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ x_out,
                                                                      float* __restrict__ rstd_out) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int hv = H >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
  const uint4* rr = res ? reinterpret_cast<const uint4*>(res + row * H) : nullptr;
  uint4* xo = x_out ? reinterpret_cast<uint4*>(x_out + row * H) : nullptr;
  uint4 xv[VPT], rv[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * NORM_THREADS;
    xv[i] = make_uint4(0, 0, 0, 0); rv[i] = make_uint4(0, 0, 0, 0);
    if (v < hv) {
      xv[i] = ldg_nc_v4(xr + v);
      if (rr) rv[i] = ldg_nc_v4(rr + v);
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * NORM_THREADS;
    float f[8];
    unpack8(xv[i], f);
    if (rr) {
      float g[8];
      unpack8(rv[i], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = bf16_round(f[j] + g[j]);
      xv[i] = pack8(f);
    }
    if (xo && v < hv) xo[v] = xv[i];
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(f[j], f[j], ss);
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)H + eps);
  if (threadIdx.x == 0 && rstd_out) rstd_out[row] = rstd;
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  uint4* yr = reinterpret_cast<uint4*>(y + row * H);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * NORM_THREADS;
    if (v < hv) {
      float f[8], wf[8];
      unpack8(xv[i], f);
      unpack8(__ldg(wr + v), wf);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = wf[j] * bf16_round(f[j] * rstd);
      yr[v] = pack8(f);
    }
  }
}

// dx = rstd * (dy*w - xhat * mean(dy*w*xhat)) (+ dres)
__global__ void __launch_bounds__(NORM_THREADS) rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                                  const __nv_bfloat16* __restrict__ w, const float* __restrict__ rstd_in,
                                                                  const __nv_bfloat16* __restrict__ dres, int H,
                                                                  __nv_bfloat16* __restrict__ dx) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int hv = H >> 3;
  const uint4* dyr = reinterpret_cast<const uint4*>(dy + row * H);
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  const float rstd = rstd_in[row];
  float dot = 0.f;
  for (int v = threadIdx.x; v < hv; v += NORM_THREADS) {
    float a[8], b[8], c[8];
    unpack8(dyr[v], a); unpack8(xr[v], b); unpack8(wr[v], c);
#pragma unroll
    for (int j = 0; j < 8; ++j) dot = fmaf(a[j] * c[j], b[j] * rstd, dot);
  }
  dot = block_sum(dot, red) / (float)H;
  const uint4* dr = dres ? reinterpret_cast<const uint4*>(dres + row * H) : nullptr;
  uint4* dxr = reinterpret_cast<uint4*>(dx + row * H);
  for (int v = threadIdx.x; v < hv; v += NORM_THREADS) {
    float a[8], b[8], c[8], o[8];
    unpack8(dyr[v], a); unpack8(xr[v], b); unpack8(wr[v], c);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = rstd * (a[j] * c[j] - b[j] * rstd * dot);
    if (dr) {
      float g[8];
      unpack8(dr[v], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] += g[j];
    }
    dxr[v] = pack8(o);
  }
}

__global__ void __launch_bounds__(NORM_THREADS) layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                                    const __nv_bfloat16* __restrict__ b, int H, float eps,
                                                                    __nv_bfloat16* __restrict__ y) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int hv = H >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
  float s = 0.f;
  for (int v = threadIdx.x; v < hv; v += NORM_THREADS) {
    float f[8]; unpack8(xr[v], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += f[j];
  }
  const float mean = block_sum(s, red) / (float)H;
  float q = 0.f;
  for (int v = threadIdx.x; v < hv; v += NORM_THREADS) {
    float f[8]; unpack8(xr[v], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { float d = f[j] - mean; q = fmaf(d, d, q); }
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)H + eps);
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  const uint4* br = reinterpret_cast<const uint4*>(b);
  uint4* yr = reinterpret_cast<uint4*>(y + row * H);
  for (int v = threadIdx.x; v < hv; v += NORM_THREADS) {
    float f[8], wf[8], bf[8];
    unpack8(xr[v], f); unpack8(wr[v], wf); unpack8(br[v], bf);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = fmaf((f[j] - mean) * rstd, wf[j], bf[j]);
    yr[v] = pack8(f);
  }
}

// rotate-half RoPE in place.  cos/sin tables are the reference's bf16 cache rows ([P, hd], emb = cat(freqs, freqs)).
// forward:  o1 = bf16(bf16(x1*c) + bf16(-x2*s)) ; o2 = bf16(bf16(x2*c) + bf16(x1*s))   (modeling_qwen2.py:181-183 in bf16)
// backward: transpose rotation.
__global__ void rope_kernel(__nv_bfloat16* __restrict__ q, int64_t ld_q, int nh, __nv_bfloat16* __restrict__ k, int64_t ld_k, int nkv,
                            int hd, const __nv_bfloat16* __restrict__ cos_t, const __nv_bfloat16* __restrict__ sin_t,
                            const int64_t* __restrict__ pos, int64_t rows, int backward) {
  const int half = hd >> 1;
  const int per_row = (nh + nkv) * half;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= rows * per_row) return;
  const int64_t row = gid / per_row;
  int r = (int)(gid % per_row);
  const int head = r / half, i = r % half;
  __nv_bfloat16* base = (head < nh) ? (q + row * ld_q + (size_t)head * hd) : (k + row * ld_k + (size_t)(head - nh) * hd);
  const int64_t pp = pos[row];
  const float c = __bfloat162float(cos_t[pp * hd + i]), s = __bfloat162float(sin_t[pp * hd + i]);
  const float x1 = __bfloat162float(base[i]), x2 = __bfloat162float(base[i + half]);
  float o1, o2;
  if (!backward) {
    o1 = bf16_round(x1 * c) + bf16_round(-x2 * s);
    o2 = bf16_round(x2 * c) + bf16_round(x1 * s);
  } else {
    o1 = x1 * c + x2 * s;
    o2 = x2 * c - x1 * s;
  }
  base[i] = __float2bfloat16_rn(o1);
  base[i + half] = __float2bfloat16_rn(o2);
}

// vectorised form (hd % 16 == 0): one thread rotates 8 (x1, x2) pairs with 16-byte accesses
__global__ void __launch_bounds__(256) rope_vec_kernel(__nv_bfloat16* __restrict__ q, int64_t ld_q, int nh, __nv_bfloat16* __restrict__ k,
                                                      int64_t ld_k, int nkv, int hd, const __nv_bfloat16* __restrict__ cos_t,
                                                      const __nv_bfloat16* __restrict__ sin_t, const int64_t* __restrict__ pos, int64_t rows,
                                                      int backward) {
  const int half = hd >> 1, vph = half >> 3;
  const int per_row = (nh + nkv) * vph;
  const int64_t row = blockIdx.x;                               // grid: (rows, ceil(per_row / 256)) -- no 64-bit divisions
  const int r = (int)(blockIdx.y * blockDim.x + threadIdx.x);
  if (r >= per_row) return;
  const int head = r / vph, v = r % vph;
  __nv_bfloat16* base = (head < nh) ? (q + row * ld_q + (size_t)head * hd) : (k + row * ld_k + (size_t)(head - nh) * hd);
  const int64_t pp = pos[row];
  float c[8], s[8], x1[8], x2[8], o1[8], o2[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(cos_t + pp * hd) + v), c);
  unpack8(__ldg(reinterpret_cast<const uint4*>(sin_t + pp * hd) + v), s);
  uint4* p1 = reinterpret_cast<uint4*>(base) + v;
  uint4* p2 = reinterpret_cast<uint4*>(base + half) + v;
  unpack8(*p1, x1);
  unpack8(*p2, x2);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (!backward) {
      o1[j] = bf16_round(x1[j] * c[j]) + bf16_round(-x2[j] * s[j]);
      o2[j] = bf16_round(x2[j] * c[j]) + bf16_round(x1[j] * s[j]);
    } else {
      o1[j] = x1[j] * c[j] + x2[j] * s[j];
      o2[j] = x2[j] * c[j] - x1[j] * s[j];
    }
  }
  *p1 = pack8(o1);
  *p2 = pack8(o2);
}

// dW of RMSNorm: dw[h] += sum_rows bf16(dy[r,h] * xhat[r,h]),  xhat = bf16(x[r,h] * rstd[r])  (autograd of `weight * hidden_states.to(dtype)`,
// modeling_qwen2.py:110; needed when the norms train: dense-student distillation / full SFT).  Grid (H/256 column slabs, row chunks);
// a CTA keeps 8 column sums per thread over its rows, folds its 8 warps through shared memory and issues one fp32 red.add per column
// into the [H] workspace; rmsnorm_wgrad_finish_kernel rounds once and accumulates into the bf16 gradient buffer.
constexpr int NWG_ROWS_PER_CTA = 256;
__global__ void __launch_bounds__(256) rmsnorm_wgrad_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                                           const float* __restrict__ rstd, int64_t rows, int H, float* __restrict__ ws) {
  __shared__ float part[8][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v = blockIdx.x * 32 + lane;                          // 16-byte vector (8 columns) of this thread
  const int hv = H >> 3;
  const int64_t r0 = (int64_t)blockIdx.y * NWG_ROWS_PER_CTA;
  const int64_t r1 = min(rows, r0 + NWG_ROWS_PER_CTA);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (v < hv) {
    for (int64_t r = r0 + warp; r < r1; r += 8) {
      float d[8], xv[8];
      unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(dy + r * H) + v), d);
      unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(x + r * H) + v), xv);
      const float rs = rstd[r];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += bf16_round(d[j] * bf16_round(xv[j] * rs));
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[warp][lane * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;                                     // column within the 256-wide slab
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += part[w][c];
  const int col = blockIdx.x * 256 + c;
  if (col < H) atomicAdd(ws + col, t);
}
__global__ void rmsnorm_wgrad_finish_kernel(float* __restrict__ ws, int H, __nv_bfloat16* __restrict__ wgrad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H) return;
  wgrad[i] = __float2bfloat16(__bfloat162float(wgrad[i]) + bf16_round(ws[i]));
  ws[i] = 0.f;                                                   // the workspace is handed back zeroed
}

// dW of the token embedding (nn.Embedding backward behind the multimodal splice, llava_arch.py:262-274, then the bf16 accumulation
// into .grad): grad[t] = bf16(grad[t] + bf16(sum of the rows of token t)).  `order` lists the rows grouped by token id (a stable sort of
// src with the rows src < 0 last, built on the host with the splice plan).  The CTA at the first row of a token's run sums the run in
// fp32 in row order and rounds once, like the reference's fp32 backward; each token has one owner, so no atomics and the same bytes
// on every run.  Rows of image patches and padding (src < 0) add nothing.
constexpr int EMB_THREADS = 128;
__global__ void __launch_bounds__(EMB_THREADS) embed_grad_kernel(const __nv_bfloat16* __restrict__ dout, const int64_t* __restrict__ src,
                                                                const int64_t* __restrict__ order, int64_t n_rows, int H,
                                                                __nv_bfloat16* __restrict__ grad) {
  const int64_t i = blockIdx.x;
  const int64_t tok = src[order[i]];
  if (tok < 0 || (i > 0 && src[order[i - 1]] == tok)) return;   // padding / image row, or not the first row of its token's run
  int64_t end = i + 1;
  while (end < n_rows && src[order[end]] == tok) ++end;
  uint4* to = reinterpret_cast<uint4*>(grad + tok * H);
  for (int v = threadIdx.x; v < (H >> 3); v += EMB_THREADS) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int64_t j = i; j < end; ++j) {
      float f[8];
      unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(dout + order[j] * H) + v), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += f[k];
    }
    float g[8];
    unpack8(to[v], g);
#pragma unroll
    for (int k = 0; k < 8; ++k) g[k] += bf16_round(acc[k]);
    to[v] = pack8(g);
  }
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

// out = bf16( bf16(silu(g)) * u ),  gate_up = [rows, 2I] (gate | up)
__global__ void silu_mul_fwd_kernel(const __nv_bfloat16* __restrict__ gu, int64_t ld, int64_t rows, int I, __nv_bfloat16* __restrict__ out) {
  const int iv = I >> 3;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= rows * iv) return;
  int64_t row; int v;
  if (rows * iv < (int64_t)1 << 31) { const uint32_t g32 = (uint32_t)gid; row = g32 / (uint32_t)iv; v = (int)(g32 % (uint32_t)iv); }   // 32-bit divide
  else { row = gid / iv; v = (int)(gid % iv); }
  float g[8], u[8];
  unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(gu + row * ld) + v), g);
  unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(gu + row * ld + I) + v), u);
#pragma unroll
  for (int j = 0; j < 8; ++j) g[j] = bf16_round(g[j] * sigmoidf_(g[j])) * u[j];
  reinterpret_cast<uint4*>(out + row * I)[v] = pack8(g);
}
__global__ void silu_mul_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ gu, int64_t ld, int64_t rows,
                                    int I, __nv_bfloat16* __restrict__ dgu) {
  const int iv = I >> 3;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= rows * iv) return;
  int64_t row; int v;
  if (rows * iv < (int64_t)1 << 31) { const uint32_t g32 = (uint32_t)gid; row = g32 / (uint32_t)iv; v = (int)(g32 % (uint32_t)iv); }   // 32-bit divide
  else { row = gid / iv; v = (int)(gid % iv); }
  float g[8], u[8], d[8], dg[8], du[8];
  unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(gu + row * ld) + v), g);
  unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(gu + row * ld + I) + v), u);
  unpack8(ldg_nc_v4(reinterpret_cast<const uint4*>(dout + row * I) + v), d);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float sg = sigmoidf_(g[j]);
    du[j] = d[j] * g[j] * sg;
    dg[j] = d[j] * u[j] * sg * (1.f + g[j] * (1.f - sg));
  }
  reinterpret_cast<uint4*>(dgu + row * ld)[v] = pack8(dg);
  reinterpret_cast<uint4*>(dgu + row * ld + I)[v] = pack8(du);
}

// y = act(x + bias): act 0 = GELU(erf) (nn.GELU), 1 = quick_gelu x*sigmoid(1.702x), 2 = identity
__global__ void bias_act_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ bias, int64_t rows, int n, int act,
                                __nv_bfloat16* __restrict__ y) {
  const int nv = n >> 3;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= rows * nv) return;
  const int v = (int)(gid % nv);
  float f[8];
  unpack8(reinterpret_cast<const uint4*>(x)[gid], f);
  if (bias) {
    float b[8];
    unpack8(reinterpret_cast<const uint4*>(bias)[v], b);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = bf16_round(f[j] + b[j]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (act == 0) f[j] = 0.5f * f[j] * (1.f + erff(f[j] * 0.70710678118654752f));
    else if (act == 1) f[j] = f[j] * sigmoidf_(1.702f * f[j]);
  }
  reinterpret_cast<uint4*>(y)[gid] = pack8(f);
}
// dx = dy * gelu'(x)
__global__ void gelu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, int64_t nvec, __nv_bfloat16* __restrict__ dx) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= nvec) return;
  float d[8], f[8];
  unpack8(reinterpret_cast<const uint4*>(dy)[gid], d);
  unpack8(reinterpret_cast<const uint4*>(x)[gid], f);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float cdf = 0.5f * (1.f + erff(f[j] * 0.70710678118654752f));
    const float pdf = 0.3989422804014327f * __expf(-0.5f * f[j] * f[j]);
    d[j] = d[j] * (cdf + f[j] * pdf);
  }
  reinterpret_cast<uint4*>(dx)[gid] = pack8(d);
}
__global__ void add_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b, int64_t nvec, __nv_bfloat16* __restrict__ o) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= nvec) return;
  float x[8], y[8];
  unpack8(reinterpret_cast<const uint4*>(a)[gid], x);
  unpack8(reinterpret_cast<const uint4*>(b)[gid], y);
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] += y[j];
  reinterpret_cast<uint4*>(o)[gid] = pack8(x);
}

// multimodal splice: one warp per output row
__global__ void __launch_bounds__(256) splice_embed_kernel(const __nv_bfloat16* __restrict__ embed_w, const __nv_bfloat16* __restrict__ feats,
                                                          const int64_t* __restrict__ src, const int64_t* __restrict__ img, int64_t n_rows,
                                                          int H, int n_patches, __nv_bfloat16* __restrict__ out) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int64_t s = src[row], im = img[row];
  const uint4* from = nullptr;
  if (s >= 0) from = reinterpret_cast<const uint4*>(embed_w + s * H);
  else if (im >= 0) from = reinterpret_cast<const uint4*>(feats + (im * n_patches + (-1 - s)) * H);
  uint4* to = reinterpret_cast<uint4*>(out + row * H);
  const uint4 z = make_uint4(0, 0, 0, 0);
  for (int v = lane; v < (H >> 3); v += 32) to[v] = from ? ldg_nc_v4(from + v) : z;
}
__global__ void __launch_bounds__(256) splice_embed_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const int64_t* __restrict__ src,
                                                              const int64_t* __restrict__ img, int64_t n_rows, int H, int n_patches,
                                                              __nv_bfloat16* __restrict__ dfeats) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int64_t s = src[row], im = img[row];
  if (s >= 0 || im < 0) return;
  const uint4* from = reinterpret_cast<const uint4*>(dout + row * H);
  uint4* to = reinterpret_cast<uint4*>(dfeats + (im * n_patches + (-1 - s)) * H);
  for (int v = lane; v < (H >> 3); v += 32) to[v] = from[v];
}

}  // namespace

#define GRID1D(n, t) (unsigned)(((n) + (t)-1) / (t))

extern "C" int lmod_rmsnorm_fwd(const void* x, const void* res, const void* w, int64_t rows, int64_t H, float eps, void* y, void* x_out,
                                float* rstd, void* stream) {
  LMOD_CHECK_ARG(x && w && y && rows > 0 && H > 0 && H % 8 == 0, "lmod_rmsnorm_fwd: bad arguments (H %% 8 == 0 required)");
  const int hv = (int)(H / 8);
#define LMOD_RMS_REG(VPT)                                                                                                              \
  rmsnorm_fwd_reg_kernel<VPT><<<(unsigned)rows, NORM_THREADS, 0, (cudaStream_t)stream>>>(                                              \
      (const __nv_bfloat16*)x, (const __nv_bfloat16*)res, (const __nv_bfloat16*)w, (int)H, eps, (__nv_bfloat16*)y, (__nv_bfloat16*)x_out, rstd)
  if (hv <= NORM_THREADS) LMOD_RMS_REG(1);
  else if (hv <= 2 * NORM_THREADS) LMOD_RMS_REG(2);
  else if (hv <= 4 * NORM_THREADS) LMOD_RMS_REG(4);
  else if (hv <= 8 * NORM_THREADS) LMOD_RMS_REG(8);
  else
    rmsnorm_fwd_kernel<<<(unsigned)rows, NORM_THREADS, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)res,
                                                                                 (const __nv_bfloat16*)w, (int)H, eps, (__nv_bfloat16*)y,
                                                                                 (__nv_bfloat16*)x_out, rstd);
#undef LMOD_RMS_REG
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, int64_t rows, int64_t H,
                                void* dx, void* stream) {
  LMOD_CHECK_ARG(dy && x && w && rstd && dx && rows > 0 && H % 8 == 0, "lmod_rmsnorm_bwd: bad arguments");
  rmsnorm_bwd_kernel<<<(unsigned)rows, NORM_THREADS, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                                                               (const __nv_bfloat16*)w, rstd, (const __nv_bfloat16*)dres,
                                                                               (int)H, (__nv_bfloat16*)dx);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_rmsnorm_wgrad(const void* dy, const void* x, const float* rstd, int64_t rows, int64_t H, float* ws_zeroed, void* wgrad,
                                  void* stream) {
  LMOD_CHECK_ARG(dy && x && rstd && ws_zeroed && wgrad && rows > 0 && H > 0 && H % 8 == 0, "lmod_rmsnorm_wgrad: bad arguments (H %% 8 == 0 required)");
  const dim3 grid((unsigned)((H + 255) / 256), (unsigned)((rows + NWG_ROWS_PER_CTA - 1) / NWG_ROWS_PER_CTA));
  rmsnorm_wgrad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, rstd, rows, (int)H, ws_zeroed);
  LMOD_LAUNCH_OK();
  rmsnorm_wgrad_finish_kernel<<<(unsigned)((H + 255) / 256), 256, 0, (cudaStream_t)stream>>>(ws_zeroed, (int)H, (__nv_bfloat16*)wgrad);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_embed_grad(const void* dout, const int64_t* src, const int64_t* order, int64_t n_rows, int64_t H, void* grad,
                               void* stream) {
  LMOD_CHECK_ARG(dout && src && order && grad && n_rows > 0 && H > 0 && H % 8 == 0 && (uintptr_t)dout % 16 == 0 && (uintptr_t)grad % 16 == 0,
                 "lmod_embed_grad: bad arguments (H %% 8 == 0, 16-byte aligned buffers required)");
  embed_grad_kernel<<<(unsigned)n_rows, EMB_THREADS, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dout, src, order, n_rows, (int)H,
                                                                               (__nv_bfloat16*)grad);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_layernorm_fwd(const void* x, const void* w, const void* b, int64_t rows, int64_t H, float eps, void* y, void* stream) {
  LMOD_CHECK_ARG(x && w && b && y && rows > 0 && H % 8 == 0, "lmod_layernorm_fwd: bad arguments");
  layernorm_fwd_kernel<<<(unsigned)rows, NORM_THREADS, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w,
                                                                                 (const __nv_bfloat16*)b, (int)H, eps, (__nv_bfloat16*)y);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_rope(void* q, int64_t ld_q, int nh, void* k, int64_t ld_k, int nkv, int hd, const void* cos_table,
                         const void* sin_table, const int64_t* position_ids, int64_t rows, int backward, void* stream) {
  LMOD_CHECK_ARG(q && k && cos_table && sin_table && position_ids && rows > 0 && hd % 2 == 0, "lmod_rope: bad arguments");
  if (hd % 16 == 0 && ld_q % 8 == 0 && ld_k % 8 == 0 && ((uintptr_t)q % 16 == 0) && ((uintptr_t)k % 16 == 0)) {
    const int per_row = (nh + nkv) * (hd / 16);
    const int thr = per_row >= 256 ? 256 : ((per_row + 31) / 32 * 32);
    rope_vec_kernel<<<dim3((unsigned)rows, (unsigned)((per_row + thr - 1) / thr)), thr, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)q, ld_q, nh, (__nv_bfloat16*)k, ld_k, nkv, hd,
                                                                     (const __nv_bfloat16*)cos_table, (const __nv_bfloat16*)sin_table,
                                                                     position_ids, rows, backward);
    LMOD_LAUNCH_OK();
    return LMOD_OK;
  }
  const int64_t n = rows * (nh + nkv) * (hd / 2);
  rope_kernel<<<GRID1D(n, 256), 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)q, ld_q, nh, (__nv_bfloat16*)k, ld_k, nkv, hd,
                                                               (const __nv_bfloat16*)cos_table, (const __nv_bfloat16*)sin_table,
                                                               position_ids, rows, backward);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_silu_mul_fwd(const void* gate_up, int64_t ld, int64_t rows, int64_t I, void* out, void* stream) {
  LMOD_CHECK_ARG(gate_up && out && rows > 0 && I % 8 == 0 && ld % 8 == 0 && ld >= 2 * I, "lmod_silu_mul_fwd: bad arguments");
  silu_mul_fwd_kernel<<<GRID1D(rows * (I / 8), 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)gate_up, ld, rows, (int)I,
                                                                                    (__nv_bfloat16*)out);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_silu_mul_bwd(const void* dout, const void* gate_up, int64_t ld, int64_t rows, int64_t I, void* dgate_up, void* stream) {
  LMOD_CHECK_ARG(dout && gate_up && dgate_up && rows > 0 && I % 8 == 0 && ld % 8 == 0 && ld >= 2 * I, "lmod_silu_mul_bwd: bad arguments");
  silu_mul_bwd_kernel<<<GRID1D(rows * (I / 8), 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)gate_up,
                                                                                    ld, rows, (int)I, (__nv_bfloat16*)dgate_up);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_bias_act_fwd(const void* x, const void* bias, int64_t rows, int64_t n, int act, void* y, void* stream) {
  LMOD_CHECK_ARG(x && y && rows > 0 && n % 8 == 0 && act >= 0 && act <= 2, "lmod_bias_act_fwd: bad arguments");
  bias_act_kernel<<<GRID1D(rows * (n / 8), 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)bias, rows,
                                                                                (int)n, act, (__nv_bfloat16*)y);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_gelu_bwd(const void* dy, const void* x_pre, int64_t count, void* dx, void* stream) {
  LMOD_CHECK_ARG(dy && x_pre && dx && count > 0 && count % 8 == 0, "lmod_gelu_bwd: bad arguments");
  gelu_bwd_kernel<<<GRID1D(count / 8, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x_pre, count / 8,
                                                                           (__nv_bfloat16*)dx);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_add(const void* a, const void* b, int64_t count, void* out, void* stream) {
  LMOD_CHECK_ARG(a && b && out && count > 0 && count % 8 == 0, "lmod_add: bad arguments");
  add_kernel<<<GRID1D(count / 8, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)a, (const __nv_bfloat16*)b, count / 8,
                                                                      (__nv_bfloat16*)out);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_splice_embed(const void* embed_w, const void* feats, const int64_t* src, const int64_t* img_index, int64_t n_rows,
                                 int64_t H, int64_t n_patches, void* out, void* stream) {
  LMOD_CHECK_ARG(embed_w && src && img_index && out && n_rows > 0 && H % 8 == 0, "lmod_splice_embed: bad arguments");
  splice_embed_kernel<<<GRID1D(n_rows * 32, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)embed_w, (const __nv_bfloat16*)feats, src,
                                                                                 img_index, n_rows, (int)H, (int)n_patches, (__nv_bfloat16*)out);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
extern "C" int lmod_splice_embed_bwd(const void* dout, const int64_t* src, const int64_t* img_index, int64_t n_rows, int64_t H,
                                     int64_t n_patches, void* dfeats, void* stream) {
  LMOD_CHECK_ARG(dout && src && img_index && dfeats && n_rows > 0 && H % 8 == 0, "lmod_splice_embed_bwd: bad arguments");
  splice_embed_bwd_kernel<<<GRID1D(n_rows * 32, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)dout, src, img_index, n_rows, (int)H,
                                                                                     (int)n_patches, (__nv_bfloat16*)dfeats);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
