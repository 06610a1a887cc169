// optim.cu -- fused AdamW on flat buffers + gradient sum-of-squares (global-norm clipping).
//
// Replaces the reference's DeepSpeed ZeRO-2 + DeepSpeedCPUAdam optimizer-offload step
// (llavamod/train/align_trainer.py:404-417, llavamod/config/dpconfig/zero2_offload.json:16-25): fp32 master
// weights and moments stay resident in HBM; one streaming pass reads grad + 3 fp32 states and writes 3 fp32
// states + the bf16 model copy (26 B/param), no PCIe traffic.  Arithmetic = torch.optim.AdamW (decoupled
// weight decay, bias correction) with HF Trainer's clip_grad_norm_(max_grad_norm) folded in as a scalar.
#include "common.cuh"
#include "adamw8_tables.cuh"

namespace {

// per-block partial sums + a ticket: the LAST block to finish adds the partials in block order, so the global gradient norm (and with it
// the clip coefficient and every weight after the step) is bit-reproducible from run to run -- a plain atomicAdd per block is not.
// One optimizer step runs at a time per process (calls on one stream are ordered), which is what the static scratch assumes.
constexpr int SUMSQ_MAX_BLOCKS = 4096;
__device__ float g_sumsq_partial[SUMSQ_MAX_BLOCKS];
__device__ unsigned int g_sumsq_ticket = 0;

__global__ void __launch_bounds__(256) sumsq_kernel(const void* __restrict__ g, int is_f32, int64_t n, float* __restrict__ out) {
  __shared__ float red[32];
  __shared__ bool s_last;
  float a = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  if (is_f32) {
    const float* p = (const float*)g;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) a = fmaf(p[i], p[i], a);
  } else {
    const __nv_bfloat16* p = (const __nv_bfloat16*)g;
    const int64_t nv = n >> 3;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
      uint4 u = ldg_nc_v4(reinterpret_cast<const uint4*>(p) + i);
      float f[8] = {bf16lo(u.x), bf16hi(u.x), bf16lo(u.y), bf16hi(u.y), bf16lo(u.z), bf16hi(u.z), bf16lo(u.w), bf16hi(u.w)};
#pragma unroll
      for (int j = 0; j < 8; ++j) a = fmaf(f[j], f[j], a);
    }
    for (int64_t i = (nv << 3) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      float f = __bfloat162float(p[i]);
      a = fmaf(f, f, a);
    }
  }
  a = block_sum(a, red);
  if (threadIdx.x == 0) {
    g_sumsq_partial[blockIdx.x] = a;
    __threadfence();
    s_last = (atomicAdd(&g_sumsq_ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    float t = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) t += __ldcg(&g_sumsq_partial[i]);     // fixed assignment of partials to threads
    t = block_sum(t, red);
    if (threadIdx.x == 0) { out[0] += t; g_sumsq_ticket = 0u; }
  }
}

struct AdamArgs {
  float lr, beta1, beta2, eps, wd, bc1, bc2_sqrt, max_norm, grad_scale;
};

__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ master, float* __restrict__ m, float* __restrict__ v,
                                                   const void* __restrict__ grad, int grad_is_f32, __nv_bfloat16* __restrict__ model,
                                                   int64_t n, const float* __restrict__ gnorm_sq, AdamArgs a) {
  float coef = a.grad_scale;
  if (gnorm_sq && a.max_norm > 0.f) {
    const float total = sqrtf(gnorm_sq[0]) * a.grad_scale;           // clip_grad_norm_: coef = max_norm / (total + 1e-6), clamped to 1
    coef *= fminf(1.f, a.max_norm / (total + 1e-6f));
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float g = grad_is_f32 ? ((const float*)grad)[i] : __bfloat162float(((const __nv_bfloat16*)grad)[i]);
    g *= coef;
    float p = master[i];
    p *= (1.f - a.lr * a.wd);
    float mi = m[i] * a.beta1 + (1.f - a.beta1) * g;
    float vi = v[i] * a.beta2 + (1.f - a.beta2) * g * g;
    const float denom = sqrtf(vi) / a.bc2_sqrt + a.eps;
    p -= (a.lr / a.bc1) * (mi / denom);
    master[i] = p; m[i] = mi; v[i] = vi;
    if (model) model[i] = __float2bfloat16_rn(p);
  }
}

// ---- 8-bit block-wise AdamW state (--optim adamw_bnb_8bit / adamw_8bit) ------------------------------------------------------------------
// Per element a 1-byte code for m (bitsandbytes' signed dynamic map) and for v (unsigned map), per block of A8_BLOCK consecutive elements
// of the slice one fp32 absmax per moment: m = T_m[qm] * absmax_m.  One pass per step: dequantise, AdamW in fp32 with the operation order
// of adamw_kernel (decay, moments, bias-corrected update), new absmax = max|m|, max v over the block AFTER the update (NaN-propagating:
// a non-finite moment poisons its own block), codes = nearest entry of m * (1/absmax) (absmax 0 -> x = 0).  Every operation on the state
// path is an explicitly rounded intrinsic, so no FMA contraction: tests/adamw8_oracle.py restates it in numpy float32 bit for bit.
constexpr int A8_BLOCK = 2048;
constexpr int A8_THREADS = 256;                    // 8 elements per thread
static_assert(A8_BLOCK == A8_THREADS * 8, "one CTA iteration covers one quantisation block");

// nearest code of x: the number of decision midpoints strictly below x (a tie goes to the lower code, NaN to code 0); `mid` is sorted
__device__ __forceinline__ uint32_t a8_code(const float* __restrict__ mid, float x) {
  uint32_t q = 0;
#pragma unroll
  for (uint32_t s = 128; s > 0; s >>= 1) q += (x > mid[q + s - 1]) ? s : 0u;
  return q;
}

__global__ void __launch_bounds__(A8_THREADS) adamw_8bit_kernel(float* __restrict__ master, uint8_t* __restrict__ qm, uint8_t* __restrict__ qv,
                                                                float* __restrict__ absmax_m, float* __restrict__ absmax_v,
                                                                const __nv_bfloat16* __restrict__ grad, __nv_bfloat16* __restrict__ model,
                                                                int64_t n, const float* __restrict__ gnorm_sq, AdamArgs a) {
  __shared__ float s_tm[256], s_tv[256], s_mid_m[256], s_mid_v[256];
  __shared__ float2 s_red[A8_THREADS / 32];
  const int t = threadIdx.x;
  s_tm[t] = __uint_as_float(LMOD_ADAMW8_CODE_M[t]);
  s_tv[t] = __uint_as_float(LMOD_ADAMW8_CODE_V[t]);
  __syncthreads();
  if (t < 255) {
    s_mid_m[t] = __fmul_rn(__fadd_rn(s_tm[t], s_tm[t + 1]), 0.5f);
    s_mid_v[t] = __fmul_rn(__fadd_rn(s_tv[t], s_tv[t + 1]), 0.5f);
  }
  __syncthreads();

  float coef = a.grad_scale;
  if (gnorm_sq && a.max_norm > 0.f) {                                    // clip_grad_norm_: coef = max_norm / (total + 1e-6), clamped to 1
    const float total = __fmul_rn(__fsqrt_rn(gnorm_sq[0]), a.grad_scale);
    coef = __fmul_rn(coef, fminf(1.f, __fdiv_rn(a.max_norm, __fadd_rn(total, 1e-6f))));
  }
  const float decay = __fsub_rn(1.f, __fmul_rn(a.lr, a.wd));
  const float omb1 = __fsub_rn(1.f, a.beta1), omb2 = __fsub_rn(1.f, a.beta2);
  const float step_size = __fdiv_rn(a.lr, a.bc1);
  const int lane = t & 31, w = t >> 5;
  const int64_t nblk = (n + A8_BLOCK - 1) / A8_BLOCK;
  for (int64_t b = blockIdx.x; b < nblk; b += gridDim.x) {
    const int64_t i0 = b * A8_BLOCK + (int64_t)t * 8;
    const bool live = i0 < n;                                            // n % 8 == 0: a thread's 8 elements are all in or all out
    float m[8], v[8];
    float am = 0.f, av = 0.f;
    if (live) {
      const uint4 gu = ldg_nc_v4(grad + i0);
      const float g[8] = {bf16lo(gu.x), bf16hi(gu.x), bf16lo(gu.y), bf16hi(gu.y), bf16lo(gu.z), bf16hi(gu.z), bf16lo(gu.w), bf16hi(gu.w)};
      const float4 p0 = *reinterpret_cast<const float4*>(master + i0), p1 = *reinterpret_cast<const float4*>(master + i0 + 4);
      float p[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
      const uint2 cm = *reinterpret_cast<const uint2*>(qm + i0), cv = *reinterpret_cast<const uint2*>(qv + i0);
      const float sm = absmax_m[b], sv = absmax_v[b];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t bm = ((j < 4 ? cm.x : cm.y) >> (8 * (j & 3))) & 0xffu, bv = ((j < 4 ? cv.x : cv.y) >> (8 * (j & 3))) & 0xffu;
        const float gj = __fmul_rn(g[j], coef);
        m[j] = __fadd_rn(__fmul_rn(__fmul_rn(s_tm[bm], sm), a.beta1), __fmul_rn(omb1, gj));
        v[j] = __fadd_rn(__fmul_rn(__fmul_rn(s_tv[bv], sv), a.beta2), __fmul_rn(__fmul_rn(omb2, gj), gj));
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v[j]), a.bc2_sqrt), a.eps);
        p[j] = __fsub_rn(__fmul_rn(p[j], decay), __fmul_rn(step_size, __fdiv_rn(m[j], denom)));
        am = max_nan(am, fabsf(m[j]));
        av = max_nan(av, v[j]);
      }
      *reinterpret_cast<float4*>(master + i0) = make_float4(p[0], p[1], p[2], p[3]);
      *reinterpret_cast<float4*>(master + i0 + 4) = make_float4(p[4], p[5], p[6], p[7]);
      if (model) {
        uint4 o;
        o.x = pack_bf16x2(p[0], p[1]); o.y = pack_bf16x2(p[2], p[3]); o.z = pack_bf16x2(p[4], p[5]); o.w = pack_bf16x2(p[6], p[7]);
        *reinterpret_cast<uint4*>(model + i0) = o;
      }
    }
    // the block's two new scales: warp shuffles, then one float2 per warp through shared memory (the leading barrier keeps the
    // previous iteration's readers ahead of this iteration's writers)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      am = max_nan(am, __shfl_xor_sync(0xffffffffu, am, o));
      av = max_nan(av, __shfl_xor_sync(0xffffffffu, av, o));
    }
    __syncthreads();
    if (lane == 0) s_red[w] = make_float2(am, av);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < A8_THREADS / 32; ++k) {
      am = max_nan(am, s_red[k].x);
      av = max_nan(av, s_red[k].y);
    }
    if (live) {
      const float inv_m = am > 0.f ? __frcp_rn(am) : 0.f, inv_v = av > 0.f ? __frcp_rn(av) : 0.f;   // NaN scale -> 0: codes stay finite
      uint2 om = make_uint2(0u, 0u), ov = make_uint2(0u, 0u);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t cmj = a8_code(s_mid_m, __fmul_rn(m[j], inv_m)) << (8 * (j & 3));
        const uint32_t cvj = a8_code(s_mid_v, __fmul_rn(v[j], inv_v)) << (8 * (j & 3));
        if (j < 4) { om.x |= cmj; ov.x |= cvj; } else { om.y |= cmj; ov.y |= cvj; }
      }
      *reinterpret_cast<uint2*>(qm + i0) = om;
      *reinterpret_cast<uint2*>(qv + i0) = ov;
    }
    if (t == 0) { absmax_m[b] = am; absmax_v[b] = av; }                  // every live thread read the old scales before the barriers above
  }
}

}  // namespace

extern "C" int lmod_sumsq(const void* g, int is_f32, int64_t count, float* out_accum, void* stream) {
  LMOD_CHECK_ARG(g && out_accum && count > 0, "lmod_sumsq: bad arguments");
  LMOD_CHECK_ARG(is_f32 || ((uintptr_t)g % 16 == 0), "lmod_sumsq: bf16 buffer must be 16B aligned");
  int64_t blocks = (count / 8 + 255) / 256;
  int64_t cap = (int64_t)lmod_num_sms() * 8;
  if (cap > SUMSQ_MAX_BLOCKS) cap = SUMSQ_MAX_BLOCKS;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  sumsq_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(g, is_f32, count, out_accum);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_adamw(float* master, float* m, float* v, const void* grad, int grad_is_f32, void* model_bf16, int64_t count,
                          float lr, float beta1, float beta2, float eps, float wd, int64_t step, const float* gnorm_sq,
                          float max_norm, float grad_scale, void* stream) {
  LMOD_CHECK_ARG(master && m && v && grad && count > 0 && step >= 1, "lmod_adamw: bad arguments");
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = wd;
  a.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  a.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  a.max_norm = max_norm; a.grad_scale = grad_scale;
  int64_t blocks = (count + 255) / 256;
  int64_t cap = (int64_t)lmod_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  adamw_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(master, m, v, grad, grad_is_f32, (__nv_bfloat16*)model_bf16, count, gnorm_sq, a);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}

extern "C" int lmod_adamw_8bit(float* master, uint8_t* m8, uint8_t* v8, float* absmax_m, float* absmax_v, const void* grad_bf16,
                               void* model_bf16, int64_t count, float lr, float beta1, float beta2, float eps, float wd, int64_t step,
                               const float* gnorm_sq, float max_norm, float grad_scale, void* stream) {
  LMOD_CHECK_ARG(master && m8 && v8 && absmax_m && absmax_v && grad_bf16 && count > 0 && step >= 1, "lmod_adamw_8bit: bad arguments");
  LMOD_CHECK_ARG(count % 8 == 0, "lmod_adamw_8bit: count (%lld) must be a multiple of 8", (long long)count);
  LMOD_CHECK_ARG(((uintptr_t)master | (uintptr_t)m8 | (uintptr_t)v8 | (uintptr_t)grad_bf16 | (uintptr_t)model_bf16) % 16 == 0,
                 "lmod_adamw_8bit: master, codes, gradient and model buffers must be 16B aligned");
  AdamArgs a;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = wd;
  a.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  a.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  a.max_norm = max_norm; a.grad_scale = grad_scale;
  int64_t blocks = (count + A8_BLOCK - 1) / A8_BLOCK;
  const int64_t cap = (int64_t)lmod_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  adamw_8bit_kernel<<<(unsigned)blocks, A8_THREADS, 0, (cudaStream_t)stream>>>(master, m8, v8, absmax_m, absmax_v, (const __nv_bfloat16*)grad_bf16,
                                                                                 (__nv_bfloat16*)model_bf16, count, gnorm_sq, a);
  LMOD_LAUNCH_OK();
  return LMOD_OK;
}
