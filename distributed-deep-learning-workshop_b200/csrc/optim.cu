// Fused optimizers over flat parameter / gradient / state buffers (SURVEY.md K16).
// One launch updates every parameter of the model: fp32 master weights and state are read and written once, the
// (all-reduced) fp32 gradient bucket is read once, and an optional bf16 working copy is emitted in the same pass.
// Hyper-parameters come from a device array so that LR warm-up / ReduceLROnPlateau never re-capture the CUDA graph.
#include <cuda_bf16.h>

#include "ops_api.h"

namespace b200 {

__device__ __forceinline__ void store_bf16x4(__nv_bfloat16* p16, int64_t i, float4 w) {
  __nv_bfloat162 a = __floats2bfloat162_rn(w.x, w.y);
  __nv_bfloat162 b = __floats2bfloat162_rn(w.z, w.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p16 + i) = u;
}

template <bool NESTEROV>
__global__ void sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ mom,
                           __nv_bfloat16* __restrict__ p16, int64_t n4, const float* __restrict__ hyper) {
  const float lr = hyper[0], mu = hyper[1], wd = hyper[4], gs = hyper[5];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 w = reinterpret_cast<float4*>(p)[i];
    float4 gr = reinterpret_cast<const float4*>(g)[i];
    float4 m = reinterpret_cast<float4*>(mom)[i];
    float* wf = &w.x; float* gf = &gr.x; float* mf = &m.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float d = fmaf(wd, wf[k], gf[k] * gs);
      mf[k] = fmaf(mu, mf[k], d);
      const float upd = NESTEROV ? fmaf(mu, mf[k], d) : mf[k];
      wf[k] = fmaf(-lr, upd, wf[k]);
    }
    reinterpret_cast<float4*>(p)[i] = w;
    reinterpret_cast<float4*>(mom)[i] = m;
    if (p16 != nullptr) store_bf16x4(p16, i * 4, w);
  }
}

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m1,
                            float* __restrict__ v1, __nv_bfloat16* __restrict__ p16, int64_t n4,
                            const float* __restrict__ hyper) {
  const float lr = hyper[0], b1 = hyper[1], b2 = hyper[2], eps = hyper[3], wd = hyper[4], gs = hyper[5];
  const float bc1 = hyper[6], bc2 = hyper[7];
  const float step = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 w = reinterpret_cast<float4*>(p)[i];
    float4 gr = reinterpret_cast<const float4*>(g)[i];
    float4 m = reinterpret_cast<float4*>(m1)[i];
    float4 v = reinterpret_cast<float4*>(v1)[i];
    float* wf = &w.x; float* gf = &gr.x; float* mf = &m.x; float* vf = &v.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float d = fmaf(wd, wf[k], gf[k] * gs);
      mf[k] = fmaf(b1, mf[k], (1.f - b1) * d);
      vf[k] = fmaf(b2, vf[k], (1.f - b2) * d * d);
      const float denom = sqrtf(vf[k]) * inv_sqrt_bc2 + eps;
      wf[k] = wf[k] - step * mf[k] / denom;
    }
    reinterpret_cast<float4*>(p)[i] = w;
    reinterpret_cast<float4*>(m1)[i] = m;
    reinterpret_cast<float4*>(v1)[i] = v;
    if (p16 != nullptr) store_bf16x4(p16, i * 4, w);
  }
}

__global__ void adadelta_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ sq,
                                float* __restrict__ acc, __nv_bfloat16* __restrict__ p16, int64_t n4,
                                const float* __restrict__ hyper) {
  const float lr = hyper[0], rho = hyper[2], eps = hyper[3], wd = hyper[4], gs = hyper[5];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 w = reinterpret_cast<float4*>(p)[i];
    float4 gr = reinterpret_cast<const float4*>(g)[i];
    float4 s = reinterpret_cast<float4*>(sq)[i];
    float4 a = reinterpret_cast<float4*>(acc)[i];
    float* wf = &w.x; float* gf = &gr.x; float* sf = &s.x; float* af = &a.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float d = fmaf(wd, wf[k], gf[k] * gs);
      sf[k] = fmaf(rho, sf[k], (1.f - rho) * d * d);
      const float delta = sqrtf(af[k] + eps) / sqrtf(sf[k] + eps) * d;
      af[k] = fmaf(rho, af[k], (1.f - rho) * delta * delta);
      wf[k] = fmaf(-lr, delta, wf[k]);
    }
    reinterpret_cast<float4*>(p)[i] = w;
    reinterpret_cast<float4*>(sq)[i] = s;
    reinterpret_cast<float4*>(acc)[i] = a;
    if (p16 != nullptr) store_bf16x4(p16, i * 4, w);
  }
}

__global__ void cast_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, int64_t n4) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
    store_bf16x4(out, i * 4, reinterpret_cast<const float4*>(x)[i]);
}

static inline int blocks_for(int64_t n4) {
  int64_t b = (n4 + 255) / 256;
  if (b > 132 * 8) b = 132 * 8;
  if (b < 1) b = 1;
  return (int)b;
}

// n must be a multiple of 4 (flat buffers are padded by the caller).
void sgd_step(float* p, const float* g, float* mom, void* p16, int64_t n, const float* hyper, bool nesterov,
              cudaStream_t s) {
  const int64_t n4 = n / 4;
  if (nesterov)
    sgd_kernel<true><<<blocks_for(n4), 256, 0, s>>>(p, g, mom, (__nv_bfloat16*)p16, n4, hyper);
  else
    sgd_kernel<false><<<blocks_for(n4), 256, 0, s>>>(p, g, mom, (__nv_bfloat16*)p16, n4, hyper);
}
void adam_step(float* p, const float* g, float* m, float* v, void* p16, int64_t n, const float* hyper,
               cudaStream_t s) {
  const int64_t n4 = n / 4;
  adam_kernel<<<blocks_for(n4), 256, 0, s>>>(p, g, m, v, (__nv_bfloat16*)p16, n4, hyper);
}
void adadelta_step(float* p, const float* g, float* sq, float* acc, void* p16, int64_t n, const float* hyper,
                   cudaStream_t s) {
  const int64_t n4 = n / 4;
  adadelta_kernel<<<blocks_for(n4), 256, 0, s>>>(p, g, sq, acc, (__nv_bfloat16*)p16, n4, hyper);
}
void cast_f32_to_bf16(const float* x, void* out, int64_t n, cudaStream_t s) {
  cast_kernel<<<blocks_for(n / 4), 256, 0, s>>>(x, (__nv_bfloat16*)out, n / 4);
}

}  // namespace b200
