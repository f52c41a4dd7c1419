// Backward kernels of MobileNetV2 fine-tuning (models/mobilenet_engine.py, `fine_tune_at`).  With the base's BatchNorm in
// inference mode (below); with training-mode BatchNorm the engine combines relu6_mask_reduce (also summing dz * c) and the
// depthwise / stem kernels here with the ResNet-50 BatchNorm kernels of elementwise.cu (DESIGN.md 3.5b).  A trainable layer computes c = conv(x, W), z = s*c + t with the folded affine s = gamma*invstd,
// t = beta - mean*s (frozen statistics), and y = act(z [+ residual]).  With g the gradient arriving at y:
//
//   dz = g * [0 < y < 6]  (ReLU6, mask from the stored bf16 y)   or   dz = g1 + g2  (linear project layer + skip)
//   dbeta = sum_px dz                                  relu6_mask_reduce
//   dx = conv_transpose(dz, s (.) W)                   ConvDgrad (pointwise) / dw_dgrad (depthwise)
//   G = sum_px dz (x) input                            ConvWgrad (pointwise) / dw_wgrad / mbv2_stem_wgrad
//   dW = s*G,  dgamma = invstd * (<W_c, G_c> - mean*dbeta)     mbv2_ft_finalize (sum_px dz*c = <W_c, G_c>)
//
// so the conv output c is never stored and gamma is never divided by.  mbv2_ft_refresh recomputes s / t and the
// bf16 dgrad filters of the trainable layers after every optimizer step.
//
// Summation order: the depthwise data gradient is a gather with a fixed tap order (no atomics, deterministic).  The
// per-channel sums and the depthwise / stem weight gradients reduce inside a CTA in a fixed order and add one fp32
// partial per CTA to the output with atomicAdd (as conv_wgrad.cu does); the output must be zeroed first.  A term
// passes at most ceil(units / (lanes * gridDim.y)) + log2(lanes) + 3 + gridDim.y additions on its way to the result.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops_api.h"

namespace b200 {

namespace {
struct alignas(16) bfx8 {
  __nv_bfloat162 v[4];
};
__device__ __forceinline__ void unpack(const bfx8& v, float* f) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 p = __bfloat1622float2(v.v[k]);
    f[2 * k] = p.x;
    f[2 * k + 1] = p.y;
  }
}
__device__ __forceinline__ bfx8 pack(const float* f) {
  bfx8 o;
#pragma unroll
  for (int k = 0; k < 4; ++k) o.v[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
  return o;
}
__device__ __forceinline__ bfx8 zero8() {
  bfx8 o;
#pragma unroll
  for (int k = 0; k < 4; ++k) o.v[k] = __floats2bfloat162_rn(0.f, 0.f);
  return o;
}
inline int blocks_for(int64_t units, int per_block, int cap) {
  int64_t b = (units + per_block - 1) / per_block;
  if (b > cap) b = cap;
  return b < 1 ? 1 : (int)b;
}
constexpr int kTW = 4;   // output (wgrad) / input (dgrad) pixels per thread along W
}  // namespace

// ------------------------------------------------------------------------------------------------ ReLU6 mask + reduction
// Block = 8 channel vectors (64 channels, blockIdx.x) x 32 row lanes; rows grid-stride over blockIdx.y.
// dz may alias g1 (element-wise, each element read before it is written by the same thread).
// DZC (training-mode BatchNorm): also sum_dzc[ch] += sum(dz * c) with c the stored bf16 conv output, the same lanes and
// the same fixed in-CTA order as sum(dz).
template <bool RELU6, bool G2, bool DZC = false>
__global__ void __launch_bounds__(256)
relu6_mask_reduce_kernel(const __nv_bfloat16* g1, const __nv_bfloat16* __restrict__ g2, const __nv_bfloat16* __restrict__ y,
                         __nv_bfloat16* dz, float* __restrict__ sum, int64_t M, int C,
                         const __nv_bfloat16* __restrict__ cin = nullptr, float* __restrict__ sum_dzc = nullptr) {
  __shared__ float red[DZC ? 2 : 1][8][64];
  const int cv = blockIdx.x * 8 + (threadIdx.x & 7);
  const bool active = cv < C / 8;
  float acc[8], acc2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = acc2[k] = 0.f;
  if (active) {
    for (int64_t m = blockIdx.y * 32 + (threadIdx.x >> 3); m < M; m += (int64_t)gridDim.y * 32) {
      const int64_t o = m * C + cv * 8;
      float g[8];
      unpack(*reinterpret_cast<const bfx8*>(g1 + o), g);
      if (G2) {
        float h[8];
        unpack(*reinterpret_cast<const bfx8*>(g2 + o), h);
#pragma unroll
        for (int k = 0; k < 8; ++k) g[k] += h[k];
      }
      if (RELU6) {
        float v[8];
        unpack(*reinterpret_cast<const bfx8*>(y + o), v);
#pragma unroll
        for (int k = 0; k < 8; ++k) g[k] = (v[k] > 0.f && v[k] < 6.f) ? g[k] : 0.f;
      }
      const bfx8 d = pack(g);
      *reinterpret_cast<bfx8*>(dz + o) = d;
      unpack(d, g);   // sum the stored (bf16) gradient
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += g[k];
      if (DZC) {
        float cc[8];
        unpack(*reinterpret_cast<const bfx8*>(cin + o), cc);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc2[k] = fmaf(g[k], cc[k], acc2[k]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 8);
    acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 16);
    if (DZC) {
      acc2[k] += __shfl_xor_sync(0xffffffffu, acc2[k], 8);
      acc2[k] += __shfl_xor_sync(0xffffffffu, acc2[k], 16);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      red[0][warp][lane * 8 + k] = acc[k];
      if (DZC) red[DZC ? 1 : 0][warp][lane * 8 + k] = acc2[k];
    }
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int c = blockIdx.x * 64 + threadIdx.x;
    if (c < C) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[0][w][threadIdx.x];
      atomicAdd(sum + c, s);
      if (DZC) {
        float s2 = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s2 += red[DZC ? 1 : 0][w][threadIdx.x];
        atomicAdd(sum_dzc + c, s2);
      }
    }
  }
}
void relu6_mask_reduce(const void* g1, const void* g2, const void* y, void* dz, float* sum, const void* c, float* sum_dzc,
                       int64_t M, int C, bool relu6, cudaStream_t s) {
  const int gx = (C / 8 + 7) / 8;
  const int gy = blocks_for(M, 32, (132 * 8 + gx - 1) / gx);
  const dim3 grid(gx, gy);
  auto a = (const __nv_bfloat16*)g1;
  auto b = (const __nv_bfloat16*)g2;
  auto v = (const __nv_bfloat16*)y;
  auto d = (__nv_bfloat16*)dz;
  if (c != nullptr) {   // training-mode BatchNorm: ReLU6 layers have no skip gradient, linear layers may have one
    auto cc = (const __nv_bfloat16*)c;
    if (relu6 && g2)      relu6_mask_reduce_kernel<true, true, true><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C, cc, sum_dzc);
    else if (relu6)       relu6_mask_reduce_kernel<true, false, true><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C, cc, sum_dzc);
    else if (g2)          relu6_mask_reduce_kernel<false, true, true><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C, cc, sum_dzc);
    else                  relu6_mask_reduce_kernel<false, false, true><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C, cc, sum_dzc);
    return;
  }
  if (relu6 && g2)        relu6_mask_reduce_kernel<true, true><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C);
  else if (relu6)         relu6_mask_reduce_kernel<true, false><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C);
  else if (g2)            relu6_mask_reduce_kernel<false, true><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C);
  else                    relu6_mask_reduce_kernel<false, false><<<grid, 256, 0, s>>>(a, b, v, d, sum, M, C);
}

// ------------------------------------------------------------------------------------------------ depthwise 3x3 dgrad
// dx[n, h, w, c] = sum_{r, s} dz[n, (h+1-r)/S, (w+1-s)/S, c] * scale[c] * wt[r*3+s, c]  over the taps whose output pixel
// exists (pad 1).  Thread = (input row h, kTW adjacent input pixels w0.., 8 channels): a gather, r outer / s inner.
template <int STRIDE>
__global__ void __launch_bounds__(256)
dw_dgrad_kernel(const __nv_bfloat16* __restrict__ dz, const float* __restrict__ wt, const float* __restrict__ scale,
                __nv_bfloat16* __restrict__ dx, int N, int H, int W, int C, int Ho, int Wo) {
  constexpr int NIN = STRIDE == 1 ? kTW + 2 : kTW / 2 + 1;   // dz vectors a row of kTW inputs reads
  const int cvec = C / 8;
  const int wt_n = (W + kTW - 1) / kTW;
  const int64_t total = (int64_t)N * H * wt_n * cvec;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % cvec);
    int64_t p = i / cvec;
    const int tw = (int)(p % wt_n);
    p /= wt_n;
    const int h = (int)(p % H);
    const int n = (int)(p / H);
    const int w0 = tw * kTW;
    const int wo0 = STRIDE == 1 ? w0 - 1 : w0 / 2;   // w0 is even, so stride-2 taps hit wo0 + (t + 1 - s) / 2
    float sc[8];
    {
      const float4 a = *reinterpret_cast<const float4*>(scale + cv * 8), b = *reinterpret_cast<const float4*>(scale + cv * 8 + 4);
      sc[0] = a.x; sc[1] = a.y; sc[2] = a.z; sc[3] = a.w; sc[4] = b.x; sc[5] = b.y; sc[6] = b.z; sc[7] = b.w;
    }
    float acc[kTW][8];
#pragma unroll
    for (int t = 0; t < kTW; ++t)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[t][k] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hh = h + 1 - r;
      if (hh < 0 || (STRIDE == 2 && (hh & 1))) continue;
      const int ho = hh / STRIDE;
      if (ho >= Ho) continue;
      const __nv_bfloat16* rowp = dz + ((int64_t)n * Ho + ho) * Wo * C + cv * 8;
      bfx8 in[NIN];
#pragma unroll
      for (int k = 0; k < NIN; ++k) {
        const int wo = wo0 + k;
        in[k] = (wo >= 0 && wo < Wo) ? *reinterpret_cast<const bfx8*>(rowp + (int64_t)wo * C) : zero8();
      }
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const float4 a = *reinterpret_cast<const float4*>(wt + (r * 3 + s) * C + cv * 8);
        const float4 b = *reinterpret_cast<const float4*>(wt + (r * 3 + s) * C + cv * 8 + 4);
        const float wr[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        float ws[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) ws[k] = __fmul_rn(sc[k], wr[k]);
#pragma unroll
        for (int t = 0; t < kTW; ++t) {
          const int d = t + 1 - s;              // (w + 1 - s) - w0
          if (STRIDE == 2 && (d & 1)) continue;   // compile-time after unrolling
          const int idx = STRIDE == 1 ? d + 1 : d / 2;
          if (idx < 0) continue;
          float f[8];
          unpack(in[idx], f);
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[t][k] = fmaf(f[k], ws[k], acc[t][k]);
        }
      }
    }
    __nv_bfloat16* orow = dx + (((int64_t)n * H + h) * W) * C + cv * 8;
#pragma unroll
    for (int t = 0; t < kTW; ++t) {
      if (w0 + t >= W) break;
      *reinterpret_cast<bfx8*>(orow + (int64_t)(w0 + t) * C) = pack(acc[t]);
    }
  }
}
void dw_dgrad(const void* dz, const float* w, const float* scale, void* dx, int N, int H, int W, int C, int stride,
              cudaStream_t s) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const int blocks = blocks_for((int64_t)N * H * ((W + kTW - 1) / kTW) * (C / 8), 256, 132 * 16);
  if (stride == 1)
    dw_dgrad_kernel<1><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)dz, w, scale, (__nv_bfloat16*)dx, N, H, W, C, Ho, Wo);
  else
    dw_dgrad_kernel<2><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)dz, w, scale, (__nv_bfloat16*)dx, N, H, W, C, Ho, Wo);
}

// ------------------------------------------------------------------------------------------------ depthwise 3x3 wgrad
// G[r*3+s, c] += sum_{n, ho, wo} dz[n, ho, wo, c] * x[n, ho*S-1+r, wo*S-1+s, c].  Block = 8 channel vectors (blockIdx.x)
// x 32 lanes; a lane takes strips of kTW output pixels (grid-stride over blockIdx.y), loading each input row of a strip
// once.  72 fp32 accumulators per thread, reduced over the block in a fixed order, one atomicAdd per (tap, channel, CTA).
template <int STRIDE>
__global__ void __launch_bounds__(256)
dw_wgrad_kernel(const __nv_bfloat16* __restrict__ dz, const __nv_bfloat16* __restrict__ x, float* __restrict__ G, int N,
                int H, int W, int C, int Ho, int Wo) {
  constexpr int NIN = (kTW - 1) * STRIDE + 3;
  __shared__ float red[8][9 * 64];
  const int cv = blockIdx.x * 8 + (threadIdx.x & 7);
  const bool active = cv < C / 8;
  const int wt_n = (Wo + kTW - 1) / kTW;
  const int64_t units = (int64_t)N * Ho * wt_n;
  float acc[9][8];
#pragma unroll
  for (int j = 0; j < 9; ++j)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[j][k] = 0.f;
  if (active) {
    for (int64_t u = blockIdx.y * 32 + (threadIdx.x >> 3); u < units; u += (int64_t)gridDim.y * 32) {
      const int tw = (int)(u % wt_n);
      const int64_t p = u / wt_n;
      const int ho = (int)(p % Ho);
      const int n = (int)(p / Ho);
      const int wo0 = tw * kTW;
      float d[kTW][8];
      const __nv_bfloat16* drow = dz + (((int64_t)n * Ho + ho) * Wo) * C + cv * 8;
#pragma unroll
      for (int t = 0; t < kTW; ++t) unpack(wo0 + t < Wo ? *reinterpret_cast<const bfx8*>(drow + (int64_t)(wo0 + t) * C) : zero8(), d[t]);
      const int wi0 = wo0 * STRIDE - 1;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int h = ho * STRIDE - 1 + r;
        if (h < 0 || h >= H) continue;
        const __nv_bfloat16* xrow = x + ((int64_t)n * H + h) * W * C + cv * 8;
        bfx8 in[NIN];
#pragma unroll
        for (int k = 0; k < NIN; ++k) {
          const int ww = wi0 + k;
          in[k] = (ww >= 0 && ww < W) ? *reinterpret_cast<const bfx8*>(xrow + (int64_t)ww * C) : zero8();
        }
#pragma unroll
        for (int s = 0; s < 3; ++s)
#pragma unroll
          for (int t = 0; t < kTW; ++t) {
            float f[8];
            unpack(in[t * STRIDE + s], f);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[r * 3 + s][k] = fmaf(f[k], d[t][k], acc[r * 3 + s][k]);
          }
      }
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 9; ++j)
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float v = acc[j][k];
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (lane < 8) red[warp][j * 64 + lane * 8 + k] = v;
    }
  __syncthreads();
  for (int e = threadIdx.x; e < 9 * 64; e += blockDim.x) {
    const int c = blockIdx.x * 64 + (e & 63);
    if (c >= C) continue;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][e];
    atomicAdd(G + (e >> 6) * C + c, s);
  }
}
void dw_wgrad(const void* dz, const void* x, float* G, int N, int H, int W, int C, int stride, cudaStream_t s) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const int gx = (C / 8 + 7) / 8;
  const int gy = blocks_for((int64_t)N * Ho * ((Wo + kTW - 1) / kTW), 32, (132 * 4 + gx - 1) / gx);
  const dim3 grid(gx, gy);
  if (stride == 1)
    dw_wgrad_kernel<1><<<grid, 256, 0, s>>>((const __nv_bfloat16*)dz, (const __nv_bfloat16*)x, G, N, H, W, C, Ho, Wo);
  else
    dw_wgrad_kernel<2><<<grid, 256, 0, s>>>((const __nv_bfloat16*)dz, (const __nv_bfloat16*)x, G, N, H, W, C, Ho, Wo);
}

// ------------------------------------------------------------------------------------------------ stem wgrad
// G[(r*3+s)*3+c, co] += sum_px dz[px, co] * bf16(x[px + tap] * mul + add)   (the input mbv2_stem convolves; 0 outside).
// Thread = (16 pixel lanes) x (combo = 8 output channels q x filter row r: 12 combos); a half-warp shares one combo, so
// the pixel reduction is four xor-shuffles; lane 0 adds its 72 partials with atomicAdd.
__global__ void __launch_bounds__(192)
mbv2_stem_wgrad_kernel(const uint8_t* __restrict__ x, const __nv_bfloat16* __restrict__ dz, float* __restrict__ G, int N,
                       int H, int W, int ldc, float mul, float add) {
  const int lane = threadIdx.x & 15, combo = threadIdx.x >> 4;
  const int q = combo / 3, r = combo % 3;
  const int Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)N * Ho * Wo;
  float acc[9][8];
#pragma unroll
  for (int j = 0; j < 9; ++j)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[j][k] = 0.f;
  for (int64_t p = blockIdx.x * 16 + lane; p < total; p += (int64_t)gridDim.x * 16) {
    const int wo = (int)(p % Wo);
    const int64_t t = p / Wo;
    const int ho = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const int h = 2 * ho - 1 + r;
    if (h < 0 || h >= H) continue;
    float d[8];
    unpack(*reinterpret_cast<const bfx8*>(dz + p * ldc + q * 8), d);
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int ww = 2 * wo - 1 + s;
      if (ww < 0 || ww >= W) continue;
      const uint8_t* px = x + (((int64_t)n * H + h) * W + ww) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = __bfloat162float(__float2bfloat16(fmaf((float)px[c], mul, add)));
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[s * 3 + c][k] = fmaf(v, d[k], acc[s * 3 + c][k]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 9; ++j)
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float v = acc[j][k];
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) atomicAdd(G + (r * 9 + j) * 32 + q * 8 + k, v);
    }
}
void mbv2_stem_wgrad(const uint8_t* x, const void* dz, float* G, int N, int H, int W, int ldc, float mul, float add,
                     cudaStream_t s) {
  const int blocks = blocks_for((int64_t)N * (H / 2) * (W / 2), 16, 132 * 8);
  mbv2_stem_wgrad_kernel<<<blocks, 192, 0, s>>>(x, (const __nv_bfloat16*)dz, G, N, H, W, ldc, mul, add);
}

// ------------------------------------------------------------------------------------------------ finalize
// One warp per (layer, real output channel c):  dot = <W_c, G_c>;  dgamma = invstd * (dot - mean * sum_dz);
// dbeta = sum_dz;  G_c *= scale[c].  W_c / G_c: `count` elements at c*cstride + j*jstride; W is bf16 (the flat bf16
// copy the pointwise forward reads) or fp32 (depthwise / stem master weights).
__global__ void __launch_bounds__(256)
mbv2_ft_finalize_kernel(const float* __restrict__ params, const __nv_bfloat16* __restrict__ w16, float* __restrict__ grads,
                        const int64_t* __restrict__ table) {
  const int64_t* e = table + blockIdx.y * kFtFinalizeFields;
  const int c_real = (int)e[0], count = (int)e[1], cstride = (int)e[2], jstride = (int)e[3];
  const bool wbf16 = e[4] != 0;
  float* G = grads + e[5];
  const float* scale = reinterpret_cast<const float*>(e[9]);
  const float* invstd = reinterpret_cast<const float*>(e[10]);
  const float* mean = reinterpret_cast<const float*>(e[11]);
  const float* sum_dz = reinterpret_cast<const float*>(e[12]);
  const int lane = threadIdx.x & 31;
  for (int c = blockIdx.x * 8 + (threadIdx.x >> 5); c < c_real; c += gridDim.x * 8) {
    float dot = 0.f;
    for (int j = lane; j < count; j += 32) {
      const int64_t o = (int64_t)c * cstride + (int64_t)j * jstride;
      const float w = wbf16 ? __bfloat162float(w16[e[6] + o]) : params[e[6] + o];
      dot = fmaf(w, G[o], dot);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    const float s = scale[c];
    for (int j = lane; j < count; j += 32) {
      const int64_t o = (int64_t)c * cstride + (int64_t)j * jstride;
      G[o] = __fmul_rn(s, G[o]);
    }
    if (lane == 0) {
      const float db = sum_dz[c];
      grads[e[8] + c] = db;
      grads[e[7] + c] = __fmul_rn(invstd[c], __fsub_rn(dot, __fmul_rn(mean[c], db)));
    }
  }
}
void mbv2_ft_finalize(const float* params, const void* w16, float* grads, const int64_t* table, int layers, cudaStream_t s) {
  mbv2_ft_finalize_kernel<<<dim3(16, layers), 256, 0, s>>>(params, (const __nv_bfloat16*)w16, grads, table);
}

// ------------------------------------------------------------------------------------------------ refresh
// Per layer:  scale[c] = gamma*invstd, shift[c] = beta - mean*scale (c < c_real; padded channels 1 / 0), rounded step by
// step exactly like the host fold (models/mobilenet_engine.py `_affine`);  and, for pointwise layers, the bf16 dgrad
// filter wd[ci, co] = bf16(scale[co] * W[co, ci]) from the fp32 master W [cp, cin_p].
__global__ void __launch_bounds__(256)
mbv2_ft_refresh_kernel(const float* __restrict__ params, const int64_t* __restrict__ table) {
  const int64_t* e = table + blockIdx.y * kFtRefreshFields;
  const int c_real = (int)e[0], cp = (int)e[1], cin_p = (int)e[2];
  const float* gamma = params + e[3];
  const float* beta = params + e[4];
  const float* W = params + e[5];
  const float* invstd = reinterpret_cast<const float*>(e[6]);
  const float* mean = reinterpret_cast<const float*>(e[7]);
  float* scale = reinterpret_cast<float*>(e[8]);
  float* shift = reinterpret_cast<float*>(e[9]);
  __nv_bfloat16* wd = reinterpret_cast<__nv_bfloat16*>(e[10]);
  const int64_t total = cp + (int64_t)cp * cin_p;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < cp) {
      const int c = (int)i;
      float sc = 1.f, sh = 0.f;
      if (c < c_real) {
        sc = __fmul_rn(gamma[c], invstd[c]);
        sh = __fsub_rn(beta[c], __fmul_rn(mean[c], sc));
      }
      scale[c] = sc;
      shift[c] = sh;
    } else {
      const int64_t k = i - cp;
      const int ci = (int)(k / cp), co = (int)(k % cp);
      const float sc = co < c_real ? __fmul_rn(gamma[co], invstd[co]) : 1.f;
      wd[k] = __float2bfloat16_rn(__fmul_rn(sc, W[(int64_t)co * cin_p + ci]));
    }
  }
}
void mbv2_ft_refresh(const float* params, const int64_t* table, int layers, cudaStream_t s) {
  mbv2_ft_refresh_kernel<<<dim3(32, layers), 256, 0, s>>>(params, table);
}

}  // namespace b200
