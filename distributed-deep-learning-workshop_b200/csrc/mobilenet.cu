// Kernels the reference's own model needs beyond the implicit-GEMM convolutions (SURVEY.md C14: frozen MobileNetV2 base +
// GAP + Dropout + Dense, P1/03:159-178): the 3-channel 3x3/2 stem and the depthwise 3x3 convolutions, both with the
// (inference-mode, i.e. folded) BatchNorm affine and ReLU6 applied in the same pass.  The pointwise (1x1) convolutions -
// ~95 % of MobileNetV2's FLOPs - run on the wgmma kernels with the kStats = 4 epilogue (csrc/conv_igemm.cuh).
// Activations are NHWC bf16 with the channel count padded to a multiple of 64 (the GEMM's K / N granularity); padded
// channels are zero everywhere (zero weights, zero shift), so they never need special handling.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops_api.h"

namespace b200 {

namespace {
struct alignas(16) bfx8 {
  __nv_bfloat162 v[4];
};
inline int capped_blocks(int64_t units, int per_block, int cap) {
  int64_t b = (units + per_block - 1) / per_block;
  if (b > cap) b = cap;
  return b < 1 ? 1 : (int)b;
}
// c = bf16(acc) into o, and s += c, q += c^2 of the rounded values (the statistics the GEMM epilogue takes)
__device__ __forceinline__ void round_and_sum(const float* acc, bfx8& o, float* s, float* q) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    o.v[k] = __floats2bfloat162_rn(acc[2 * k], acc[2 * k + 1]);
    const float2 f = __bfloat1622float2(o.v[k]);
    s[2 * k] += f.x;
    s[2 * k + 1] += f.y;
    q[2 * k] = fmaf(f.x, f.x, q[2 * k]);
    q[2 * k + 1] = fmaf(f.y, f.y, q[2 * k + 1]);
  }
}
}  // namespace

// ------------------------------------------------------------------------------------------------ stem 3x3 / 2, 3 -> 32
// x: uint8 [N, H, W, 3];  w: fp32 [27][32] (k = (r*3 + s)*3 + c, tap-major);  out: bf16 [N, H/2, W/2, ldc] (first 32 channels
// written, the rest of the buffer stays zero);  v = x * mul + add  (MobileNet preprocess_input),  y = relu6(conv * scale + shift)
__global__ void __launch_bounds__(256)
mbv2_stem_kernel(const uint8_t* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                 const float* __restrict__ shift, __nv_bfloat16* __restrict__ out, int N, int H, int W, int ldc, float mul,
                 float add) {
  __shared__ float sw[27 * 32];
  __shared__ float ssc[32], ssh[32];
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x) sw[i] = w[i];
  if (threadIdx.x < 32) {
    ssc[threadIdx.x] = scale[threadIdx.x];
    ssh[threadIdx.x] = shift[threadIdx.x];
  }
  __syncthreads();
  const int Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)N * Ho * Wo * 4;  // 4 threads per output pixel, 8 channels each
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int q = (int)(i & 3);
    int64_t p = i >> 2;
    const int wo = (int)(p % Wo);
    p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    // TF/Keras 'same' padding for stride 2 on an even input pads bottom/right only: input row = 2*ho + r (r = 0..2);
    // torchvision pads 1 on both sides: input row = 2*ho - 1 + r.  The parity model follows torchvision (models/mobilenet.py).
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int h = 2 * ho - 1 + r;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ww = 2 * wo - 1 + s;
        if (ww < 0 || ww >= W) continue;
        const uint8_t* px = x + (((int64_t)n * H + h) * W + ww) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          // bf16 rounding of the normalised input: the same value the GEMM-based layers would read
          const float v = __bfloat162float(__float2bfloat16(fmaf((float)px[c], mul, add)));
          const float* wr = sw + ((r * 3 + s) * 3 + c) * 32 + q * 8;
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(v, wr[k], acc[k]);
        }
      }
    }
    bfx8 o;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = fminf(fmaxf(fmaf(acc[2 * k], ssc[q * 8 + 2 * k], ssh[q * 8 + 2 * k]), 0.f), 6.f);
      const float b = fminf(fmaxf(fmaf(acc[2 * k + 1], ssc[q * 8 + 2 * k + 1], ssh[q * 8 + 2 * k + 1]), 0.f), 6.f);
      o.v[k] = __floats2bfloat162_rn(a, b);
    }
    *reinterpret_cast<bfx8*>(out + ((((int64_t)n * Ho + ho) * Wo + wo) * ldc) + q * 8) = o;
  }
}
void mbv2_stem(const uint8_t* x, const float* w, const float* scale, const float* shift, void* out, int N, int H, int W,
               int ldc, float mul, float add, cudaStream_t s) {
  const int64_t total = (int64_t)N * (H / 2) * (W / 2) * 4;
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  mbv2_stem_kernel<<<(int)blocks, 256, 0, s>>>(x, w, scale, shift, (__nv_bfloat16*)out, N, H, W, ldc, mul, add);
}

// Training-mode BatchNorm variant: c = conv3x3/2(x*mul + add) stored as bf16 (no affine, no clamp), and the per-channel
// sum(c), sum(c^2) of the stored values.  Same thread mapping and fmaf order as mbv2_stem_kernel; the grid stride is a
// multiple of 4, so a thread keeps its 8 channels q for the whole loop.  Reduction: xor-shuffles over the 8 lanes of a
// warp that share q, then the 8 warps in a fixed order, one atomicAdd per channel per CTA.
__global__ void __launch_bounds__(256)
mbv2_stem_stats_kernel(const uint8_t* __restrict__ x, const float* __restrict__ w, __nv_bfloat16* __restrict__ out,
                       float* __restrict__ sum, float* __restrict__ sqsum, int N, int H, int W, int ldc, float mul,
                       float add) {
  __shared__ float sw[27 * 32];
  __shared__ float red[2][8][32];
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int Ho = H / 2, Wo = W / 2;
  const int q = threadIdx.x & 3;
  float ssum[8], ssq[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) ssum[k] = ssq[k] = 0.f;
  const int64_t total = (int64_t)N * Ho * Wo * 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = i >> 2;
    const int wo = (int)(p % Wo);
    p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int h = 2 * ho - 1 + r;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ww = 2 * wo - 1 + s;
        if (ww < 0 || ww >= W) continue;
        const uint8_t* px = x + (((int64_t)n * H + h) * W + ww) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float v = __bfloat162float(__float2bfloat16(fmaf((float)px[c], mul, add)));
          const float* wr = sw + ((r * 3 + s) * 3 + c) * 32 + q * 8;
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(v, wr[k], acc[k]);
        }
      }
    }
    bfx8 o;
    round_and_sum(acc, o, ssum, ssq);
    *reinterpret_cast<bfx8*>(out + ((((int64_t)n * Ho + ho) * Wo + wo) * ldc) + q * 8) = o;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      ssum[k] += __shfl_xor_sync(0xffffffffu, ssum[k], o);
      ssq[k] += __shfl_xor_sync(0xffffffffu, ssq[k], o);
    }
  }
  if (lane < 4) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      red[0][warp][lane * 8 + k] = ssum[k];
      red[1][warp][lane * 8 + k] = ssq[k];
    }
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int j = threadIdx.x >> 5, c = threadIdx.x & 31;
    float t = 0.f;
#pragma unroll
    for (int v = 0; v < 8; ++v) t += red[j][v][c];
    atomicAdd((j == 0 ? sum : sqsum) + c, t);
  }
}
void mbv2_stem_stats(const uint8_t* x, const float* w, void* out, float* sum, float* sqsum, int N, int H, int W, int ldc,
                     float mul, float add, cudaStream_t s) {
  const int blocks = capped_blocks((int64_t)N * (H / 2) * (W / 2) * 4, 256, 132 * 16);
  mbv2_stem_stats_kernel<<<blocks, 256, 0, s>>>(x, w, (__nv_bfloat16*)out, sum, sqsum, N, H, W, ldc, mul, add);
}

// ------------------------------------------------------------------------------------------------ depthwise 3x3
// x: bf16 [N, H, W, C];  w: fp32 [9][C];  y = relu6(dwconv(x) * scale + shift), stride 1 or 2, pad 1;  C % 8 == 0.
// Thread = (output pixel, 8 channels): nine 16-byte loads (neighbouring threads share them through L1), 72 FMAs, one store.
template <int STRIDE>
__global__ void __launch_bounds__(256)
dwconv3x3_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                 const float* __restrict__ shift, __nv_bfloat16* __restrict__ out, int N, int H, int W, int C, int Ho, int Wo) {
  const int cvec = C / 8;
  const int64_t total = (int64_t)N * Ho * Wo * cvec;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % cvec);
    int64_t p = i / cvec;
    const int wo = (int)(p % Wo);
    p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int h = ho * STRIDE - 1 + r;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ww = wo * STRIDE - 1 + s;
        if (ww < 0 || ww >= W) continue;
        const bfx8 v = *reinterpret_cast<const bfx8*>(x + (((int64_t)n * H + h) * W + ww) * C + cv * 8);
        const float4 w0 = *reinterpret_cast<const float4*>(w + (r * 3 + s) * C + cv * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(w + (r * 3 + s) * C + cv * 8 + 4);
        const float wk[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __bfloat1622float2(v.v[k]);
          acc[2 * k] = fmaf(f.x, wk[2 * k], acc[2 * k]);
          acc[2 * k + 1] = fmaf(f.y, wk[2 * k + 1], acc[2 * k + 1]);
        }
      }
    }
    const float4 s0 = *reinterpret_cast<const float4*>(scale + cv * 8), s1 = *reinterpret_cast<const float4*>(scale + cv * 8 + 4);
    const float4 h0 = *reinterpret_cast<const float4*>(shift + cv * 8), h1 = *reinterpret_cast<const float4*>(shift + cv * 8 + 4);
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
    bfx8 o;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float a = fminf(fmaxf(fmaf(acc[2 * k], sc[2 * k], sh[2 * k]), 0.f), 6.f);
      const float b = fminf(fmaxf(fmaf(acc[2 * k + 1], sc[2 * k + 1], sh[2 * k + 1]), 0.f), 6.f);
      o.v[k] = __floats2bfloat162_rn(a, b);
    }
    *reinterpret_cast<bfx8*>(out + i * 8) = o;
  }
}
// Register-tiled version: a thread produces TW horizontally adjacent output pixels of its 8 channels.  The one-pixel kernel
// above is L1-bound, not DRAM-bound (ncu, 256x56x56x256: 1.04 ms = 0.39 TB/s algorithmic, L1/TEX 91 % busy, 94 % hit rate,
// DRAM 9 %): per output vector it issues nine 16-byte activation loads plus eighteen 16-byte weight loads = 432 B of L1
// traffic for 32 B of result.  With TW = 4 a thread loads each input row once ((TW-1)*STRIDE + 3 vectors) and each tap's
// weights once for four outputs: 72 + 72 B (stride 1) per output vector.  Same fmaf order per output as the kernel above
// (r outer, s inner; padded taps contribute fmaf(0, w, acc) = acc), so the results are bit-identical.
template <int STRIDE, int TW>
__global__ void __launch_bounds__(256)
dwconv3x3_tiled_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                       const float* __restrict__ shift, __nv_bfloat16* __restrict__ out, int N, int H, int W, int C, int Ho,
                       int Wo) {
  constexpr int NIN = (TW - 1) * STRIDE + 3;
  const int cvec = C / 8;
  const int wt = (Wo + TW - 1) / TW;
  const int64_t total = (int64_t)N * Ho * wt * cvec;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % cvec);
    int64_t p = i / cvec;
    const int tw = (int)(p % wt);
    p /= wt;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    const int wo0 = tw * TW;
    const int wi0 = wo0 * STRIDE - 1;
    float acc[TW][8];
#pragma unroll
    for (int t = 0; t < TW; ++t)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[t][k] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int h = ho * STRIDE - 1 + r;
      if (h < 0 || h >= H) continue;
      const __nv_bfloat16* rowp = x + ((int64_t)n * H + h) * W * C + cv * 8;
      bfx8 in[NIN];
#pragma unroll
      for (int k = 0; k < NIN; ++k) {
        const int ww = wi0 + k;
        if (ww >= 0 && ww < W) {
          in[k] = *reinterpret_cast<const bfx8*>(rowp + (int64_t)ww * C);
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) in[k].v[q] = __floats2bfloat162_rn(0.f, 0.f);
        }
      }
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const float4 w0 = *reinterpret_cast<const float4*>(w + (r * 3 + s) * C + cv * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(w + (r * 3 + s) * C + cv * 8 + 4);
        const float wk[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int t = 0; t < TW; ++t) {
          const bfx8& v = in[t * STRIDE + s];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 f = __bfloat1622float2(v.v[k]);
            acc[t][2 * k] = fmaf(f.x, wk[2 * k], acc[t][2 * k]);
            acc[t][2 * k + 1] = fmaf(f.y, wk[2 * k + 1], acc[t][2 * k + 1]);
          }
        }
      }
    }
    const float4 s0 = *reinterpret_cast<const float4*>(scale + cv * 8), s1 = *reinterpret_cast<const float4*>(scale + cv * 8 + 4);
    const float4 h0 = *reinterpret_cast<const float4*>(shift + cv * 8), h1 = *reinterpret_cast<const float4*>(shift + cv * 8 + 4);
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
    __nv_bfloat16* orow = out + (((int64_t)n * Ho + ho) * Wo) * C + cv * 8;
#pragma unroll
    for (int t = 0; t < TW; ++t) {
      const int wo = wo0 + t;
      if (wo >= Wo) break;
      bfx8 o;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float a = fminf(fmaxf(fmaf(acc[t][2 * k], sc[2 * k], sh[2 * k]), 0.f), 6.f);
        const float b = fminf(fmaxf(fmaf(acc[t][2 * k + 1], sc[2 * k + 1], sh[2 * k + 1]), 0.f), 6.f);
        o.v[k] = __floats2bfloat162_rn(a, b);
      }
      *reinterpret_cast<bfx8*>(orow + (int64_t)wo * C) = o;
    }
  }
}

// tile_w: output pixels per thread along W (4 = register-tiled kernel, the default; 1 = the one-pixel kernel)
void dwconv3x3(const void* x, const float* w, const float* scale, const float* shift, void* out, int N, int H, int W, int C,
               int stride, int tile_w, cudaStream_t s) {
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  if (tile_w == 4) {
    const int64_t total = (int64_t)N * Ho * ((Wo + 3) / 4) * (C / 8);
    int64_t blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) blocks = 1;
    if (stride == 1)
      dwconv3x3_tiled_kernel<1, 4><<<(int)blocks, 256, 0, s>>>((const __nv_bfloat16*)x, w, scale, shift, (__nv_bfloat16*)out, N, H, W, C, Ho, Wo);
    else
      dwconv3x3_tiled_kernel<2, 4><<<(int)blocks, 256, 0, s>>>((const __nv_bfloat16*)x, w, scale, shift, (__nv_bfloat16*)out, N, H, W, C, Ho, Wo);
    return;
  }
  const int64_t total = (int64_t)N * Ho * Wo * (C / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  if (stride == 1)
    dwconv3x3_kernel<1><<<(int)blocks, 256, 0, s>>>((const __nv_bfloat16*)x, w, scale, shift, (__nv_bfloat16*)out, N, H, W, C, Ho, Wo);
  else
    dwconv3x3_kernel<2><<<(int)blocks, 256, 0, s>>>((const __nv_bfloat16*)x, w, scale, shift, (__nv_bfloat16*)out, N, H, W, C, Ho, Wo);
}


// Training-mode BatchNorm variant of the two kernels above: c = dwconv(x) stored as bf16 (no affine, no clamp), and the
// per-channel sum(c), sum(c^2) of the stored values.  TW = 1 or 4 output pixels per thread along W, with the fmaf order
// of dwconv3x3_tiled_kernel.  Block = 8 channel vectors (64 channels, blockIdx.x) x 32 lanes, a lane takes TW-pixel
// strips grid-stride over blockIdx.y, so a thread keeps its channels for the whole loop; its partial sums are reduced
// over the block in a fixed order (xor-shuffles, then the 8 warps), one atomicAdd per channel per CTA.
template <int STRIDE, int TW>
__global__ void __launch_bounds__(256, 2)   // 2 CTAs per SM: at most 128 registers (the TW = 4 loop wants ~130)
dwconv3x3_stats_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, __nv_bfloat16* __restrict__ out,
                       float* __restrict__ sum, float* __restrict__ sqsum, int N, int H, int W, int C, int Ho, int Wo) {
  constexpr int NIN = (TW - 1) * STRIDE + 3;
  __shared__ float red[2][8][64];
  const int cv = blockIdx.x * 8 + (threadIdx.x & 7);
  const bool active = cv < C / 8;
  const int wt = (Wo + TW - 1) / TW;
  const int64_t units = (int64_t)N * Ho * wt;
  float ssum[8], ssq[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) ssum[k] = ssq[k] = 0.f;
  if (active) {
    for (int64_t u = blockIdx.y * 32 + (threadIdx.x >> 3); u < units; u += (int64_t)gridDim.y * 32) {
      const int tw = (int)(u % wt);
      const int64_t p = u / wt;
      const int ho = (int)(p % Ho);
      const int n = (int)(p / Ho);
      const int wo0 = tw * TW;
      const int wi0 = wo0 * STRIDE - 1;
      float acc[TW][8];
#pragma unroll
      for (int t = 0; t < TW; ++t)
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[t][k] = 0.f;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int h = ho * STRIDE - 1 + r;
        if (h < 0 || h >= H) continue;
        const __nv_bfloat16* rowp = x + ((int64_t)n * H + h) * W * C + cv * 8;
        bfx8 in[NIN];
#pragma unroll
        for (int k = 0; k < NIN; ++k) {
          const int ww = wi0 + k;
          if (ww >= 0 && ww < W) {
            in[k] = *reinterpret_cast<const bfx8*>(rowp + (int64_t)ww * C);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) in[k].v[q] = __floats2bfloat162_rn(0.f, 0.f);
          }
        }
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const float4 w0 = *reinterpret_cast<const float4*>(w + (r * 3 + s) * C + cv * 8);
          const float4 w1 = *reinterpret_cast<const float4*>(w + (r * 3 + s) * C + cv * 8 + 4);
          const float wk[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int t = 0; t < TW; ++t) {
            const bfx8& v = in[t * STRIDE + s];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 f = __bfloat1622float2(v.v[k]);
              acc[t][2 * k] = fmaf(f.x, wk[2 * k], acc[t][2 * k]);
              acc[t][2 * k + 1] = fmaf(f.y, wk[2 * k + 1], acc[t][2 * k + 1]);
            }
          }
        }
      }
      __nv_bfloat16* orow = out + (((int64_t)n * Ho + ho) * Wo) * C + cv * 8;
#pragma unroll
      for (int t = 0; t < TW; ++t) {
        const int wo = wo0 + t;
        if (wo >= Wo) break;
        bfx8 o;
        round_and_sum(acc[t], o, ssum, ssq);
        *reinterpret_cast<bfx8*>(orow + (int64_t)wo * C) = o;
      }
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    ssum[k] += __shfl_xor_sync(0xffffffffu, ssum[k], 8);
    ssum[k] += __shfl_xor_sync(0xffffffffu, ssum[k], 16);
    ssq[k] += __shfl_xor_sync(0xffffffffu, ssq[k], 8);
    ssq[k] += __shfl_xor_sync(0xffffffffu, ssq[k], 16);
  }
  if (lane < 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      red[0][warp][lane * 8 + k] = ssum[k];
      red[1][warp][lane * 8 + k] = ssq[k];
    }
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int j = threadIdx.x >> 6, e = threadIdx.x & 63;
    const int c = blockIdx.x * 64 + e;
    if (c < C) {
      float t = 0.f;
#pragma unroll
      for (int v = 0; v < 8; ++v) t += red[j][v][e];
      atomicAdd((j == 0 ? sum : sqsum) + c, t);
    }
  }
}
void dwconv3x3_stats(const void* x, const float* w, void* out, float* sum, float* sqsum, int N, int H, int W, int C,
                     int stride, int tile_w, cudaStream_t s) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const int gx = (C / 8 + 7) / 8;
  const int gy = capped_blocks((int64_t)N * Ho * ((Wo + tile_w - 1) / tile_w), 32, (132 * 8 + gx - 1) / gx);
  const dim3 grid(gx, gy);
  auto X = (const __nv_bfloat16*)x;
  auto O = (__nv_bfloat16*)out;
  if (tile_w == 4) {
    if (stride == 1) dwconv3x3_stats_kernel<1, 4><<<grid, 256, 0, s>>>(X, w, O, sum, sqsum, N, H, W, C, Ho, Wo);
    else             dwconv3x3_stats_kernel<2, 4><<<grid, 256, 0, s>>>(X, w, O, sum, sqsum, N, H, W, C, Ho, Wo);
  } else {
    if (stride == 1) dwconv3x3_stats_kernel<1, 1><<<grid, 256, 0, s>>>(X, w, O, sum, sqsum, N, H, W, C, Ho, Wo);
    else             dwconv3x3_stats_kernel<2, 1><<<grid, 256, 0, s>>>(X, w, O, sum, sqsum, N, H, W, C, Ho, Wo);
  }
}

}  // namespace b200
