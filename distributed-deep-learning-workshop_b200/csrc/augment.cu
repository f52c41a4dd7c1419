// Random data augmentation inside the training step (flip, rotation, zoom, translation, and MixUp or CutMix), on the
// uint8 NHWC batch ahead of the stem.  Two launches per step:
//
//   augment_params  one thread per image: draws the image's transform from the counter-based hash (csrc/hash.cuh) keyed
//                   by (seed, rank) and the step word, which it reads from DEVICE memory (a replayed CUDA graph sees the
//                   step the host wrote before the replay, not a value frozen at capture), and writes one int32 row
//                   [a00 a01 b0 a10 a11 b1 flags 0]: a Q16.16 inverse-affine map from output pixel (x, y) to source pixel
//                   coordinates  sx = a00*x + a01*y + b0,  sy = a10*x + a11*y + b1  (pixel centres at integers).
//   augment_warp    bilinear resampling of every output pixel from that map, with reflect or constant fill per tap;
//                   neighbouring lanes own neighbouring pixels, and each block writes its tile with 16-byte stores.
//
// Everything on the device is integer arithmetic: the (cos, sin) of the rotation angles come from a host-built Q16.16
// table, zoom and translation are Q16.16 products of hash bits, and the bilinear blend uses weights quantised to 1/256.
// models/augment.py reproduces every kernel bit for bit.  Draw k of image n is hash_u32(key, step, 8 n + k):
//   k = 0: flip bits (bit 0 horizontal, bit 1 vertical, kept only where the flip mode allows them)
//   k = 1: rotation table index (top 12 bits)     k = 2: zoom        k = 3 / 4: x / y translation   (top 16 bits)
//   k = 5: lambda table index (top 12 bits)       k = 6 / 7: CutMix box centre x / y (top 16 bits)
// and the batch's partner rotation is hash_u32(key, step, 8 N).  With MixUp or CutMix on, augment_mix_params and
// augment_mix_warp take the places of augment_params and augment_warp: still two launches.
#include <cuda_runtime.h>
#include <stdint.h>

#include "hash.cuh"
#include "ops_api.h"

namespace b200 {

// ------------------------------------------------------------------------------------------------ per-image parameters
// The geometric row of image n at step t (draws 0..4): [a00 a01 b0 a10 a11 b1 flags 0] as two int4.
__device__ __forceinline__ void geometric_row(int n, uint32_t t, uint32_t key, const int2* __restrict__ rot, int H,
                                              int W, int flip_mode, int32_t zq, int32_t txq, int32_t tyq, int4& lo,
                                              int4& hi) {
  const uint32_t c = (uint32_t)n * 8u;
  const uint32_t r0 = hash_u32(key, t, c), r1 = hash_u32(key, t, c + 1), r2 = hash_u32(key, t, c + 2);
  const uint32_t r3 = hash_u32(key, t, c + 3), r4 = hash_u32(key, t, c + 4);
  const int hf = (flip_mode & 1) ? (int)(r0 & 1u) : 0;
  const int vf = (flip_mode & 2) ? (int)((r0 >> 1) & 1u) : 0;
  const int2 cs = rot[r1 >> (32 - kAugRotBits)];
  // uniform in [-q, q) on a 2^-16 grid: -q + floor(2 q u / 2^16), u = top 16 bits of the draw
  const int64_t s = 65536 - zq + ((2 * (int64_t)zq * (int64_t)(r2 >> 16)) >> 16);
  const int64_t tx = -txq + ((2 * (int64_t)txq * (int64_t)(r3 >> 16)) >> 16);
  const int64_t ty = -tyq + ((2 * (int64_t)tyq * (int64_t)(r4 >> 16)) >> 16);
  const int64_t mc = (s * cs.x + 32768) >> 16, ms = (s * cs.y + 32768) >> 16;
  // A = s * Flip * Rot;  source = centre + A (out - centre - t)
  const int64_t a00 = hf ? -mc : mc, a01 = hf ? ms : -ms, a10 = vf ? -ms : ms, a11 = vf ? -mc : mc;
  const int64_t b0 = (int64_t)(W - 1) * 32768 - ((a00 * (W - 1) + a01 * (H - 1)) >> 1) - ((a00 * tx + a01 * ty) >> 16);
  const int64_t b1 = (int64_t)(H - 1) * 32768 - ((a10 * (W - 1) + a11 * (H - 1)) >> 1) - ((a10 * tx + a11 * ty) >> 16);
  lo = make_int4((int)a00, (int)a01, (int)b0, (int)a10);
  hi = make_int4((int)a11, (int)b1, hf | (vf << 1), 0);
}

__global__ void __launch_bounds__(256)
augment_params_kernel(int4* __restrict__ out, const int32_t* __restrict__ step, const int2* __restrict__ rot, int N, int H,
                      int W, uint32_t key, int flip_mode, int32_t zq, int32_t txq, int32_t tyq) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  int4 lo, hi;
  geometric_row(n, (uint32_t)*step, key, rot, H, W, flip_mode, zq, txq, tyq, lo, hi);
  out[2 * n] = lo;
  out[2 * n + 1] = hi;
}

void augment_params(int32_t* params, const int32_t* step, const int32_t* rot_table, int N, int H, int W, uint32_t key,
                    int flip_mode, int32_t zq, int32_t txq, int32_t tyq, cudaStream_t s) {
  augment_params_kernel<<<(N + 255) / 256, 256, 0, s>>>((int4*)params, step, (const int2*)rot_table, N, H, W, key,
                                                        flip_mode, zq, txq, tyq);
}

// The geometric row and the mix row of every image in one launch.  Mix row: [partner, w, x0, y0, x1, y1, num, den].
//   partner(n) = (n + s) mod N with s = 1 + hash(key, t, 8 N) mod (N - 1): one rotation of the batch per step, so no
//                image is its own partner (N = 1: image 0 mixes with itself);
//   draw 5      the lambda-table row (top kAugLamBits bits);  draws 6 / 7: the CutMix box centre (top 16 bits).
//   MixUp:  w = (Q16 lambda + 128) >> 8 (the own image's weight in 1/256), mu = (256 - w) / 256.
//   CutMix: box side (W, H) * sqrt(1 - lambda) around the centre, clipped to the image; mu = clipped area / (H W).
__global__ void __launch_bounds__(256)
augment_mix_params_kernel(int4* __restrict__ out, int4* __restrict__ mix, const int32_t* __restrict__ step,
                          const int2* __restrict__ rot, const int2* __restrict__ lam, int N, int H, int W, uint32_t key,
                          int flip_mode, int32_t zq, int32_t txq, int32_t tyq, int mode) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const uint32_t t = (uint32_t)*step;
  int4 lo, hi;
  geometric_row(n, t, key, rot, H, W, flip_mode, zq, txq, tyq, lo, hi);
  out[2 * n] = lo;
  out[2 * n + 1] = hi;
  const uint32_t c = (uint32_t)n * 8u;
  const int shift = N > 1 ? 1 + (int)(hash_u32(key, t, (uint32_t)N * 8u) % (uint32_t)(N - 1)) : 0;
  const int partner = (n + shift) % N;
  const int2 lq = lam[hash_u32(key, t, c + 5) >> (32 - kAugLamBits)];
  if (mode == kMixUp) {
    const int w = (lq.x + 128) >> 8;
    mix[2 * n] = make_int4(partner, w, 0, 0);
    mix[2 * n + 1] = make_int4(0, 0, 256 - w, 256);
  } else {
    const int cx = (int)(((uint32_t)W * (hash_u32(key, t, c + 6) >> 16)) >> 16);
    const int cy = (int)(((uint32_t)H * (hash_u32(key, t, c + 7) >> 16)) >> 16);
    const int hw = ((W * lq.y + 32768) >> 16) >> 1, hh = ((H * lq.y + 32768) >> 16) >> 1;
    const int x0 = min(max(cx - hw, 0), W), x1 = min(max(cx + hw, 0), W);
    const int y0 = min(max(cy - hh, 0), H), y1 = min(max(cy + hh, 0), H);
    mix[2 * n] = make_int4(partner, 0, x0, y0);
    mix[2 * n + 1] = make_int4(x1, y1, (x1 - x0) * (y1 - y0), H * W);
  }
}

void augment_mix_params(int32_t* params, int32_t* mix, const int32_t* step, const int32_t* rot_table,
                        const int32_t* lam_table, int N, int H, int W, uint32_t key, int flip_mode, int32_t zq,
                        int32_t txq, int32_t tyq, int mode, cudaStream_t s) {
  augment_mix_params_kernel<<<(N + 255) / 256, 256, 0, s>>>((int4*)params, (int4*)mix, step, (const int2*)rot_table,
                                                            (const int2*)lam_table, N, H, W, key, flip_mode, zq, txq,
                                                            tyq, mode);
}

// ------------------------------------------------------------------------------------------------ bilinear warp
// Tap index along one axis of extent n, and whether it reads the image: reflect is symmetric ("d c b a | a b c d |
// d c b a", period 2n); constant fill marks an outside tap invalid (its address is clamped to 0, its value replaced).
__device__ __forceinline__ int tap_index(int i, int n, bool reflect, bool& valid) {
  valid = (unsigned)i < (unsigned)n;
  if (valid) return i;
  if (!reflect) return 0;
  valid = true;
  int m = i % (2 * n);
  if (m < 0) m += 2 * n;
  return m < n ? m : 2 * n - 1 - m;
}

constexpr int kWarpThreads = 256;
constexpr int kWarpPix = 8;                              // output pixels per thread
constexpr int kWarpTile = kWarpThreads * kWarpPix;      // consecutive output pixels (of the flattened batch) per block
constexpr int kWarpTileBytes = kWarpTile * 3;            // 6144: a multiple of 16

// The two horizontal taps ix0 / ix1 of one source row, 3 channels each.  When both read the row and are neighbours
// (every tap pair away from the image border), their 6 bytes come from two or three aligned 4-byte loads; otherwise
// byte by byte, with `fill` for a tap outside the image.  (An aligned word that holds a byte of the row is readable.)
__device__ __forceinline__ void row_taps(const uint8_t* __restrict__ row, bool vy, int ix0, bool v0, int ix1, bool v1,
                                         int fill, int (&a)[3], int (&b)[3]) {
  if (vy && v0 && v1 && ix1 == ix0 + 1) {
    const uintptr_t addr = reinterpret_cast<uintptr_t>(row + ix0 * 3);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(addr & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(addr & 3) * 8;
    const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1);
    const uint32_t w2 = sh > 16 ? __ldg(w + 2) : 0u;   // bytes o .. o+5 of the words reach the third one only at o = 3
    const uint32_t lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);
    a[0] = lo & 255u; a[1] = (lo >> 8) & 255u; a[2] = (lo >> 16) & 255u;
    b[0] = lo >> 24; b[1] = hi & 255u; b[2] = (hi >> 8) & 255u;
    return;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    a[c] = (vy && v0) ? __ldg(row + ix0 * 3 + c) : fill;
    b[c] = (vy && v1) ? __ldg(row + ix1 * 3 + c) : fill;
  }
}

// Output pixel (xo, y) of one image warped by its map (A, B): the bilinear blend of its four taps, 0..255 per channel.
__device__ __forceinline__ void warp_pixel(const uint8_t* __restrict__ img, const int4& A, const int4& B, int xo, int y,
                                           int H, int W, int reflect, int fill, int (&v)[3]) {
  const int sx = A.x * xo + A.y * y + A.z, sy = A.w * xo + B.x * y + B.y;
  const int fx = (sx >> 8) & 255, fy = (sy >> 8) & 255;
  bool vx0, vx1, vy0, vy1;
  const int ix0 = tap_index(sx >> 16, W, reflect, vx0), ix1 = tap_index((sx >> 16) + 1, W, reflect, vx1);
  const int iy0 = tap_index(sy >> 16, H, reflect, vy0), iy1 = tap_index((sy >> 16) + 1, H, reflect, vy1);
  int p00[3], p01[3], p10[3], p11[3];
  row_taps(img + (int64_t)iy0 * W * 3, vy0, ix0, vx0, ix1, vx1, fill, p00, p01);
  row_taps(img + (int64_t)iy1 * W * 3, vy1, ix0, vx0, ix1, vx1, fill, p10, p11);
  const int w00 = (256 - fx) * (256 - fy), w01 = fx * (256 - fy), w10 = (256 - fx) * fy, w11 = fx * fy;
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = (int)((uint32_t)(w00 * p00[c] + w01 * p01[c] + w10 * p10[c] + w11 * p11[c] + 32768) >> 16);
}

// The staged tile leaves as 16-byte stores of consecutive addresses (a ragged tail byte by byte).
__device__ __forceinline__ void store_tile(uint8_t* __restrict__ o, const uint8_t* tile, int count) {
  const int nbytes = count * 3, nvec = nbytes / 16;
  for (int i = threadIdx.x; i < nvec; i += kWarpThreads)
    reinterpret_cast<uint4*>(o)[i] = reinterpret_cast<const uint4*>(tile)[i];
  for (int i = nvec * 16 + threadIdx.x; i < nbytes; i += kWarpThreads) o[i] = tile[i];
}

// One block per tile of 2048 consecutive output pixels.  Pixel k of thread t is tile pixel k * 256 + t, so the 32 lanes
// of a warp resample 32 neighbouring pixels and the tap loads of a warp touch a few cache lines.  The 3-byte results
// are staged in shared memory and the tile leaves as 16-byte stores of consecutive addresses.
__global__ void __launch_bounds__(kWarpThreads, 6)
augment_warp_kernel(const uint8_t* __restrict__ x, uint8_t* __restrict__ out, const int4* __restrict__ params, int N,
                    int H, int W, int reflect, int fill) {
  __shared__ __align__(16) uint8_t tile[kWarpTileBytes];
  const int HW = H * W;
  const int64_t total = (int64_t)N * HW;
  const int64_t tiles = (total + kWarpTile - 1) / kWarpTile;
  const int step_y = kWarpThreads / W, step_x = kWarpThreads - step_y * W;   // a thread's next pixel: 256 further
  for (int64_t ti = blockIdx.x; ti < tiles; ti += gridDim.x) {
    const int64_t base = ti * kWarpTile;
    const int count = (int)min((int64_t)kWarpTile, total - base);
    const int64_t p = base + threadIdx.x;
    int n = (int)(p / HW);
    const int r = (int)(p - (int64_t)n * HW);
    int y = r / W, xo = r - y * W;
    int pn = -1;
    int4 A, B;
    for (int k = 0; k < kWarpPix; ++k) {
      const int j = k * kWarpThreads + threadIdx.x;
      if (j >= count) break;
      if (n != pn) {
        A = __ldg(params + 2 * n);
        B = __ldg(params + 2 * n + 1);
        pn = n;
      }
      int v[3];
      warp_pixel(x + (int64_t)n * HW * 3, A, B, xo, y, H, W, reflect, fill, v);
#pragma unroll
      for (int c = 0; c < 3; ++c) tile[j * 3 + c] = (uint8_t)v[c];
      xo += step_x;
      if (xo >= W) { xo -= W; ++y; }
      y += step_y;
      while (y >= H) { y -= H; ++n; }
    }
    __syncthreads();
    store_tile(out + base * 3, tile, count);
    __syncthreads();   // the tile buffer is refilled by the next iteration
  }
}

void augment_warp(const uint8_t* x, uint8_t* out, const int32_t* params, int N, int H, int W, bool reflect, int fill,
                  cudaStream_t s) {
  // at most one wave of resident blocks: every block then loops over the same number of tiles (+-1), where a grid
  // larger than one wave would leave its late blocks running alone at the end
  static int resident = 0;
  if (resident == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, augment_warp_kernel, kWarpThreads, 0);
    resident = sms * per_sm > 0 ? sms * per_sm : kAugWarpMaxBlocks;
  }
  int64_t blocks = ((int64_t)N * H * W + kWarpTile - 1) / kWarpTile;
  blocks = blocks < resident ? blocks : resident;
  if (blocks > kAugWarpMaxBlocks) blocks = kAugWarpMaxBlocks;
  augment_warp_kernel<<<(int)blocks, kWarpThreads, 0, s>>>(x, out, (const int4*)params, N, H, W, reflect ? 1 : 0, fill);
}

// ------------------------------------------------------------------------------------------------ mixing warp
// augment_warp's tiling (2048-pixel tiles, shared-memory staging, 16-byte stores, one wave of blocks) with the partner
// image mixed in.  MODE == kMixUp: out = (w * own + (256 - w) * partner + 128) >> 8, both bilinear warps rounded as
// augment_warp rounds them, so every pixel gathers the taps of two images.  MODE == kCutMix: pixels inside the box
// are the partner's warped pixel, the others the image's own; each pixel gathers from one image only.  A partner index
// outside the batch (a malformed mix row) mixes the image with itself instead of reading outside x.
template <int MODE>
__global__ void __launch_bounds__(kWarpThreads, 4)
augment_mix_warp_kernel(const uint8_t* __restrict__ x, uint8_t* __restrict__ out, const int4* __restrict__ params,
                        const int4* __restrict__ mix, int N, int H, int W, int reflect, int fill) {
  __shared__ __align__(16) uint8_t tile[kWarpTileBytes];
  const int HW = H * W;
  const int64_t total = (int64_t)N * HW;
  const int64_t tiles = (total + kWarpTile - 1) / kWarpTile;
  const int step_y = kWarpThreads / W, step_x = kWarpThreads - step_y * W;
  for (int64_t ti = blockIdx.x; ti < tiles; ti += gridDim.x) {
    const int64_t base = ti * kWarpTile;
    const int count = (int)min((int64_t)kWarpTile, total - base);
    const int64_t p = base + threadIdx.x;
    int n = (int)(p / HW);
    const int r = (int)(p - (int64_t)n * HW);
    int y = r / W, xo = r - y * W;
    int pn = -1, q = 0;
    int4 A, B, PA, PB, M0, M1;
    for (int k = 0; k < kWarpPix; ++k) {
      const int j = k * kWarpThreads + threadIdx.x;
      if (j >= count) break;
      if (n != pn) {
        A = __ldg(params + 2 * n);
        B = __ldg(params + 2 * n + 1);
        M0 = __ldg(mix + 2 * n);
        M1 = __ldg(mix + 2 * n + 1);
        q = (unsigned)M0.x < (unsigned)N ? M0.x : n;
        PA = __ldg(params + 2 * q);
        PB = __ldg(params + 2 * q + 1);
        pn = n;
      }
      int v[3];
      if (MODE == kMixUp) {
        int u[3];
        warp_pixel(x + (int64_t)n * HW * 3, A, B, xo, y, H, W, reflect, fill, v);
        warp_pixel(x + (int64_t)q * HW * 3, PA, PB, xo, y, H, W, reflect, fill, u);
        const int w = M0.y;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = (w * v[c] + (256 - w) * u[c] + 128) >> 8;
      } else {
        const bool in = xo >= M0.z && xo < M1.x && y >= M0.w && y < M1.y;
        warp_pixel(x + (int64_t)(in ? q : n) * HW * 3, in ? PA : A, in ? PB : B, xo, y, H, W, reflect, fill, v);
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) tile[j * 3 + c] = (uint8_t)v[c];
      xo += step_x;
      if (xo >= W) { xo -= W; ++y; }
      y += step_y;
      while (y >= H) { y -= H; ++n; }
    }
    __syncthreads();
    store_tile(out + base * 3, tile, count);
    __syncthreads();
  }
}

template <int MODE>
static void launch_mix_warp(const uint8_t* x, uint8_t* out, const int32_t* params, const int32_t* mix, int N, int H,
                            int W, bool reflect, int fill, cudaStream_t s) {
  static int resident = 0;   // one wave of resident blocks, as augment_warp
  if (resident == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, augment_mix_warp_kernel<MODE>, kWarpThreads, 0);
    resident = sms * per_sm > 0 ? sms * per_sm : kAugWarpMaxBlocks;
  }
  int64_t blocks = ((int64_t)N * H * W + kWarpTile - 1) / kWarpTile;
  blocks = blocks < resident ? blocks : resident;
  if (blocks > kAugWarpMaxBlocks) blocks = kAugWarpMaxBlocks;
  augment_mix_warp_kernel<MODE><<<(int)blocks, kWarpThreads, 0, s>>>(x, out, (const int4*)params, (const int4*)mix, N,
                                                                     H, W, reflect ? 1 : 0, fill);
}

void augment_mix_warp(const uint8_t* x, uint8_t* out, const int32_t* params, const int32_t* mix, int N, int H, int W,
                      int mode, bool reflect, int fill, cudaStream_t s) {
  if (mode == kMixUp)
    launch_mix_warp<kMixUp>(x, out, params, mix, N, H, W, reflect, fill, s);
  else
    launch_mix_warp<kCutMix>(x, out, params, mix, N, H, W, reflect, fill, s);
}

}  // namespace b200
