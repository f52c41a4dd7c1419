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
// augment_mix_warp take the places of augment_params and augment_warp: still two launches.  Color augmentation adds a
// third, augment_color, in place on the warp's output (or alone, from the raw batch, when nothing else is on).
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

// ------------------------------------------------------------------------------------------------ color
// Brightness, contrast, saturation, hue and grayscale of every image, in that order, on the batch the warp wrote (in
// place) or on the raw batch.  Every channel value is v = 256 p (Q8) in int32 / int64; v is clamped to [0, 255 * 256]
// after brightness and after contrast and rounded once at the end, (v + 128) >> 8.  Draw k of image n is
// hash_u32(ckey, step, 8 n + k) with ckey = hash_u32(key, 0x436F6C72, 0) (models/augment.py color_key), so the
// geometric and mix draws are untouched:
//   k = 0: brightness delta  -bq + floor(2 bq u / 2^16)           (Q8 levels)
//   k = 1: contrast factor   f = 1 - cq + floor(2 cq u / 2^16)    (Q16)
//   k = 2: saturation factor S, likewise from sq                  (Q16)
//   k = 3: hue shift         -hq + floor(2 hq u / 2^16)           (Q16 sixths of a turn)
//   k = 4: grayscale         u < pq                               (u = top 16 bits of the draw)
// A stage whose half-range is 0 is skipped, not computed as an identity.
//
// One cluster of G CTAs per image (G in 1, 2, 4, 8).  The image's 16-pixel groups that start on a 16-pixel boundary
// of the flattened batch (48 bytes: three 16-byte accesses) are split into G contiguous slices; the pixels before the
// first and after the last whole group go byte by byte to ranks 0 and G - 1.  With contrast on, each CTA first sums
// its slice's post-brightness values into three uint64 partials in shared memory; after barrier.cluster every CTA adds
// the G partials in rank order over DSMEM, so every CTA holds the same exact sums and means, and applies the chain to
// its own slice (a slice is read twice; the second read is meant to come from L2).  A CTA arrives on a second cluster barrier after its DSMEM reads
// and waits on it before exiting, so no shared memory is released while a peer may still read it.  Without contrast
// there is no reduction and no barrier.
constexpr int kColorThreads = 256;
constexpr int kColorMax = 255 * 256;              // Q8 ceiling of a channel
constexpr uint32_t kGrayR = 19589, kGrayG = 38470, kGrayB = 7471;   // rint(65536 x (0.2989, 0.5870, 0.1140))
enum ColorStage : int { kBright = 1, kContrast = 2, kSaturate = 4, kHue = 8, kGray = 16 };

struct ColorImage {
  int flags, delta, f, sat, dh;
  int mean[3];
};

// uniform in [-q, q) on a 2^-16 grid from the top 16 bits of a draw
__device__ __forceinline__ int color_uniform(uint32_t r, int32_t q) {
  return -q + (int)((2 * (int64_t)q * (int64_t)(r >> 16)) >> 16);
}

__device__ __forceinline__ int clamp_q8(int v) { return min(max(v, 0), kColorMax); }

// Q16 fraction a / dl of a sixth of a turn, rounded half up (0 <= a <= dl; a 65536 + dl / 2 < 2^32)
__device__ __forceinline__ int hue_frac(int a, uint32_t dl) {
  return (int)(((uint32_t)a * 65536u + (dl >> 1)) / dl);
}

// Saturation, hue and grayscale of one Q8 pixel (brightness and contrast come before, per channel).
__device__ __forceinline__ void color_hsv(int& r, int& g, int& b, const ColorImage& ci) {
  if (ci.flags & kSaturate) {
    // v' = mx - (mx - v) k, k = min(S, mx / dl): value (the max) kept, saturation dl / mx scaled by k and capped at
    // 1.  S <= 1 already satisfies the cap (mx >= dl), so the division only runs above 1.  (mx - v) k <= mx 2^16.
    const int mx = max(r, max(g, b)), dl = mx - min(r, min(g, b));
    if (dl > 0) {
      const uint32_t k = ci.sat <= 65536 ? (uint32_t)ci.sat : min((uint32_t)ci.sat, ((uint32_t)mx << 16) / (uint32_t)dl);
      r = mx - (int)(((uint32_t)(mx - r) * k + 32768u) >> 16);
      g = mx - (int)(((uint32_t)(mx - g) * k + 32768u) >> 16);
      b = mx - (int)(((uint32_t)(mx - b) * k + 32768u) >> 16);
    }
  }
  if (ci.flags & kHue) {
    // hue position P in Q16 sixths of a turn (the max channel taken in the order R, G, B), rotated by dh; the pixel
    // is rebuilt from (sector, fraction) with its max and min kept
    const int mx = max(r, max(g, b)), mn = min(r, min(g, b));
    const uint32_t dl = (uint32_t)(mx - mn);
    if (dl > 0) {
      // P = base + (a / dl) sixths, a signed: (g - b) / dl around R, 2 + (b - r) / dl around G, 4 + (r - g) / dl
      // around B; |a| is rounded, so one division serves every branch
      const int a = r == mx ? g - b : g == mx ? b - r : r - g;
      const int base = r == mx ? 0 : g == mx ? 2 * 65536 : 4 * 65536;
      const int q = hue_frac(abs(a), dl);
      int P = base + (a < 0 ? -q : q);
      P = (P + ci.dh + 12 * 65536) % (6 * 65536);
      const int part = (int)(((uint32_t)(P & 65535) * dl + 32768u) >> 16);
      const int rise = mn + part, fall = mx - part;
      switch (P >> 16) {
        case 0: r = mx; g = rise; b = mn; break;
        case 1: r = fall; g = mx; b = mn; break;
        case 2: r = mn; g = mx; b = rise; break;
        case 3: r = mn; g = fall; b = mx; break;
        case 4: r = rise; g = mn; b = mx; break;
        default: r = mx; g = mn; b = fall; break;
      }
    }
  }
  if (ci.flags & kGray) {
    r = g = b = (int)((kGrayR * (uint32_t)r + kGrayG * (uint32_t)g + kGrayB * (uint32_t)b + 32768u) >> 16);
  }
}

__device__ __forceinline__ int color_bright(int p, const ColorImage& ci) {
  return (ci.flags & kBright) ? clamp_q8((p << 8) + ci.delta) : p << 8;
}

// The whole chain on one pixel's three bytes.
__device__ __forceinline__ void color_pixel(int (&p)[3], const ColorImage& ci) {
  int v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    v[c] = color_bright(p[c], ci);
    if (ci.flags & kContrast)
      v[c] = clamp_q8(ci.mean[c] + (int)(((int64_t)(v[c] - ci.mean[c]) * ci.f + 32768) >> 16));
  }
  color_hsv(v[0], v[1], v[2], ci);
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = (v[c] + 128) >> 8;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
// a uint64 in the shared memory of CTA `rank` of the cluster, at the offset of `p` in this CTA's
__device__ __forceinline__ uint64_t ld_dsmem_u64(const uint64_t* p, uint32_t rank) {
  const uint32_t local = (uint32_t)__cvta_generic_to_shared(p);
  uint32_t remote;
  uint64_t v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(rank));
  asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(remote) : "memory");
  return v;
}

__device__ __forceinline__ uint32_t byte_of(const uint32_t (&w)[12], int j) { return (w[j >> 2] >> ((j & 3) * 8)) & 255u; }

__global__ void __launch_bounds__(kColorThreads, 4)
augment_color_kernel(const uint8_t* src, uint8_t* dst, const int32_t* __restrict__ step, int HW, uint32_t ckey,
                     int32_t bq, int32_t cq, int32_t sq, int32_t hq, int32_t pq) {
  __shared__ uint64_t partial[3];
  __shared__ uint64_t warp_sum[kColorThreads / 32][3];
  __shared__ int mean_s[3];
  const int G = (int)cluster_nctarank(), rank = (int)cluster_ctarank();
  const int n = blockIdx.x / G;
  const uint32_t t = (uint32_t)*step, c8 = (uint32_t)n * 8u;

  ColorImage ci;
  ci.flags = (bq ? kBright : 0) | (cq ? kContrast : 0) | (sq ? kSaturate : 0) | (hq ? kHue : 0);
  ci.delta = bq ? color_uniform(hash_u32(ckey, t, c8), bq) : 0;
  ci.f = cq ? 65536 + color_uniform(hash_u32(ckey, t, c8 + 1), cq) : 65536;
  ci.sat = sq ? 65536 + color_uniform(hash_u32(ckey, t, c8 + 2), sq) : 65536;
  ci.dh = hq ? color_uniform(hash_u32(ckey, t, c8 + 3), hq) : 0;
  if (pq && (int32_t)(hash_u32(ckey, t, c8 + 4) >> 16) < pq) ci.flags |= kGray;

  // global pixel range of the image, its whole 16-pixel groups [g0, g1) and this CTA's share of them
  const int64_t a = (int64_t)n * HW, e = a + HW;
  const int64_t g0 = (a + 15) >> 4, g1 = max(e >> 4, g0);
  const int64_t head_end = min(g0 * 16, e), tail_begin = max(g1 * 16, head_end);
  const int64_t ng = g1 - g0;
  const int64_t gs = g0 + ng * rank / G, ge = g0 + ng * (rank + 1) / G;
  const int64_t sa = rank == 0 ? a : 0, sb = rank == 0 ? head_end : 0;                 // single pixels of this CTA
  const int64_t ta = rank == G - 1 ? tail_begin : 0, tb = rank == G - 1 ? e : 0;
  const int tid = threadIdx.x;

  if (ci.flags & kContrast) {
    uint64_t s0 = 0, s1 = 0, s2 = 0;
    for (int64_t i = gs + tid; i < ge; i += kColorThreads) {
      const uint4* p = reinterpret_cast<const uint4*>(src + i * 48);
      const uint4 q0 = p[0], q1 = p[1], q2 = p[2];
      const uint32_t w[12] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
      uint32_t u[3] = {0, 0, 0};   // 16 values of at most 255 * 256 each
#pragma unroll
      for (int j = 0; j < 48; ++j) u[j % 3] += (uint32_t)color_bright((int)byte_of(w, j), ci);
      s0 += u[0]; s1 += u[1]; s2 += u[2];
    }
    for (int64_t P = sa + tid; P < sb; P += kColorThreads) {
      s0 += (uint32_t)color_bright(src[3 * P], ci);
      s1 += (uint32_t)color_bright(src[3 * P + 1], ci);
      s2 += (uint32_t)color_bright(src[3 * P + 2], ci);
    }
    for (int64_t P = ta + tid; P < tb; P += kColorThreads) {
      s0 += (uint32_t)color_bright(src[3 * P], ci);
      s1 += (uint32_t)color_bright(src[3 * P + 1], ci);
      s2 += (uint32_t)color_bright(src[3 * P + 2], ci);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if ((tid & 31) == 0) {
      warp_sum[tid >> 5][0] = s0;
      warp_sum[tid >> 5][1] = s1;
      warp_sum[tid >> 5][2] = s2;
    }
    __syncthreads();
    if (tid < 3) {
      uint64_t s = 0;
      for (int w = 0; w < kColorThreads / 32; ++w) s += warp_sum[w][tid];
      partial[tid] = s;
    }
    cluster_arrive();   // partials visible to the cluster
    cluster_wait();
    if (tid < 3) {
      uint64_t s = 0;
      for (int q = 0; q < G; ++q) s += ld_dsmem_u64(&partial[tid], (uint32_t)q);
      mean_s[tid] = (int)((s + (uint64_t)(HW >> 1)) / (uint64_t)HW);
    }
    __syncthreads();
    cluster_arrive();   // this CTA is done reading its peers; it waits for theirs before exiting
    ci.mean[0] = mean_s[0];
    ci.mean[1] = mean_s[1];
    ci.mean[2] = mean_s[2];
  } else {
    ci.mean[0] = ci.mean[1] = ci.mean[2] = 0;
  }

  for (int64_t i = gs + tid; i < ge; i += kColorThreads) {
    const uint4* p = reinterpret_cast<const uint4*>(src + i * 48);
    const uint4 q0 = __ldcs(p), q1 = __ldcs(p + 1), q2 = __ldcs(p + 2);
    const uint32_t w[12] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
    uint32_t o[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) o[k] = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      int px[3] = {(int)byte_of(w, 3 * j), (int)byte_of(w, 3 * j + 1), (int)byte_of(w, 3 * j + 2)};
      color_pixel(px, ci);
#pragma unroll
      for (int c = 0; c < 3; ++c) o[(3 * j + c) >> 2] |= (uint32_t)px[c] << (((3 * j + c) & 3) * 8);
    }
    uint4* d = reinterpret_cast<uint4*>(dst + i * 48);
    d[0] = make_uint4(o[0], o[1], o[2], o[3]);
    d[1] = make_uint4(o[4], o[5], o[6], o[7]);
    d[2] = make_uint4(o[8], o[9], o[10], o[11]);
  }
  for (int half = 0; half < 2; ++half) {
    const int64_t lo = half ? ta : sa, hi = half ? tb : sb;
    for (int64_t P = lo + tid; P < hi; P += kColorThreads) {
      int px[3] = {src[3 * P], src[3 * P + 1], src[3 * P + 2]};
      color_pixel(px, ci);
#pragma unroll
      for (int c = 0; c < 3; ++c) dst[3 * P + c] = (uint8_t)px[c];
    }
  }
  if (ci.flags & kContrast) cluster_wait();
}

int augment_color(const uint8_t* src, uint8_t* dst, const int32_t* step, int N, int H, int W, uint32_t ckey, int32_t bq,
                  int32_t cq, int32_t sq, int32_t hq, int32_t pq, int cluster, cudaStream_t s) {
  // G: the smallest cluster that gives at least two waves of resident CTAs (at most 8), so a batch of a few dozen
  // images still spreads over every SM, and CTAs waiting at the cluster barrier leave room for others to run
  static int resident = 0;
  if (resident == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, augment_color_kernel, kColorThreads, 0);
    resident = sms * per_sm > 0 ? sms * per_sm : 132 * 4;
  }
  int G = cluster;
  if (G == 0) {
    G = 1;
    while (G < kAugColorMaxCluster && (int64_t)N * G < 2 * (int64_t)resident) G *= 2;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(N * G));
  cfg.blockDim = dim3(kColorThreads);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)G;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (cudaLaunchKernelEx(&cfg, augment_color_kernel, src, dst, step, H * W, ckey, bq, cq, sq, hq, pq) != cudaSuccess)
    return -1;
  return G;
}

}  // namespace b200
