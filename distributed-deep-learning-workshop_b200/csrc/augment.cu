// Random data augmentation inside the training step (flip, rotation, zoom, translation), on the uint8 NHWC batch ahead
// of the stem.  Two launches per step:
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
// models/augment.py reproduces both kernels bit for bit.  Draw k of image n is hash_u32(key, step, 8 n + k):
//   k = 0: flip bits (bit 0 horizontal, bit 1 vertical, kept only where the flip mode allows them)
//   k = 1: rotation table index (top 12 bits)     k = 2: zoom        k = 3 / 4: x / y translation   (top 16 bits)
#include <cuda_runtime.h>
#include <stdint.h>

#include "hash.cuh"
#include "ops_api.h"

namespace b200 {

// ------------------------------------------------------------------------------------------------ per-image parameters
__global__ void __launch_bounds__(256)
augment_params_kernel(int4* __restrict__ out, const int32_t* __restrict__ step, const int2* __restrict__ rot, int N, int H,
                      int W, uint32_t key, int flip_mode, int32_t zq, int32_t txq, int32_t tyq) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const uint32_t t = (uint32_t)*step;
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
  out[2 * n] = make_int4((int)a00, (int)a01, (int)b0, (int)a10);
  out[2 * n + 1] = make_int4((int)a11, (int)b1, hf | (vf << 1), 0);
}

void augment_params(int32_t* params, const int32_t* step, const int32_t* rot_table, int N, int H, int W, uint32_t key,
                    int flip_mode, int32_t zq, int32_t txq, int32_t tyq, cudaStream_t s) {
  augment_params_kernel<<<(N + 255) / 256, 256, 0, s>>>((int4*)params, step, (const int2*)rot_table, N, H, W, key,
                                                        flip_mode, zq, txq, tyq);
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
      const int sx = A.x * xo + A.y * y + A.z, sy = A.w * xo + B.x * y + B.y;
      const int fx = (sx >> 8) & 255, fy = (sy >> 8) & 255;
      bool vx0, vx1, vy0, vy1;
      const int ix0 = tap_index(sx >> 16, W, reflect, vx0), ix1 = tap_index((sx >> 16) + 1, W, reflect, vx1);
      const int iy0 = tap_index(sy >> 16, H, reflect, vy0), iy1 = tap_index((sy >> 16) + 1, H, reflect, vy1);
      const uint8_t* img = x + (int64_t)n * HW * 3;
      int p00[3], p01[3], p10[3], p11[3];
      row_taps(img + (int64_t)iy0 * W * 3, vy0, ix0, vx0, ix1, vx1, fill, p00, p01);
      row_taps(img + (int64_t)iy1 * W * 3, vy1, ix0, vx0, ix1, vx1, fill, p10, p11);
      const int w00 = (256 - fx) * (256 - fy), w01 = fx * (256 - fy), w10 = (256 - fx) * fy, w11 = fx * fy;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        tile[j * 3 + c] =
            (uint8_t)((uint32_t)(w00 * p00[c] + w01 * p01[c] + w10 * p10[c] + w11 * p11[c] + 32768) >> 16);
      xo += step_x;
      if (xo >= W) { xo -= W; ++y; }
      y += step_y;
      while (y >= H) { y -= H; ++n; }
    }
    __syncthreads();
    uint8_t* o = out + base * 3;
    const int nbytes = count * 3, nvec = nbytes / 16;
    for (int i = threadIdx.x; i < nvec; i += kWarpThreads)
      reinterpret_cast<uint4*>(o)[i] = reinterpret_cast<const uint4*>(tile)[i];
    for (int i = nvec * 16 + threadIdx.x; i < nbytes; i += kWarpThreads) o[i] = tile[i];
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

}  // namespace b200
