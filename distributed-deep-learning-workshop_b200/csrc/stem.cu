// ResNet stem (7x7 stride-2 pad-3 conv on a 3-channel uint8 image) on the tensor cores, forward and weight gradient.
//
// A 3-channel pixel is 3 bytes - below TMA's 16-byte granule - so the im2col operand is built by threads:
// 256 "builder" threads gather each output pixel's 7x7x3 = 147-byte patch straight from the uint8 batch
// (L1/L2 resident), apply the input normalisation (x/127.5 - 1: the reference's `preprocess_input`, C13), convert
// to bf16 and write a [128 pixels x 192 k] tile into shared memory in the canonical SWIZZLE_128B layout
// (3 k-blocks of 128 rows x 128 B).  That single tile is
//   * the K-major A operand of the forward GEMM   y[px, co]  = sum_k patch[px, k] * W[co, k]   (wgmma, 2 x M=64, N=64)
//   * the MN-major B operand of the weight-gradient GEMM  dW[co, k] = sum_px dy[px, co] * patch[px, k]  (N=192)
// so the preprocess kernel, the bf16 copy of the input and cuDNN's padded-NHWC stem kernels all disappear.
// Forward fuses the BatchNorm statistics like conv_igemm.cuh; wgrad keeps its 64x192 fp32 accumulator in the registers
// of one warpgroup for the CTA's whole pixel range and flushes once with atomics.
#include <stdexcept>
#include <string>

#include "conv_api.h"
#include "ptx.cuh"

namespace b200 {

constexpr int kStemStages = 3;
constexpr int kStemTileBytes = 3 * 128 * 128;  // 48 KB im2col tile
constexpr int kPatchRowMax = 16 + 256 * 3 + 16;
constexpr int kPatchBytes = 7 * kPatchRowMax;  // one output row needs 7 input rows (uint8, zero padded)

// A tile is ONE output row (n, ho): Wo <= 128 output pixels.
// Step 1 (all 256 builder threads): stage the 7 input rows the tile needs in shared memory with 16-byte loads;
//         rows outside the image are zero, 16 zero bytes on either side provide the horizontal padding.
// Step 2: thread (pixel m, half) converts its half of the 147-byte patch: 6 aligned LDS.32 + funnel shifts per
//         input row, PRMT into an exact integer float, FADD/FFMA normalisation, bf16 pack, 16-byte smem stores
//         into the SWIZZLE_128B tile.
// global -> registers (issued early so the latency overlaps the previous tile's build), registers -> smem
__device__ __forceinline__ void stem_ldg_patch(const StemParams& p, int tile_idx, int bt, uint4 (&v)[2]) {
  const int n = tile_idx / p.Ho;
  const int ho = tile_idx - n * p.Ho;
  const int row_vec = p.W * 3 / 16;  // W % 16 == 0
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int i = bt + q * 256;
    v[q] = make_uint4(0u, 0u, 0u, 0u);
    if (i < 7 * row_vec) {
      const int r = i / row_vec;
      const int c16 = i - r * row_vec;
      const int h = 2 * ho - 3 + r;
      if (h >= 0 && h < p.H) v[q] = *reinterpret_cast<const uint4*>(p.x + ((int64_t)(n * p.H + h) * p.W) * 3 + c16 * 16);
    }
  }
}
__device__ __forceinline__ void stem_sts_patch(const StemParams& p, uint8_t* patch, int bt, const uint4 (&v)[2]) {
  const int row_vec = p.W * 3 / 16;
  const int stride = 16 + p.W * 3 + 16;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int i = bt + q * 256;
    if (i < 7 * row_vec) {
      const int r = i / row_vec;
      const int c16 = i - r * row_vec;
      *reinterpret_cast<uint4*>(patch + r * stride + 16 + c16 * 16) = v[q];
    }
  }
}

template <int R0, int NROWS>
__device__ __forceinline__ void stem_fetch_rows(const uint8_t* patch, int stride, int wo, uint32_t (&S)[NROWS][6]) {
#pragma unroll
  for (int r = 0; r < NROWS; ++r) {
    const uint32_t a = (R0 + r) * stride + 7 + 6 * wo;  // byte address of (h, w = 2*wo-3, c = 0) in the patch
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(patch + (a & ~3u));
    const uint32_t sh = (a & 3u) * 8u;
    uint32_t w[7];
#pragma unroll
    for (int i = 0; i < 6; ++i) w[i] = wp[i];
    w[6] = 0u;
#pragma unroll
    for (int i = 0; i < 6; ++i) S[r][i] = __funnelshift_r(w[i], w[i + 1], sh);
  }
}

__device__ __forceinline__ float stem_elem(uint32_t word, int byte_in_word, float mul, float add, bool valid) {
  // byte -> exact float via the 2^23 trick (PRMT + FADD), then the input normalisation (FFMA).
  // Zero padding applies to the NORMALISED image, so out-of-image taps must produce 0 (not 0*mul+add).
  const uint32_t u = __byte_perm(word, 0x4B000000u, 0x7540u | (uint32_t)byte_in_word);
  return valid ? fmaf(__uint_as_float(u) - 8388608.0f, mul, add) : 0.f;
}

__device__ __forceinline__ void stem_build_rows(const StemParams& p, const uint8_t* patch, uint8_t* tile, int bt,
                                                int ho) {
  const int m = bt & 127;   // output pixel wo
  const int half = bt >> 7;
  if (m >= p.Wo) return;
  const int stride = 16 + p.W * 3 + 16;
  bool rv[7], cv[7];  // validity of input row 2*ho-3+r and input column 2*wo-3+s
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    rv[i] = (2 * ho - 3 + i) >= 0 && (2 * ho - 3 + i) < p.H;
    cv[i] = (2 * m - 3 + i) >= 0 && (2 * m - 3 + i) < p.W;
  }
  if (half == 0) {
    uint32_t S[5][6];  // rows 0..4 (row 4: bytes 0..11 only)
    stem_fetch_rows<0, 5>(patch, stride, m, S);
#pragma unroll
    for (int cc = 0; cc < 12; ++cc) {
      uint32_t w32[4];
#pragma unroll
      for (int e2 = 0; e2 < 4; ++e2) {
        const int k0 = cc * 8 + e2 * 2, k1 = k0 + 1;
        const float f0 = stem_elem(S[k0 / 21][(k0 % 21) >> 2], (k0 % 21) & 3, p.mul, p.add,
                                   rv[k0 / 21] && cv[(k0 % 21) / 3]);
        const float f1 = stem_elem(S[k1 / 21][(k1 % 21) >> 2], (k1 % 21) & 3, p.mul, p.add,
                                   rv[k1 / 21] && cv[(k1 % 21) / 3]);
        w32[e2] = pack_bf16x2(f0, f1);
      }
      const int kb = cc >> 3, c8 = cc & 7;
      *reinterpret_cast<uint4*>(tile + kb * (128 * 128) + m * 128 + ((c8 ^ (m & 7)) << 4)) =
          make_uint4(w32[0], w32[1], w32[2], w32[3]);
    }
  } else {
    uint32_t S[3][6];  // rows 4..6
    stem_fetch_rows<4, 3>(patch, stride, m, S);
#pragma unroll
    for (int cc = 0; cc < 7; ++cc) {  // k = 96 .. 151 (147.. are zero); chunks 12..18
      uint32_t w32[4];
#pragma unroll
      for (int e2 = 0; e2 < 4; ++e2) {
        const int k0 = 96 + cc * 8 + e2 * 2, k1 = k0 + 1;
        const float f0 = k0 < 147 ? stem_elem(S[k0 / 21 - 4][(k0 % 21) >> 2], (k0 % 21) & 3, p.mul, p.add,
                                              rv[(k0 / 21) % 7] && cv[(k0 % 21) / 3]) : 0.f;
        const float f1 = k1 < 147 ? stem_elem(S[k1 / 21 - 4][(k1 % 21) >> 2], (k1 % 21) & 3, p.mul, p.add,
                                              rv[(k1 / 21) % 7] && cv[(k1 % 21) / 3]) : 0.f;
        w32[e2] = pack_bf16x2(f0, f1);
      }
      const int chunk = 12 + cc;
      const int kb = chunk >> 3, c8 = chunk & 7;
      *reinterpret_cast<uint4*>(tile + kb * (128 * 128) + m * 128 + ((c8 ^ (m & 7)) << 4)) =
          make_uint4(w32[0], w32[1], w32[2], w32[3]);
    }
  }
}

// builder-side main loop shared by forward and wgrad; `tile_at(i)` enumerates the CTA's tiles
template <int STAGE_BYTES, class TileFn>
__device__ __forceinline__ void stem_builder_loop(const StemParams& p, uint8_t* stage_base, uint8_t* patches,
                                                  uint64_t* full_bar, uint64_t* empty_bar, int n_my_tiles, TileFn tile_at,
                                                  int bt, int lane) {
  int stage = 0;
  uint32_t phase = 0;
  uint4 pre[2];
  if (n_my_tiles > 0) stem_ldg_patch(p, tile_at(0), bt, pre);
  for (int i = 0; i < n_my_tiles; ++i) {
    uint8_t* patch = patches + (i & 1) * kPatchBytes;
    const int tile = tile_at(i);
    stem_sts_patch(p, patch, bt, pre);
    named_bar_sync(4, 256);  // patch complete; also: every builder is done with the previous tile's patch buffer
    if (i + 1 < n_my_tiles) stem_ldg_patch(p, tile_at(i + 1), bt, pre);  // prefetch: lands while this tile is built
    mbar_wait(&empty_bar[stage], phase ^ 1);
    stem_build_rows(p, patch, stage_base + stage * STAGE_BYTES, bt, tile % p.Ho);
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(&full_bar[stage]);
    if (++stage == kStemStages) { stage = 0; phase ^= 1; }
  }
}

// ------------------------------------------------------------------------------------------------ forward
// warps 0-7: two consumer warpgroups (wgmma rows 64g .. 64g+63 of the tile + epilogue), warps 8-15: im2col builders
constexpr int kStemFwdThreads = 512;
struct StemFwdSmem {
  static constexpr int kB = 3 * 64 * 128;            // weights: 3 k-blocks of [64 co x 64 k]
  static constexpr int kStaging = 2 * 128 * 128;
  static constexpr int kTotal = kStemStages * kStemTileBytes + kB + kStaging + 256 + 2 * 64 * 4 + 2 * kPatchBytes + 1024;
};

__global__ void __launch_bounds__(kStemFwdThreads, 1)
stem_fwd_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmY,
                const __grid_constant__ StemParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint8_t* sA = smem;
  uint8_t* sB = smem + kStemStages * kStemTileBytes;
  uint8_t* sStage = sB + StemFwdSmem::kB;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStage + StemFwdSmem::kStaging);
  uint64_t* full_bar = bars;                // [3]  builders -> MMA
  uint64_t* empty_bar = bars + 3;           // [3]  MMA -> builders
  uint64_t* w_bar = bars + 6;
  float* sStat = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);  // [2][64]
  uint8_t* sPatch = reinterpret_cast<uint8_t*>(sStat) + 2 * 64 * 4;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmY);
    for (int i = 0; i < kStemStages; ++i) {
      mbar_init(&full_bar[i], 8);   // one arrival per builder warp
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    mbar_init(w_bar, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 128; i += blockDim.x) sStat[i] = 0.f;
  // zero the im2col stages (rows >= Wo and the k >= 152 chunks are never written) and the patch padding
  for (int i = threadIdx.x; i < kStemStages * kStemTileBytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sA)[i] = make_uint4(0u, 0u, 0u, 0u);
  for (int i = threadIdx.x; i < 2 * kPatchBytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sPatch)[i] = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async_smem();
  __syncthreads();

  if (warp < 8) {
    // ---------------------------------------------------------------- consumers: wgmma + epilogue (256 threads)
    const int ctid = threadIdx.x;
    const int wg = warp >> 2;
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // accumulator rows row0, row0 + 8 (output pixel wo)
    if (ctid == 0) {
      // weights stay resident for the whole kernel
      mbar_arrive_expect_tx(w_bar, StemFwdSmem::kB);
      for (int kb = 0; kb < 3; ++kb) tma_load_2d(sB + kb * (64 * 128), &tmW, w_bar, kb * 64, 0);
    }
    mbar_wait(w_bar, 0);
    const uint64_t da0 = gmma_desc_sw128(smem_u32(sA) + wg * 64 * 128, 16, 1024);
    const uint64_t db0 = gmma_desc_sw128(smem_u32(sB), 16, 1024);
    int stage = 0;
    uint32_t phase = 0;
    int ctr = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++ctr) {
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      fence_acc(acc);
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
      const uint64_t da_s = da0 + static_cast<uint32_t>(stage * (kStemTileBytes >> 4));
#pragma unroll
      for (int kb = 0; kb < 3; ++kb) {
        const uint64_t da = da_s + kb * ((128 * 128) >> 4);
        const uint64_t db = db0 + kb * ((64 * 128) >> 4);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n64k16<0, 0>(acc, da + 2 * k, db + 2 * k);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == kStemStages) { stage = 0; phase ^= 1; }

      // ---------------------------------------------------------------- epilogue: registers -> bf16 -> TMA store (+ stats)
      uint8_t* sbuf = sStage + (ctr & 1) * (128 * 128);
      if (ctid == 0) tma_store_wait_read<1>();
      named_bar_sync(1, 256);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + 8 * h;
          *reinterpret_cast<uint32_t*>(sbuf + row * 128 + ((j ^ (row & 7)) << 4) + (lane & 3) * 4) =
              pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 256);
      if (ctid == 0) {
        tma_store_2d(&tmY, sbuf, 0, tile * p.Wo);
        tma_store_commit();
      }
      if (p.stat_sum != nullptr) {
        const int cp = ctid & 31, rg = ctid >> 5;
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
        const int r_end = min(rg * 16 + 16, p.Wo);
#pragma unroll 8
        for (int r = rg * 16; r < r_end; ++r) {
          const uint32_t w = *reinterpret_cast<const uint32_t*>(sbuf + r * 128 + (((cp >> 2) ^ (r & 7)) << 4) + ((cp & 3) << 2));
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
          s0 += f.x; s1 += f.y;
          q0 = fmaf(f.x, f.x, q0); q1 = fmaf(f.y, f.y, q1);
        }
        atomicAdd(&sStat[cp * 2], s0);
        atomicAdd(&sStat[cp * 2 + 1], s1);
        atomicAdd(&sStat[64 + cp * 2], q0);
        atomicAdd(&sStat[64 + cp * 2 + 1], q1);
      }
    }
    if (p.stat_sum != nullptr) {
      named_bar_sync(3, 256);
      if (ctid < 64) atomicAdd(p.stat_sum + ctid, sStat[ctid]);
      else if (ctid < 128) atomicAdd(p.stat_sqsum + (ctid - 64), sStat[ctid]);
    }
    if (ctid == 0) tma_store_wait_all<0>();
  } else {
    // ---------------------------------------------------------------- im2col builders (256 threads)
    const int bt = threadIdx.x - 256;
    const int n_my = blockIdx.x < p.num_tiles ? (p.num_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    stem_builder_loop<kStemTileBytes>(p, sA, sPatch, full_bar, empty_bar, n_my,
                                      [&](int i) { return (int)blockIdx.x + i * (int)gridDim.x; }, bt, lane);
  }
}

// ------------------------------------------------------------------------------------------------ weight gradient
// warps 0-3: one consumer warpgroup (M = 64 output channels), warps 4-11: im2col builders, warp 12: dY TMA producer
constexpr int kStemWgThreads = 416;
struct StemWgSmem {
  static constexpr int kStage = kStemTileBytes + 128 * 128;   // im2col tile + dY tile
  static constexpr int kTotal = kStemStages * kStage + 256 + 2 * kPatchBytes + 1024;
};

__global__ void __launch_bounds__(kStemWgThreads, 1)
stem_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ StemParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStemStages * StemWgSmem::kStage);
  uint64_t* full_bar = bars;      // [3]  8 builder warps + TMA producer
  uint64_t* empty_bar = bars + 3; // [3]  4 consumer warps
  uint8_t* sPatch = reinterpret_cast<uint8_t*>(bars) + 256;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmDY);
    for (int i = 0; i < kStemStages; ++i) {
      mbar_init(&full_bar[i], 9);
      mbar_init(&empty_bar[i], 4);
    }
    fence_barrier_init();
  }
  // zero all stages: pixel rows >= Wo of both operands must be exact zeros (they are never written)
  for (int i = threadIdx.x; i < kStemStages * StemWgSmem::kStage / 16; i += blockDim.x) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
  for (int i = threadIdx.x; i < 2 * kPatchBytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sPatch)[i] = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async_smem();
  __syncthreads();
  // contiguous tile range per CTA
  const int per = (p.num_tiles + gridDim.x - 1) / gridDim.x;
  const int t0 = blockIdx.x * per;
  const int t1 = min(t0 + per, p.num_tiles);

  if (warp == 12) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = t0; tile < t1; ++tile) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], p.Wo * 128);
        tma_load_2d(smem + stage * StemWgSmem::kStage + kStemTileBytes, &tmDY, &full_bar[stage], 0, tile * p.Wo);
        if (++stage == kStemStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp < 4) {
    // A = dY tile [px][64 co] (M = co, MN-major), B = im2col tile, 3 chunks of [px][64 k] 16 KB apart (N = 192, MN-major);
    // 16 pixels = two 8-row swizzle atoms = 2048 B along K
    float acc[96];
#pragma unroll
    for (int i = 0; i < 96; ++i) acc[i] = 0.f;
    fence_acc(acc);
    const int ksteps = (p.Wo + 15) / 16;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = t0; tile < t1; ++tile) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence();
      const uint32_t b0 = smem_u32(smem + stage * StemWgSmem::kStage);
      const uint32_t a0 = b0 + kStemTileBytes;
      for (int ks = 0; ks < ksteps; ++ks)
        wgmma_m64n192k16<1, 1>(acc, gmma_desc_sw128(a0 + ks * 2048, 128 * 128, 1024),
                               gmma_desc_sw128(b0 + ks * 2048, 128 * 128, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == kStemStages) { stage = 0; phase ^= 1; }
    }
    if (t1 > t0) {
      // rows = output channels, columns = k = tap * 3 + c
      const int co0 = warp * 16 + (lane >> 2);
      const int cq = (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < 24; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = i * 8 + cq + (e & 1);
          const int co = co0 + 8 * (e >> 1);
          if (k < 147) atomicAdd(p.dw + ((k / 3) * 64 + co) * 3 + (k % 3), acc[4 * i + e]);
        }
      }
    }
  } else {
    const int bt = threadIdx.x - 128;
    stem_builder_loop<StemWgSmem::kStage>(p, smem, sPatch, full_bar, empty_bar, t1 > t0 ? t1 - t0 : 0,
                                          [&](int i) { return t0 + i; }, bt, lane);
  }
}

static void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void stem_fwd_launch(const StemPlanRaw& pl, cudaStream_t s) {
  static bool attr = false;
  if (!attr) {
    check(cudaFuncSetAttribute(stem_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, StemFwdSmem::kTotal),
          "stem_fwd attr");
    attr = true;
  }
  stem_fwd_kernel<<<pl.grid, kStemFwdThreads, StemFwdSmem::kTotal, s>>>(pl.tmW, pl.tmY, pl.p);
  check(cudaGetLastError(), "stem_fwd launch");
}
void stem_wgrad_launch(const StemPlanRaw& pl, cudaStream_t s) {
  static bool attr = false;
  if (!attr) {
    check(cudaFuncSetAttribute(stem_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, StemWgSmem::kTotal),
          "stem_wgrad attr");
    attr = true;
  }
  stem_wgrad_kernel<<<pl.grid, kStemWgThreads, StemWgSmem::kTotal, s>>>(pl.tmY, pl.p);
  check(cudaGetLastError(), "stem_wgrad launch");
}

}  // namespace b200
