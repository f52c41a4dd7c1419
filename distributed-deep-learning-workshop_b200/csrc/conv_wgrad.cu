// Weight-gradient convolution kernel for sm_90a (wgmma + TMA), split-K over pixels.
//
//   dW[tap][co][ci] += sum_px dY[px, co] * X_tap[px, ci]
//
// Both operands are "MN-major" for the tensor core (the reduction index, the pixel, is the slow smem dimension):
// the very same TMA boxes the forward kernel loads ([P pixels] x [64 channels], SWIZZLE_128B) are consumed
// directly with the transpose flags of wgmma set, so there is no transpose pass.
// A unit of work = (pixel chunk, 128-wide co block, group of G <= 4 (tap, ci-block) chunks of one filter row).
// Warpgroup g (warps 4g .. 4g+3) owns co chunk g of the block; its 64 x (64 * G) fp32 accumulator lives in registers for
// the whole pixel chunk and is flushed once with vector atomics into the fp32 gradient buffer that the all-reduce consumes.
// Warp 8 is the TMA producer (lane j issues chunk j of a stage).
#include <stdexcept>
#include <string>

#include "conv_api.h"
#include "ptx.cuh"

namespace b200 {

constexpr int kWgMaxStages = 8;
constexpr int kWgConsumers = 256;
constexpr int kWgThreads = kWgConsumers + 32;

template <int G>
__device__ __forceinline__ void wgrad_mma(float (&acc)[32 * G], uint64_t da, uint64_t db) {
  if constexpr (G == 1) wgmma_m64n64k16<1, 1>(acc, da, db);
  else if constexpr (G == 2) wgmma_m64n128k16<1, 1>(acc, da, db);
  else if constexpr (G == 3) wgmma_m64n192k16<1, 1>(acc, da, db);
  else wgmma_m64n256k16<1, 1>(acc, da, db);
}

template <int G>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX0,
                  const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                  const __grid_constant__ CUtensorMap tmX3, const __grid_constant__ WgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  const int slot_bytes = p.P * 128;
  const int stage_bytes = (p.a_chunks + G) * slot_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes);
  uint64_t* full_bar = bars;                   // [stages]
  uint64_t* empty_bar = bars + kWgMaxStages;   // [stages]

  // provably warp-uniform (see conv_igemm.cuh)
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmX0);
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kWgConsumers / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int combos = p.co_blocks * p.groups;

  if (warp == kWgConsumers / 32) {
    // ------------------------------------------------------------------ TMA producer (one warp; lane j issues chunk j)
    // All per-chunk parameters (tensor map, channel coordinate, tap offset) are hoisted out of the k loop and the
    // <= 6 loads of a stage are issued by 6 lanes in parallel.
    const int n_loads = p.a_chunks + G;
    int stage = 0;
    uint32_t phase = 0;
    const uint32_t tx = static_cast<uint32_t>(stage_bytes);
    for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
      const int pxc = unit / combos;
      const int combo = unit - pxc * combos;
      const int cob = combo / p.groups;
      const int g = combo - cob * p.groups;
      const int r = g / p.cgroups;
      const int cbg = g - r * p.cgroups;
      const int it0 = pxc * p.iters_per_chunk;
      const int it1 = min(it0 + p.iters_per_chunk, p.iters_total);
      // this lane's load
      const CUtensorMap* my_map = &tmDY;
      int my_c = 0, my_dw = 0, my_dh = 0;
      if (lane < p.a_chunks) {
        my_c = (cob * 2 + lane) * 64;
      } else if (lane < n_loads) {
        const int j = lane - p.a_chunks;
        const int cbi = j / p.S;
        const int sx = j - cbi * p.S;
        const int tap = r * p.S + sx;
        my_c = (cbg * p.cb_per_group + cbi) * 64;
        my_dw = p.tap_dw[tap];
        my_dh = p.tap_dh[tap];
        my_map = &tmX0;
        if (p.tap_map[tap] == 1) my_map = &tmX1;
        if (p.tap_map[tap] == 2) my_map = &tmX2;
        if (p.tap_map[tap] == 3) my_map = &tmX3;
      }
      // pixel-box coordinates advance incrementally (no div/mod in the loop)
      int tw = 0, th = 0, tn = 0;
      if (p.mode == 1) {
        tw = it0 % p.tiles_w;
        const int rest = it0 / p.tiles_w;
        th = rest % p.tiles_h;
        tn = rest / p.tiles_h;
      }
      for (int it = it0; it < it1; ++it) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (lane == 0) mbar_arrive_expect_tx(&full_bar[stage], tx);
        __syncwarp();
        if (lane < n_loads) {
          uint8_t* dst = smem + stage * stage_bytes + lane * slot_bytes;
          if (p.mode == 0)
            tma_load_2d(dst, my_map, &full_bar[stage], my_c, it * p.P);
          else
            tma_load_4d(dst, my_map, &full_bar[stage], my_c, tw * p.bw + my_dw, th * p.bh + my_dh, tn * p.bn);
        }
        if (++tw == p.tiles_w) {
          tw = 0;
          if (++th == p.tiles_h) {
            th = 0;
            ++tn;
          }
        }
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: warpgroup wg <-> co chunk wg
  const int wg = warp >> 2;
  const bool active = wg < p.a_chunks;  // Cout == 64: warpgroup 1 only releases the stages
  const int rrow = (warp & 3) * 16 + (lane >> 2);  // accumulator rows rrow, rrow + 8 (output channels within the chunk)
  const int cq = (lane & 3) * 2;
  // A = dY chunk wg (M = 64 co, MN-major, one 64-wide chunk); B = the G X chunks (N = 64 G ci, MN-major, chunks one slot
  // apart = LBO).  16 pixels = two 8-row swizzle atoms = 2048 B along the (slow) K dimension -> +128 in the address field.
  const uint64_t da0 = gmma_desc_sw128(smem_u32(smem) + wg * slot_bytes, slot_bytes, 1024);
  const uint64_t db0 = gmma_desc_sw128(smem_u32(smem) + p.a_chunks * slot_bytes, slot_bytes, 1024);
  const uint32_t stage_step = static_cast<uint32_t>(stage_bytes) >> 4;
  const uint32_t full0 = smem_u32(full_bar);
  const int ksteps = p.P / 16;
  int stage = 0;
  uint32_t phase = 0;
  for (int unit = blockIdx.x; unit < p.num_units; unit += gridDim.x) {
    const int pxc = unit / combos;
    const int combo = unit - pxc * combos;
    const int cob = combo / p.groups;
    const int g = combo - cob * p.groups;
    const int r = g / p.cgroups;
    const int cbg = g - r * p.cgroups;
    const int it0 = pxc * p.iters_per_chunk;
    const int it1 = min(it0 + p.iters_per_chunk, p.iters_total);
    float acc[32 * G];
#pragma unroll
    for (int i = 0; i < 32 * G; ++i) acc[i] = 0.f;
    fence_acc(acc);
    int prev = -1;
    for (int it = it0; it < it1; ++it) {
      mbar_wait_u32(full0 + stage * 8, phase);
      if (active) {
        wgmma_fence();
        const uint64_t da_s = da0 + stage * stage_step;
        const uint64_t db_s = db0 + stage * stage_step;
        for (int ks = 0; ks < ksteps; ++ks) wgrad_mma<G>(acc, da_s + ks * 128, db_s + ks * 128);
        wgmma_commit();
        wgmma_wait<1>();
      }
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == p.stages) {
        stage = 0;
        phase ^= 1;
      }
    }
    if (active) wgmma_wait<0>();
    fence_acc(acc);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }
    if (!active) continue;
    // ---------------------------------------------------------------- flush: registers -> vector atomics
    const int co = cob * 128 + wg * 64 + rrow;
#pragma unroll
    for (int j = 0; j < G; ++j) {
      const int cbi = j / p.S;
      const int s = j - cbi * p.S;
      const int tap = r * p.S + s;
      const int ci0 = (cbg * p.cb_per_group + cbi) * 64;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2* dst = reinterpret_cast<float2*>(p.dw + (static_cast<size_t>(tap) * p.cout + co + 8 * h) * p.cin + ci0 + cq);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int i = j * 8 + q;
          atomicAdd(dst + 4 * q, make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]));
        }
      }
    }
  }
}

void wgrad_plan_launch(const WgradPlanRaw& pl, cudaStream_t s) {
  const int smem_bytes = pl.p.stages * (pl.p.a_chunks + pl.p.G) * pl.p.P * 128 + 256 + 1024;
  if (pl.p.G < 1 || pl.p.G > 4 || pl.p.stages < 1 || pl.p.stages > kWgMaxStages || smem_bytes > 232448)
    throw std::runtime_error("conv_wgrad: plan out of range (G 1..4, stages <= 8, <= 227 KB)");
  static bool attr_set[4] = {false, false, false, false};
  auto launch = [&](auto kern) {
    if (!attr_set[pl.p.G - 1]) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
      if (e != cudaSuccess)
        throw std::runtime_error(std::string("conv_wgrad: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
      attr_set[pl.p.G - 1] = true;
    }
    kern<<<pl.grid, kWgThreads, smem_bytes, s>>>(pl.tmDY, pl.tmX[0], pl.tmX[1], pl.tmX[2], pl.tmX[3], pl.p);
  };
  switch (pl.p.G) {
    case 1: launch(conv_wgrad_kernel<1>); break;
    case 2: launch(conv_wgrad_kernel<2>); break;
    case 3: launch(conv_wgrad_kernel<3>); break;
    default: launch(conv_wgrad_kernel<4>); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("conv_wgrad launch: ") + cudaGetErrorString(e));
}

}  // namespace b200
