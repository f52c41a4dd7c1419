// Host side of the wgmma implicit-GEMM convolution: tensor-map encoding, plan object, launch.
#include <mutex>
#include <stdexcept>
#include <vector>

#include "conv_igemm.cuh"
#include "conv_api.h"

namespace b200 {

template <int BN, int ST, bool RB = false, bool HL = false>
static void launch_t(const ConvPlanRaw& pl, cudaStream_t s) {
  auto kern = conv_igemm_kernel<BN, ST, RB, HL>;
  using L = ConvSmem<BN, ST, RB, HL>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
    if (e != cudaSuccess) throw std::runtime_error(std::string("conv_igemm: cudaFuncSetAttribute: ") + cudaGetErrorString(e));
    attr_set = true;
  }
  TmapArray4 a;
  for (int i = 0; i < 4; ++i) a.m[i] = pl.tmA[i];
  kern<<<pl.grid, kConvThreads, L::kTotal, s>>>(a, pl.tmB, pl.tmD, pl.tmY, pl.p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("conv_igemm launch: ") + cudaGetErrorString(e));
}

template <int ST>
static void launch_n(const ConvPlanRaw& pl, cudaStream_t s) {
  if (pl.block_n == 128) launch_t<128, ST>(pl, s);
  else if (pl.res_b && pl.halo) launch_t<64, ST, true, true>(pl, s);
  else if (pl.res_b) launch_t<64, ST, true>(pl, s);
  else launch_t<64, ST>(pl, s);
}

void conv_plan_launch(const ConvPlanRaw& pl, cudaStream_t s) {
  if (pl.block_n != 64 && pl.block_n != 128) throw std::runtime_error("conv_igemm: block_n must be 64 or 128");
  if (pl.stats == 1) launch_n<1>(pl, s);
  else if (pl.stats == 2) launch_n<2>(pl, s);
  else if (pl.stats == 3) {
    // block-gradient merge epilogue: flat 1x1 plans only, no resident-filter / halo variants
    if (pl.block_n == 128) launch_t<128, 3>(pl, s);
    else launch_t<64, 3>(pl, s);
  } else if (pl.stats == 4) launch_n<4>(pl, s);
  else launch_n<0>(pl, s);
}

}  // namespace b200
