// Plain (torch-free) interface between the CUDA translation units and the pybind layer.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_params.h"

namespace b200 {

struct ConvPlanRaw {
  CUtensorMap tmA[4];
  CUtensorMap tmB;
  CUtensorMap tmD;
  CUtensorMap tmY;  // stats mode 2: pre-BN tensor on the output's geometry
  ConvParams p;
  int block_n;
  int grid;
  int stats;  // 0 none, 1 forward BN statistics, 2 fused BN-backward reduction, 3 block-gradient merge + reduction
  int halo;   // 1: halo mode (needs res_b); tmA[1] is the [bw x (bh+2)] halo map of view 0
  int res_b;  // 1: the CTA's whole filter slice stays resident in shared memory (block_n == 64, n_blocks == 1, <= 9 tiles)
};

// dims/strides innermost first; strides in BYTES for dims 1..rank-1; SWIZZLE_128B, zero OOB fill.
CUtensorMap encode_bf16(void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box);
void conv_plan_launch(const ConvPlanRaw& plan, cudaStream_t stream);

struct WgradPlanRaw {
  CUtensorMap tmDY;     // grad of conv output, NHWC view, box (64ch, bw, bh, bn)
  CUtensorMap tmX[4];   // input views (parity views for strided convs)
  WgradParams p;
  int grid;
};
void wgrad_plan_launch(const WgradPlanRaw& plan, cudaStream_t stream);

struct StemPlanRaw {
  CUtensorMap tmW;  // forward: bf16 [64 co, 192 k] weights
  CUtensorMap tmY;  // forward: output [M, 64];  wgrad: dY [M, 64]
  StemParams p;
  int grid;
};
void stem_fwd_launch(const StemPlanRaw& plan, cudaStream_t stream);
void stem_wgrad_launch(const StemPlanRaw& plan, cudaStream_t stream);
struct TmaProbeParams {
  int mode;        // 0: 2-D [pixels, C] map, 1: 4-D NHWC map with a (bw, bh, bn) pixel box
  int box_bytes;   // bytes one load brings in (rows * 128)
  int stages;
  int loads_per_cta;
  int bw, bh, bn;
  int tiles_w, tiles_h, tiles_n;  // 4-D: how many distinct box positions exist (walked round-robin, offset per CTA)
  int m_tiles;                    // 2-D: number of 128-row tiles
  int dw, dh;                     // 4-D: coordinate offset (a filter tap), exercises the out-of-bounds path
};
// TMA load-throughput probe (csrc/tma_probe.cu): box loads into a ring of stages, consumer only releases them.
void tma_probe_launch(const CUtensorMap& tm, const TmaProbeParams& p, int grid, cudaStream_t s);

}  // namespace b200
