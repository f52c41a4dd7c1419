// Implicit-GEMM convolution (forward and data-gradient) for sm_90a.
//
//   D[m, n] = sum_{tap, c} A_tap[m, c] * B[tap][n][c]            (bf16 x bf16 -> fp32 in registers -> bf16)
//
// * A is an NHWC bf16 activation.  An M-tile is either 128 consecutive pixels of the flattened
//   [N*H*W, C] view ("flat", 1x1 stride-1 convs) or a TMA box (bw x bh x bn pixels, <=128) of the 4-D tensor
//   ("box", 3x3 / strided convs).  A filter tap is a coordinate offset of the box; zero padding is the TMA
//   out-of-bounds fill, so there is no im2col buffer.  Strided convs pass up to 4 "parity" views of the input (each a
//   strided NHWC view) and a tap table that says which view + offset each tap reads.
// * B is the filter as a [taps*Cout, Cin] K-major matrix.
// * Warp-specialised, persistent: warp 8 = TMA producer (ONE thread chosen with elect.sync, integer smem addresses;
//   warps 9-11 only complete its warpgroup so that setmaxnreg can move registers to the consumers),
//   warps 0-7 = two consumer warpgroups in ping-pong.  Warpgroup g owns the CTA's tiles g, g + 2, g + 4, ... whole: it
//   issues two wgmma.m64nBLOCK_Nk16 per k-step (A rows 0 and 64 of the stage, 128 x BLOCK_N fp32 accumulators in
//   registers), then runs the epilogue of that tile itself (bf16 -> its own swizzled staging buffers -> TMA store).
//   The epilogue of tile i overlaps the main loop of tile i+1 on the other warpgroup.  An ordering barrier hands the
//   main loop from one warpgroup to the other once all of a tile's MMAs are issued: the tensor cores see the tiles in
//   CTA order, and a warpgroup never waits on a stage of the ring more than one lap ahead of the producer (with tiles
//   of >= kStages stages that parity wait would pass on the previous lap's phase).
// * kStats = 1: after staging each 64-column chunk the warpgroup reduces per-channel sum / sum-of-squares of its staged
//   bf16 tile (register accumulators across its tiles, one global atomic per channel and 32-row group whenever its next
//   tile moves to another n-block) - no separate BatchNorm statistics pass (SURVEY.md K10).
//   kStats = 2: the same reduction for the BatchNorm-BACKWARD inside a dgrad GEMM (sum dz, sum dz*y with
//   dz = g * [y*scale + shift > 0]; the pre-BN tile y arrives by an extra TMA load).
// * kResB: the CTA's whole filter slice (<= 9 tiles of 8 KB, single N-block of 64 channels) stays resident in shared
//   memory.  kHalo (on top of kResB; 3x3 stride 1, full-width single-image boxes, width a multiple of 8): one
//   [bw x (bh+2)] box per horizontal tap offset; its three vertical taps read the same stage 0 / bw / 2*bw rows in.  With
//   bw % 8 == 0 those row offsets are whole 1024 B swizzle atoms, so the shifted descriptors stay exact.
#pragma once
#include "conv_params.h"
#include "ptx.cuh"

namespace b200 {

// kStats: 0 = plain epilogue, 1 = forward BatchNorm statistics (sum y, sum y^2), 2 = BatchNorm-backward reduction
// fused into a dgrad GEMM: the output tile is g = dL/d(activation); with the activation's pre-BN tensor y (extra TMA
// load per chunk) the consumers accumulate sum(dz), sum(dz*y) for dz = g * [y*scale + shift > 0].
// kStats = 3 (flat 1x1 dgrad of a residual block's first conv): the whole gradient merge of the PREVIOUS block's output
// happens in the epilogue - dz = (acc + skip_gradient) * relu_bitmask is what gets stored, and the consumers
// accumulate sum(dz), sum(dz*y3) for that block's final BatchNorm.  The separate reduce pass (4 tensor reads + 1 write of
// the widest activation of the block) and the store / re-read of the main-path gradient disappear.
// kStats = 4 (inference): per-channel affine (folded BatchNorm: y*scale + shift) + optional residual add (flat mode) +
// ReLU / ReLU6 applied in the epilogue - the convolution writes the block's activation directly, no BatchNorm pass at all.
// The (up to four) parity views of the A operand as ONE kernel parameter: the per-tap choice is an index.
struct TmapArray4 {
  CUtensorMap m[4];
};

// kResB: the whole filter slice this CTA needs (taps * kblocks tiles of [BLOCK_N x 64]) stays resident in shared memory
// (loaded once per CTA) and the pipeline stages carry only the A tile: a third of the bytes a 3x3 64->64 layer would
// otherwise move per tile are the same 72 KB of weights.
constexpr int kResBBytes = 9 * 64 * kBlockK * 2;  // 72 KB = nine [64 x 64] bf16 filter tiles (taps * kblocks <= 9)

constexpr int kHaloRows = 224;  // largest halo box: bw * (bh + 2) pixels (56 x 4); 28 KB per stage

constexpr int kConvConsumers = 256;                // two warpgroups
constexpr int kConvThreads = kConvConsumers + 128;  // + the producer warpgroup (one working warp)
// Register split (setmaxnreg): the kernel launches at 65536 / 384 -> 168 registers per thread; the producer warpgroup
// drops to 40 and the consumers rise to 232, room for a whole tile's 128 fp32 accumulators at BLOCK_N = 128.
// 128 * 40 + 256 * 232 = 64512 <= 65536.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
constexpr int kSmemLimit = 232448;                 // 227 KB per block
constexpr int kAlignSlack = 1024;                  // dynamic smem is rounded up to 1024 B in the kernel
constexpr int kTileChunkBytes = kBlockM * 128;     // one 128 x 64 bf16 tile chunk (16 KB)

template <int BLOCK_N, int kStats = 0, bool kResB = false, bool kHalo = false>
struct ConvSmem {
  // Per warpgroup: one pre-BN tile buffer (loaded at the start of its own chunk) and one store buffer per 64-column
  // chunk of the tile, so neither warpgroup's stores or loads wait for the other's.
  static constexpr int kYBytes = (kStats == 2 || kStats == 3) ? 2 * kTileChunkBytes : 0;  // 128x64 bf16 tiles of y
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kASlot = kHalo ? kHaloRows * 128 : kABytes;     // bytes of A per pipeline stage
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kResB ? kASlot : kASlot + kBBytes;
  static constexpr int kResBytes = kResB ? kResBBytes : 0;
  static constexpr int kStagingBytes = 2 * (BLOCK_N / 64) * kTileChunkBytes;  // per warpgroup: BLOCK_N / 64 buffers
  static constexpr int kBarBytes = 256;
  static constexpr int kFixed = kResBytes + kStagingBytes + kYBytes + kBarBytes + 16;
  static constexpr int kFit = (kSmemLimit - kAlignSlack - kFixed) / kStageBytes;  // stages that fit beside the fixed buffers
  static constexpr int kCap = kResB ? 8 : (BLOCK_N == 128 ? 5 : 6);
  static constexpr int kStages = kFit > kCap ? kCap : kFit;
  static constexpr int kTotal = kStages * kStageBytes + kFixed + kAlignSlack;
  static_assert(BLOCK_N == 64 || BLOCK_N == 128, "BLOCK_N: 64 or 128");
  static_assert(!kResB || BLOCK_N == 64, "resident filter: BLOCK_N == 64 only");
  static_assert(!kHalo || kResB, "halo mode builds on the resident filter");
  static_assert(kStages >= 2 && 2 * kStages + 3 <= kBarBytes / 8, "pipeline depth / barrier area");
  static_assert(kTotal <= kSmemLimit, "exceeds 227 KB of shared memory");
};

// Four K-steps of 16 (one 64-wide k-block, one 128 B swizzle row): +32 B = +2 in the descriptor's address field each.
// Each K-step runs twice, for A rows 0..63 into acc[0] and rows 64..127 (8 KB further: +512, whole swizzle atoms) into
// acc[1].
template <int BLOCK_N>
__device__ __forceinline__ void mma_kblock(float (&acc)[2][BLOCK_N / 2], uint64_t da, uint64_t db) {
#pragma unroll
  for (int k = 0; k < kBlockK / 16; ++k) {
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
      if constexpr (BLOCK_N == 128)
        wgmma_m64n128k16<0, 0>(acc[mh], da + mh * 512 + 2 * k, db + 2 * k);
      else
        wgmma_m64n64k16<0, 0>(acc[mh], da + mh * 512 + 2 * k, db + 2 * k);
    }
  }
}

template <int BLOCK_N, int kStats, bool kResB = false, bool kHalo = false>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_igemm_kernel(const __grid_constant__ TmapArray4 tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmY,
                  const __grid_constant__ ConvParams p) {
  using L = ConvSmem<BLOCK_N, kStats, kResB, kHalo>;
  constexpr int kStages = L::kStages;
  constexpr bool kStatsOn = kStats >= 1 && kStats <= 3;  // per-channel reductions of the staged tiles
  constexpr bool kHasY = kStats == 2 || kStats == 3;     // a pre-BN tile accompanies every output chunk
  constexpr bool kAffine = kStats == 4;                  // epilogue: acc*scale + shift (+ residual) -> activation
  constexpr int kChunks = BLOCK_N / 64;
  constexpr int kAcc = BLOCK_N / 2;                      // fp32 accumulators per thread and 64-row half of the tile
  // kStats == 3: chunk 0's skip-gradient and mask words are loaded while the tile's last MMAs drain.  At BLOCK_N = 128
  // their 40 registers beside the 128 accumulators would spill, so that tile loads chunk 0 row by row in the epilogue.
  constexpr bool kSkipEarly = BLOCK_N == 64;
  // kHasY: chunk 0's pre-BN tile is requested when the warpgroup starts the tile's main loop, instead of after it.  This
  // pays where the main loop is short next to the epilogue (kStats == 3: 1-8 k-blocks per tile) and on the BLOCK_N = 64
  // plans; the long main loops of the BLOCK_N = 128 kStats == 2 plans hide the load already, and there the early
  // request measured slower, so they keep the epilogue's request.
  constexpr bool kEarlyY = kHasY && (kStats == 3 || BLOCK_N == 64);

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint8_t* sA = smem;
  uint8_t* sB = smem + kStages * L::kASlot;  // per-stage B tiles, or (kResB) the resident filter slice
  uint8_t* sStage = smem + kStages * L::kStageBytes + L::kResBytes;
  uint8_t* sY = sStage + L::kStagingBytes;  // kHasY only
  uint64_t* bars = reinterpret_cast<uint64_t*>(sY + L::kYBytes);
  uint64_t* full_bar = bars;                     // [kStages]
  uint64_t* empty_bar = bars + kStages;          // [kStages]
  uint64_t* y_bar = bars + 2 * kStages;          // [2] (kHasY): one per warpgroup
  uint64_t* bres_bar = bars + 2 * kStages + 2;   // resident filter loaded (kResB)
  int* s_last = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(bars) + L::kBarBytes);

  // Provably warp-uniform (the compiler cannot see that threadIdx.x >> 5 is): together with elect.sync for the
  // single-thread producer this keeps the TMA / mbarrier instructions free of per-instruction serialisation loops.
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA.m[0]);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmD);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);  // one arrival per warp of the warpgroup that consumed the stage
    }
    for (int i = 0; i < 2; ++i) mbar_init(&y_bar[i], 1);
    mbar_init(bres_bar, 1);
    fence_barrier_init();
  }
  if (kHasY) {
    // rows past the pixel box are never written by TMA: keep them finite (0 * NaN would poison the sums)
    for (int i = threadIdx.x; i < L::kYBytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sY)[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async_smem();
  }
  __syncthreads();

  const int k_iters = p.taps * p.kblocks;
  const uint32_t a_bytes = (p.mode == 0 ? kBlockM : p.valid_rows) * 128;
  const uint32_t stage_tx = kHalo ? static_cast<uint32_t>(p.halo_bytes) : (kResB ? a_bytes : a_bytes + L::kBBytes);

  if (warp >= kConvConsumers / 32) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kConvConsumers / 32 && elect_one()) {
      // ---------------------------------------------------------------- TMA producer (one elected thread)
      const int taps = p.taps, kblocks = p.kblocks, n_blocks = p.n_blocks, num_tiles = p.num_tiles, cout = p.cout;
      const bool flat = p.mode == 0;
      const int tiles_w = p.tiles_w, tiles_h = p.tiles_h, bw = p.bw, bh = p.bh, bn = p.bn;
      const uint32_t sA0 = smem_u32(sA), sB0 = smem_u32(sB);
      const uint32_t full0 = smem_u32(full_bar), empty0 = smem_u32(empty_bar);
      if (kResB && static_cast<int>(blockIdx.x) < num_tiles) {
        // n_blocks == 1 (host-checked): every tile of this CTA uses the same taps * kblocks filter tiles, tile
        // (t, kb) at index t * kblocks + kb.
        mbar_arrive_expect_tx_u32(smem_u32(bres_bar), static_cast<uint32_t>(taps * kblocks) * L::kBBytes);
        for (int t = 0; t < taps; ++t)
          for (int kb = 0; kb < kblocks; ++kb)
            tma_load_2d_u32(sB0 + (t * kblocks + kb) * L::kBBytes, &tmB, smem_u32(bres_bar), kb * kBlockK, t * cout);
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_tile = tile / n_blocks;
        const int nb = tile - m_tile * n_blocks;
        int w0 = 0, h0 = 0, n0 = 0;
        if (!flat) {
          const int tw = m_tile % tiles_w;
          const int rest = m_tile / tiles_w;
          const int th = rest % tiles_h;
          w0 = tw * bw;
          h0 = th * bh;
          n0 = (rest / tiles_h) * bn;
        }
        if (kHalo) {
          // one [bw x (bh+2)] box per horizontal tap offset; rows above / below / beside the image are zero-filled
          for (int hs = 0; hs < 3; ++hs) {
            const int cw = w0 + p.halo_dw[hs];
            const int ch = h0 + p.halo_dh0;
            for (int kb = 0; kb < kblocks; ++kb) {
              mbar_wait_u32(empty0 + stage * 8, phase ^ 1);
              const uint32_t fb = full0 + stage * 8;
              mbar_arrive_expect_tx_u32(fb, stage_tx);
              tma_load_4d_u32(sA0 + stage * L::kASlot, &tmA.m[1], fb, kb * kBlockK, cw, ch, n0);
              if (++stage == kStages) {
                stage = 0;
                phase ^= 1;
              }
            }
          }
          continue;
        }
        const int m0 = m_tile * kBlockM;
        const int brow = nb * BLOCK_N;
        for (int t = 0; t < taps; ++t) {
          const CUtensorMap* am = &tmA.m[p.tap_map[t]];
          const int cw = w0 + p.tap_dw[t];
          const int ch = h0 + p.tap_dh[t];
          const int b1 = t * cout + brow;
          for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait_u32(empty0 + stage * 8, phase ^ 1);
            const uint32_t fb = full0 + stage * 8;
            mbar_arrive_expect_tx_u32(fb, stage_tx);
            if (flat)
              tma_load_2d_u32(sA0 + stage * L::kASlot, am, fb, kb * kBlockK, m0);
            else
              tma_load_4d_u32(sA0 + stage * L::kASlot, am, fb, kb * kBlockK, cw, ch, n0);
            if (!kResB) tma_load_2d_u32(sB0 + stage * L::kBBytes, &tmB, fb, kb * kBlockK, b1);
            if (++stage == kStages) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: two warpgroups (256 threads)
  setmaxnreg_inc<kConsumerRegs>();
  const int ctid = threadIdx.x;
  const int wg = warp >> 2;                       // warpgroup: the CTA's tiles wg, wg + 2, wg + 4, ...
  const int wtid = ctid & 127;                    // thread in the warpgroup
  const int r16 = (warp & 3) * 16 + (lane >> 2);  // accumulator rows of this thread: r16 + 8h + 64mh (h, mh in {0, 1})
  const int cq = (lane & 3) * 2;                  // column pair inside each 8-column group
  const uint32_t full0 = smem_u32(full_bar);
  // named barriers: 1 + wg = this warpgroup's epilogue, 3 + wg = "warpgroup wg may start its next main loop"
  // (bar.arrive by the other warpgroup + bar.sync by this one), 5 = both warpgroups before the last-CTA tail
  const uint32_t epi_bar = 1 + wg, my_turn = 3 + wg, their_turn = 4 - wg;
  // descriptors differ only in the 14-bit start-address field (addr >> 4): build once, add per stage / k-step.
  const uint64_t da0 = gmma_desc_sw128(smem_u32(sA), 16, 1024);
  const uint64_t db0 = gmma_desc_sw128(smem_u32(sB), 16, 1024);
  uint8_t* const sStageW = sStage + wg * (kChunks * kTileChunkBytes);  // this warpgroup's store buffers, one per chunk
  uint8_t* const sYW = sY + wg * kTileChunkBytes;                      // and its pre-BN tile buffer (kHasY)
  // statistics: this thread reduces column pair cp of each staged chunk over the 32 rows of row group rg
  const int cp = wtid & 31, rg = wtid >> 5;
  uint32_t xoff[8];  // byte offset of column pair cp in a row with (row & 7) == j
#pragma unroll
  for (int j = 0; j < 8; ++j) xoff[j] = (((cp >> 2) ^ j) << 4) + ((cp & 3) << 2);
  float sacc[kChunks][4];
#pragma unroll
  for (int c = 0; c < kChunks; ++c) sacc[c][0] = sacc[c][1] = sacc[c][2] = sacc[c][3] = 0.f;

  // Stages are consumed in CTA tile order, n_stages per tile: local tile i starts at ring position i * n_stages.
  const int n_stages = kHalo ? 3 * p.kblocks : k_iters;
  int ring = wg * n_stages;
  int chunk_ctr = 0;
  if (kResB && static_cast<int>(blockIdx.x) < p.num_tiles) mbar_wait(bres_bar, 0);

  for (int tile = blockIdx.x + wg * gridDim.x, i = wg; tile < p.num_tiles; tile += 2 * gridDim.x, i += 2) {
    const int m_tile = tile / p.n_blocks;
    const int nb = tile - m_tile * p.n_blocks;
    int w0 = 0, h0 = 0, n0 = 0;
    if (p.mode == 1) {
      const int tw = m_tile % p.tiles_w;
      const int rest = m_tile / p.tiles_w;
      const int th = rest % p.tiles_h;
      w0 = tw * p.bw;
      h0 = th * p.bh;
      n0 = (rest / p.tiles_h) * p.bn;
    }
    int stage = ring % kStages;
    uint32_t phase = (ring / kStages) & 1;
    ring += 2 * n_stages;

    // kStats == 3 / kAffine residual: this thread's four rows of the additive tensor (flat mode: tile row == pixel
    // index), row r16 + 8 * (q & 1) + 64 * (q >> 1) for q = 2 * mh + h.  Computed before the main loop (scalar work
    // the MMAs hide).  The loads sit in the epilogue, under the other warpgroup's MMAs, except where kStats == 3 issues
    // them earlier (skip_ld below).
    const __nv_bfloat16* arow[4] = {nullptr, nullptr, nullptr, nullptr};
    const uint8_t* mrow[4] = {nullptr, nullptr, nullptr, nullptr};
    if ((kStats == 3 || kAffine) && p.mode == 0 && (kStats == 3 || p.add_src != nullptr)) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int64_t grow = static_cast<int64_t>(m_tile) * kBlockM + r16 + 8 * (q & 1) + 64 * (q >> 1);
        if (grow < p.m_rows) {
          if (kStats == 3) mrow[q] = p.relu_mask + grow * (p.cout >> 3) + ((nb * BLOCK_N) >> 3);
          if (p.add_mode == 0) {
            arow[q] = p.add_src + grow * p.cout + nb * BLOCK_N;
          } else {
            // compact skip gradient of a stride-2 1x1 projection: only even (h, w) positions carry a value
            const int wq = static_cast<int>(grow % p.add_w);
            const int64_t t = grow / p.add_w;
            const int hq = static_cast<int>(t % p.add_h);
            const int64_t nq = t / p.add_h;
            if (((wq | hq) & 1) == 0)
              arow[q] = p.add_src + ((nq * (p.add_h >> 1) + (hq >> 1)) * (p.add_w >> 1) + (wq >> 1)) * p.cout + nb * BLOCK_N;
          }
        }
      }
    }
    // kStats == 3: row q's skip-gradient words and ReLU-mask bits of one chunk, all issued before any is used (one
    // memory latency per row, not per 8-column group).  skg[q][j]: columns 8j + cq, cq + 1; skm[q]: bit k of byte j =
    // column 8j + k.  Chunk c + 1's are issued once chunk c is staged, chunk 0's before wgmma_wait<0> (kSkipEarly).
    uint32_t skg[4][8];
    uint64_t skm[4];
    auto skip_ld = [&](int q, int c) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        skg[q][j] = arow[q] != nullptr ? __ldg(reinterpret_cast<const unsigned int*>(arow[q] + c * 64 + j * 8 + cq)) : 0u;
      skm[q] = mrow[q] != nullptr ? __ldg(reinterpret_cast<const unsigned long long*>(mrow[q] + c * 8)) : 0ull;
    };
    // kHasY: the pre-BN tile of chunk c into sYW (one per warpgroup), by the warpgroup's thread 0
    auto y_ld = [&](int c) {
      mbar_arrive_expect_tx(&y_bar[wg], static_cast<uint32_t>(p.valid_rows) * 128u);
      if (p.mode == 0)
        tma_load_2d(sYW, &tmY, &y_bar[wg], nb * BLOCK_N + c * 64, m_tile * kBlockM);
      else
        tma_load_4d(sYW, &tmY, &y_bar[wg], nb * BLOCK_N + c * 64, w0, h0, n0);
    };
    // ---------------------------------------------------------------- main loop
    // One stage = one k-block (or, in halo mode, three vertical taps of one k-block).  The MMAs of a stage stay in
    // flight while the next stage is waited for; a stage is released once the group after it has been issued.
    // The other warpgroup has issued all MMAs of the previous tile (so every stage before this tile's is filled).
    if (i > 0) named_bar_sync(my_turn, kConvConsumers);
    if (kEarlyY) {
      // Chunk 0's pre-BN tile lands during the main loop.  This barrier stands in for chunk 0's epilogue barrier.
      if (wtid == 0) tma_store_wait_read<kChunks - 1>();  // the store from staging buffer 0 one tile ago has read it
      named_bar_sync(epi_bar, 128);  // the previous tile's statistics are done reading sYW and the staging buffers
      if (wtid == 0) y_ld(0);
    }
    float acc[2][kAcc];
#pragma unroll
    for (int mh = 0; mh < 2; ++mh)
#pragma unroll
      for (int k = 0; k < kAcc; ++k) acc[mh][k] = 0.f;
    fence_acc(acc[0]);
    fence_acc(acc[1]);
    int prev = -1;
    for (int it = 0; it < n_stages; ++it) {
      mbar_wait_u32(full0 + stage * 8, phase);
      wgmma_fence();
      const uint64_t da_s = da0 + static_cast<uint32_t>(stage * (L::kASlot >> 4));
      if (kHalo) {
        const int hs = it / p.kblocks, kb = it - hs * p.kblocks;
        const uint32_t shift16 = static_cast<uint32_t>(p.bw) * 8;  // bw rows of 128 B, in the (addr >> 4) field
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          // vertical tap r reads the same stage bw * r rows further down (bw % 8 == 0: whole swizzle atoms); rows past
          // the pixel box feed discarded accumulator rows
          const uint64_t db = db0 + static_cast<uint32_t>((p.halo_tap[hs * 3 + r] * p.kblocks + kb) * (L::kBBytes >> 4));
          mma_kblock<BLOCK_N>(acc, da_s + r * shift16, db);
        }
      } else {
        const uint64_t db = db0 + static_cast<uint32_t>((kResB ? it : stage) * (L::kBBytes >> 4));
        mma_kblock<BLOCK_N>(acc, da_s, db);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);  // the MMAs that read stage `prev` have retired
      }
      prev = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    // every stage of this tile has been waited for: the other warpgroup may start its tile while these MMAs drain
    if (tile + static_cast<int>(gridDim.x) < p.num_tiles) named_bar_arrive(their_turn, kConvConsumers);
    if (kStats == 3 && kSkipEarly) {
#pragma unroll
      for (int q = 0; q < 4; ++q) skip_ld(q, 0);
    }
    wgmma_wait<0>();
    fence_acc(acc[0]);
    fence_acc(acc[1]);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
    }

    // ---------------------------------------------------------------- epilogue (this warpgroup only)
#pragma unroll
    for (int c = 0; c < kChunks; ++c, ++chunk_ctr) {
      uint8_t* sbuf = sStageW + c * kTileChunkBytes;
      if (!kEarlyY || c > 0) {  // kEarlyY chunk 0: the barrier before the main loop
        if (wtid == 0) tma_store_wait_read<kChunks - 1>();  // the store from this buffer one tile ago has read it
        named_bar_sync(epi_bar, 128);  // the store has read this buffer and the statistics are done with it and sYW
      }
      if (kHasY && (c > 0 || !kEarlyY) && wtid == 0) y_ld(c);  // the last statistics are done with sYW: barrier above
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int mh = q >> 1, h = q & 1;
        const int row = 64 * mh + r16 + 8 * h;
        // This row's residual / skip-gradient words and ReLU-mask bits.  kAffine issues all of its residual loads
        // before any is used: one memory latency per row instead of one per 8-column group (the smem stores below would
        // otherwise keep the compiler from hoisting the loads).  gv[j]: columns 8j + cq, cq + 1; mv: bit k of byte j =
        // column 8j + k.
        uint32_t gv[8];
        uint64_t mv = 0ull;
        if (kStats == 3) {
          if (c == 0 && !kSkipEarly) skip_ld(q, 0);
#pragma unroll
          for (int j = 0; j < 8; ++j) gv[j] = skg[q][j];
          mv = skm[q];
        } else if (kAffine) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            gv[j] = arow[q] != nullptr ? __ldg(reinterpret_cast<const unsigned int*>(arow[q] + c * 64 + j * 8 + cq)) : 0u;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int ig = c * 8 + j;      // 8-column group of the accumulator
          const int col = ig * 8 + cq;   // tile column of v[0]
          float v0 = acc[mh][4 * ig + 2 * h], v1 = acc[mh][4 * ig + 2 * h + 1];
          if (kAffine) {
            // out = act(acc * scale[c] + shift[c] [+ residual])
            v0 = fmaf(v0, __ldg(p.ep_scale + nb * BLOCK_N + col), __ldg(p.ep_shift + nb * BLOCK_N + col)) +
                 __uint_as_float(gv[j] << 16);
            v1 = fmaf(v1, __ldg(p.ep_scale + nb * BLOCK_N + col + 1), __ldg(p.ep_shift + nb * BLOCK_N + col + 1)) +
                 __uint_as_float(gv[j] & 0xFFFF0000u);
            if (p.ep_act >= 1) v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
            if (p.ep_act == 2) v0 = fminf(v0, 6.f), v1 = fminf(v1, 6.f);
          }
          if (kStats == 3) {
            // dz = (main-path gradient + skip gradient) * [block output > 0]
            const uint32_t m = static_cast<uint32_t>(mv >> (8 * j + cq));
            v0 = (m & 1u) ? v0 + __uint_as_float(gv[j] << 16) : 0.f;
            v1 = (m & 2u) ? v1 + __uint_as_float(gv[j] & 0xFFFF0000u) : 0.f;
          }
          // bf16 pack + swizzled smem write (16 B chunk j of row r lives at chunk j ^ (r & 7))
          uint32_t w = pack_bf16x2(v0, v1);
          if (kStatsOn && row >= p.valid_rows) w = 0u;  // rows past the pixel box: no statistics
          *reinterpret_cast<uint32_t*>(sbuf + row * 128 + ((j ^ (row & 7)) << 4) + (lane & 3) * 4) = w;
        }
      }
      if (kStats == 3 && c + 1 < kChunks) {
#pragma unroll
        for (int q = 0; q < 4; ++q) skip_ld(q, c + 1);  // next chunk's rows, in flight from here on
      }
      fence_proxy_async_smem();
      named_bar_sync(epi_bar, 128);  // every staging write is done before the TMA store and the statistics read them
      if (wtid == 0) {
        const int ccol = nb * BLOCK_N + c * 64;
        if (p.mode == 0)
          tma_store_2d(&tmD, sbuf, ccol, m_tile * kBlockM);
        else
          tma_store_4d(&tmD, sbuf, ccol, w0, h0, n0);
        tma_store_commit();
      }
      if (kStatsOn) {
        // column sums of the bf16 tile just staged (exactly the values BatchNorm will read): one conflict-free LDS.32
        // per row with precomputed swizzled offsets; two 16-row partials per thread, added once
        float part[2][4];
        float sc0 = 0.f, sc1 = 0.f, sh0 = 0.f, sh1 = 0.f;
        if (kStats == 2) {
          const int gc = nb * BLOCK_N + c * 64 + cp * 2;
          sc0 = p.bn_scale[gc], sc1 = p.bn_scale[gc + 1];
          sh0 = p.bn_shift[gc], sh1 = p.bn_shift[gc + 1];
        }
        if (kHasY) mbar_wait(&y_bar[wg], chunk_ctr & 1);
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint8_t* srow = sbuf + (rg * 32 + hf * 16) * 128;
          const uint8_t* yrow = sYW + (rg * 32 + hf * 16) * 128;
          float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
          for (int r = 0; r < 16; ++r) {
            const uint32_t w = *reinterpret_cast<const uint32_t*>(srow + xoff[r & 7] + r * 128);
            float g0 = __uint_as_float(w << 16), g1 = __uint_as_float(w & 0xFFFF0000u);
            if (kStats == 1) {
              s0 += g0;
              s1 += g1;
              q0 = fmaf(g0, g0, q0);
              q1 = fmaf(g1, g1, q1);
            } else {
              const uint32_t u = *reinterpret_cast<const uint32_t*>(yrow + xoff[r & 7] + r * 128);
              const float y0 = __uint_as_float(u << 16), y1 = __uint_as_float(u & 0xFFFF0000u);
              if (kStats == 2) {
                // dz = g * [y*scale + shift > 0]  (kStats == 3: the staged tile already is dz)
                g0 = fmaf(y0, sc0, sh0) > 0.f ? g0 : 0.f;
                g1 = fmaf(y1, sc1, sh1) > 0.f ? g1 : 0.f;
              }
              s0 += g0;
              s1 += g1;
              q0 = fmaf(g0, y0, q0);
              q1 = fmaf(g1, y1, q1);
            }
          }
          part[hf][0] = s0, part[hf][1] = s1, part[hf][2] = q0, part[hf][3] = q1;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) sacc[c][k] += part[0][k] + part[1][k];
      }
    }
    if (kStatsOn) {
      // register accumulators are flushed with global atomics only when this warpgroup moves to another n-block
      const int next = tile + 2 * gridDim.x;
      if (next >= p.num_tiles || (next % p.n_blocks) != nb) {
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          const int col = nb * BLOCK_N + c * 64 + cp * 2;
          atomicAdd(p.stat_sum + col, sacc[c][0]);
          atomicAdd(p.stat_sum + col + 1, sacc[c][1]);
          atomicAdd(p.stat_sqsum + col, sacc[c][2]);
          atomicAdd(p.stat_sqsum + col + 1, sacc[c][3]);
          sacc[c][0] = sacc[c][1] = sacc[c][2] = sacc[c][3] = 0.f;
        }
      }
    }
  }
  if (wtid == 0) tma_store_wait_all<0>();

  if (kStatsOn) {
    // ---- last-CTA tail: every CTA's sums are in L2 once its consumers have fenced and taken a ticket; the CTA
    // that takes the last ticket turns the sums into the per-channel coefficients the NEXT kernel needs (and zeroes them),
    // so no tiny dependent kernel sits between this GEMM and its consumer.
    const bool want_tail = (kStats == 1) ? (p.fin.enable != 0) : (p.bfin.enable != 0);
    if (want_tail) {
      unsigned int* counter = (kStats == 1) ? p.fin.counter : p.bfin.counter;
      __threadfence();
      named_bar_sync(5, kConvConsumers);
      if (ctid == 0) *s_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1 : 0;
      named_bar_sync(5, kConvConsumers);
      if (*reinterpret_cast<volatile int*>(s_last) != 0) {
        __threadfence();
        for (int c = ctid; c < p.cout; c += kConvConsumers) {
          const float s0 = __ldcg(p.stat_sum + c), s1 = __ldcg(p.stat_sqsum + c);
          p.stat_sum[c] = 0.f;
          p.stat_sqsum[c] = 0.f;
          if (kStats == 1) {
            const ConvParams::Fin& f = p.fin;
            const float m = s0 * f.inv_count;
            const float var = fmaxf(s1 * f.inv_count - m * m, 0.f);
            f.running_mean[c] = (1.f - f.momentum) * f.running_mean[c] + f.momentum * m;
            f.running_var[c] = (1.f - f.momentum) * f.running_var[c] + f.momentum * var * f.unbias;
            const float is = rsqrtf(var + f.eps);
            f.mean[c] = m;
            f.invstd[c] = is;
            const float sc = f.gamma[c] * is;
            f.scale[c] = sc;
            f.shift[c] = f.beta[c] - m * sc;
          } else {
            const ConvParams::BFin& f = p.bfin;
            const float db = s0, dzy = s1;
            const float m = f.mean[c], is = f.invstd[c];
            const float dg = is * (dzy - m * db);
            f.dgamma[c] = dg;
            f.dbeta[c] = db;
            const float A = f.gamma[c] * is;
            const float B = -A * is * dg * f.inv_count;
            f.cA[c] = A;
            f.cB[c] = B;
            f.cC[c] = -A * db * f.inv_count - B * m;
          }
        }
        if (ctid == 0) *counter = 0u;
      }
    }
  }
}

}  // namespace b200
