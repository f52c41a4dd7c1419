// pybind layer of the hardware probe (csrc/tma_probe.cu): a measurement tool the kernel design rests
// on, kept OUT of the hot-path extension (_b200_conv) - they are built as their own module, _b200_probe.
#include <ATen/cuda/CUDAContext.h>
#include <torch/extension.h>

#include <algorithm>
#include <cstring>

#include "conv_api.h"

namespace b200 {

static int sm_count() { return at::cuda::getCurrentDeviceProperties()->multiProcessorCount; }

static CUtensorMap map_nhwc(const at::Tensor& t, int box_c, int bw, int bh, int bn) {
  uint64_t dims[4] = {(uint64_t)t.size(3), (uint64_t)t.size(2), (uint64_t)t.size(1), (uint64_t)t.size(0)};
  uint64_t strides[3] = {(uint64_t)t.stride(2) * 2, (uint64_t)t.stride(1) * 2, (uint64_t)t.stride(0) * 2};
  uint32_t box[4] = {(uint32_t)box_c, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
  return encode_bf16(t.data_ptr(), 4, dims, strides, box);
}
static CUtensorMap map_2d(void* ptr, int64_t rows, int64_t cols, int64_t pitch, int box_cols, int box_rows) {
  uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows};
  uint64_t strides[1] = {(uint64_t)pitch * 2};
  uint32_t box[2] = {(uint32_t)box_cols, (uint32_t)box_rows};
  return encode_bf16(ptr, 2, dims, strides, box);
}

// hardware probe (see csrc/tma_probe.cu): x is an NHWC bf16 tensor with C == 64.
//   rows_2d > 0: 2-D [N*H*W, 64] map with boxes of rows_2d pixels;  otherwise a 4-D map with a (bw, bh, bn) pixel box
//   offset by (dw, dh) - a filter tap, so border boxes exercise the out-of-bounds fill.
static void tma_probe(at::Tensor x, int64_t rows_2d, int64_t bw, int64_t bh, int64_t bn, int64_t dw, int64_t dh,
                      int64_t stages, int64_t loads_per_cta, int64_t grid) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 4 && x.size(3) == 64 && x.is_contiguous());
  TmaProbeParams p;
  std::memset(&p, 0, sizeof(p));
  const int64_t N = x.size(0), H = x.size(1), W = x.size(2);
  CUtensorMap tm;
  if (rows_2d > 0) {
    TORCH_CHECK(rows_2d <= 256 && rows_2d % 8 == 0);
    p.mode = 0;
    p.box_bytes = (int)rows_2d * 128;
    p.m_tiles = (int)((N * H * W) / 128) - 2;  // positions are multiples of 128 rows; keep the box inside the tensor
    tm = map_2d(x.data_ptr(), N * H * W, 64, 64, 64, (int)rows_2d);
  } else {
    TORCH_CHECK(bw >= 1 && bh >= 1 && bn >= 1 && bw <= 256 && bh <= 256 && bn <= 256 && bw * bh * bn * 128 <= 114688);
    p.mode = 1;
    p.box_bytes = (int)(bw * bh * bn) * 128;
    p.bw = (int)bw; p.bh = (int)bh; p.bn = (int)bn;
    p.tiles_w = (int)std::max<int64_t>(1, W / bw); p.tiles_h = (int)std::max<int64_t>(1, H / bh);
    p.tiles_n = (int)std::max<int64_t>(1, N / bn);
    p.dw = (int)dw; p.dh = (int)dh;
    tm = map_nhwc(x, 64, (int)bw, (int)bh, (int)bn);
  }
  p.stages = (int)stages;
  p.loads_per_cta = (int)loads_per_cta;
  TORCH_CHECK(stages >= 1 && stages <= 16);
  tma_probe_launch(tm, p, grid > 0 ? (int)grid : sm_count(), at::cuda::getCurrentCUDAStream());
}

}  // namespace b200

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  namespace py = pybind11;
  m.doc() = "b200ddl hardware probe: TMA load-pipeline throughput (sm_90a)";
  m.def("tma_probe", &b200::tma_probe);
}
