// pybind layer for the fused all-reduce kernels.  Symmetric allocations / handle exchange / multicast binding are
// done with torch.distributed._symmetric_memory on the Python side; this layer only receives the raw addresses.
#include <ATen/cuda/CUDAContext.h>
#include <torch/extension.h>

#include "comm_api.h"

namespace {

int64_t g_launches = 0;

struct Comm {
  b200::CommCtx ctx;
  // peer_bufs_dev / peer_flags_dev: device arrays of pointers (int64 addresses) as given by the symm-mem handle
  Comm(int64_t peer_bufs_dev, int64_t peer_flags_dev, int64_t mc_ptr, int64_t rank, int64_t world) {
    ctx.peer_bufs = reinterpret_cast<void* const*>(peer_bufs_dev);
    ctx.peer_flags = reinterpret_cast<uint32_t* const*>(peer_flags_dev);
    ctx.mc_buf = reinterpret_cast<void*>(mc_ptr);
    ctx.rank = (int)rank;
    ctx.world = (int)world;
    TORCH_CHECK(world >= 1 && world <= 32);
  }
  bool has_multicast() const { return ctx.mc_buf != nullptr; }
  static b200::CommDtype dt(const std::string& s) {
    if (s == "f32") return b200::kF32;
    if (s == "bf16") return b200::kBF16;
    TORCH_CHECK(false, "dtype must be 'f32' or 'bf16'");
  }
  static void check_range(int64_t off, int64_t n, b200::CommDtype t) {
    const int e = t == b200::kF32 ? 4 : 8;
    TORCH_CHECK(n % e == 0 && off % e == 0, "all-reduce ranges must be multiples of 16 bytes");
  }
  void oneshot(int64_t off, int64_t n, const std::string& in_t, at::Tensor dst, double scale, int64_t blocks) {
    auto it = dt(in_t);
    auto ot = dst.scalar_type() == at::kFloat ? b200::kF32 : b200::kBF16;
    TORCH_CHECK(dst.is_cuda() && dst.is_contiguous() && dst.numel() >= n);
    check_range(off, n, it);
    b200::allreduce_oneshot(ctx, off, n, it, dst.data_ptr(), ot, (float)scale, (int)blocks, at::cuda::getCurrentCUDAStream());
    ++g_launches;
  }
  void twoshot_p2p(int64_t off, int64_t n, const std::string& t, double scale, int64_t blocks) {
    check_range(off, n, dt(t));
    b200::allreduce_twoshot_p2p(ctx, off, n, dt(t), (float)scale, (int)blocks, at::cuda::getCurrentCUDAStream());
    ++g_launches;
  }
  void twoshot_nvls(int64_t off, int64_t n, const std::string& t, double scale, int64_t blocks) {
    check_range(off, n, dt(t));
    b200::allreduce_twoshot_nvls(ctx, off, n, dt(t), (float)scale, (int)blocks, at::cuda::getCurrentCUDAStream());
    ++g_launches;
  }
  void broadcast(int64_t off, int64_t n, const std::string& t, int64_t root, int64_t blocks) {
    check_range(off, n, dt(t));
    b200::broadcast_sym(ctx, off, n, dt(t), (int)root, (int)blocks, at::cuda::getCurrentCUDAStream());
    ++g_launches;
  }
  void allreduce_sgd(const Comm& weight, int64_t off, int64_t n, at::Tensor mom, int64_t w16_mc, double scale,
                     at::Tensor hyper, int64_t blocks) {
    TORCH_CHECK(mom.is_cuda() && mom.scalar_type() == at::kFloat && mom.is_contiguous());
    TORCH_CHECK(hyper.is_cuda() && hyper.scalar_type() == at::kFloat && hyper.numel() >= 8);
    check_range(off, n, b200::kF32);
    b200::allreduce_sgd_nvls(ctx, weight.ctx, off, n, mom.data_ptr<float>(), reinterpret_cast<void*>(w16_mc),
                             (float)scale, hyper.data_ptr<float>(), (int)blocks, at::cuda::getCurrentCUDAStream());
    ++g_launches;
  }
};

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  namespace py = pybind11;
  m.doc() = "b200ddl fused all-reduce kernels over NVLink symmetric memory (sm_90a)";
  py::class_<Comm>(m, "Comm")
      .def(py::init<int64_t, int64_t, int64_t, int64_t, int64_t>(), py::arg("peer_bufs_dev"),
           py::arg("peer_flags_dev"), py::arg("mc_ptr"), py::arg("rank"), py::arg("world"))
      .def("has_multicast", &Comm::has_multicast)
      .def("oneshot", &Comm::oneshot)
      .def("twoshot_p2p", &Comm::twoshot_p2p)
      .def("twoshot_nvls", &Comm::twoshot_nvls)
      .def("broadcast", &Comm::broadcast)
      .def("allreduce_sgd", &Comm::allreduce_sgd);
  m.attr("MAX_BLOCKS") = b200::kCommMaxBlocks;
  m.attr("FLAG_WORDS") = 2 * b200::kCommMaxBlocks * 32;
  m.def("launch_count", [] { return g_launches; });
  m.def("reset_launch_count", [] { g_launches = 0; });
}
