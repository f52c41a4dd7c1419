// GPU JPEG decode for the sharded loader (`make_dataset(decode='gpu')`): the reference decodes with tf.io.decode_jpeg inside the
// tf.data pipeline (P1/03:182-189); a host's CPU decoders can fall behind even ONE GPU's training rate, so the JPEG
// bitstreams cross PCIe compressed and are decoded on the
// device: nvJPEG (library, like cuDNN is for the baseline) with the HARDWARE backend (the NVJPG engines - no SM time, no CPU
// Huffman decode) when the GPU has them, the GPU-hybrid backend otherwise; every image lands interleaved RGB in ONE scratch
// buffer and OUR batched resize kernel (jpeg_resize.cu) writes the [n, H, W, 3] uint8 batch the stem kernels read.
// All work is enqueued on the caller's current stream; nothing here synchronises the device.
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>
#include <nvjpeg.h>
#include <torch/extension.h>

#include <stdexcept>
#include <string>
#include <vector>

namespace b200 {
void resize_triangle_batched(const uint8_t* src, const int64_t* table_dev, uint8_t* out, int n, int OH, int OW, cudaStream_t s);
}

namespace {

const char* status_name(nvjpegStatus_t s) {
  switch (s) {
    case NVJPEG_STATUS_SUCCESS: return "SUCCESS";
    case NVJPEG_STATUS_NOT_INITIALIZED: return "NOT_INITIALIZED";
    case NVJPEG_STATUS_INVALID_PARAMETER: return "INVALID_PARAMETER";
    case NVJPEG_STATUS_BAD_JPEG: return "BAD_JPEG";
    case NVJPEG_STATUS_JPEG_NOT_SUPPORTED: return "JPEG_NOT_SUPPORTED";
    case NVJPEG_STATUS_ALLOCATOR_FAILURE: return "ALLOCATOR_FAILURE";
    case NVJPEG_STATUS_EXECUTION_FAILED: return "EXECUTION_FAILED";
    case NVJPEG_STATUS_ARCH_MISMATCH: return "ARCH_MISMATCH";
    case NVJPEG_STATUS_INTERNAL_ERROR: return "INTERNAL_ERROR";
    case NVJPEG_STATUS_IMPLEMENTATION_NOT_SUPPORTED: return "IMPLEMENTATION_NOT_SUPPORTED";
    case NVJPEG_STATUS_INCOMPLETE_BITSTREAM: return "INCOMPLETE_BITSTREAM";
    default: return "UNKNOWN";
  }
}
#define NVJ(call)                                                                                  \
  do {                                                                                             \
    nvjpegStatus_t st_ = (call);                                                                   \
    if (st_ != NVJPEG_STATUS_SUCCESS)                                                              \
      throw std::runtime_error(std::string(#call) + " -> NVJPEG_STATUS_" + status_name(st_));      \
  } while (0)

nvjpegBackend_t backend_of(const std::string& name) {
  if (name == "hardware") return NVJPEG_BACKEND_HARDWARE;
  if (name == "gpu_hybrid") return NVJPEG_BACKEND_GPU_HYBRID;
  if (name == "hybrid") return NVJPEG_BACKEND_HYBRID;
  if (name == "default") return NVJPEG_BACKEND_DEFAULT;
  throw std::runtime_error("unknown nvJPEG backend '" + name + "' (hardware | gpu_hybrid | hybrid | default)");
}

class JpegDecoder {
 public:
  JpegDecoder(int64_t max_batch, const std::string& backend, int64_t cpu_threads, int64_t device)
      : max_batch_((int)max_batch), cpu_threads_((int)cpu_threads), device_((int)device), backend_(backend) {
    c10::cuda::CUDAGuard guard((c10::DeviceIndex)device_);
    NVJ(nvjpegCreateEx(backend_of(backend), nullptr, nullptr, NVJPEG_FLAGS_DEFAULT, &handle_));
    try {
      NVJ(nvjpegJpegStateCreate(handle_, &state_));
    } catch (...) {
      nvjpegDestroy(handle_);
      handle_ = nullptr;
      throw;
    }
    if (cudaHostAlloc((void**)&table_host_, sizeof(int64_t) * 4 * max_batch_ * kTables, cudaHostAllocDefault) != cudaSuccess)
      throw std::runtime_error("JpegDecoder: cudaHostAlloc failed");
    table_dev_ = at::empty({(int64_t)kTables, max_batch_ * 4},
                           at::TensorOptions().dtype(at::kLong).device(at::kCUDA, (c10::DeviceIndex)device_));
  }
  ~JpegDecoder() {
    if (state_) nvjpegJpegStateDestroy(state_);
    if (handle_) nvjpegDestroy(handle_);
    if (table_host_) cudaFreeHost(table_host_);
  }

  std::string backend() const { return backend_; }

  // (engines, cores per engine) of the hardware JPEG decoder; (0, 0) when the query is not supported by this handle
  std::vector<int64_t> hardware_info() const {
    unsigned int e = 0, c = 0;
    if (nvjpegGetHardwareDecoderInfo(handle_, &e, &c) != NVJPEG_STATUS_SUCCESS) return {0, 0};
    return {(int64_t)e, (int64_t)c};
  }

  // ptrs / lens: host addresses and sizes of n JPEG bitstreams (they must stay valid until the stream has consumed them:
  // the caller keeps the Arrow buffers alive for two more batches);  out: uint8 CUDA [n, OH, OW, 3].
  // Returns the decoded sizes [(w, h)] flattened.
  std::vector<int64_t> decode_resize(const std::vector<int64_t>& ptrs, const std::vector<int64_t>& lens, at::Tensor out) {
    const int n = (int)ptrs.size();
    TORCH_CHECK(n > 0 && n <= max_batch_ && lens.size() == ptrs.size(), "decode_resize: 1..max_batch bitstreams");
    TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kByte && out.is_contiguous() && out.dim() == 4 &&
                    out.size(0) == n && out.size(3) == 3, "decode_resize: out must be uint8 CUDA [n, H, W, 3]");
    c10::cuda::CUDAGuard guard(out.device());
    cudaStream_t stream = c10::cuda::getCurrentCUDAStream(out.device().index()).stream();
    std::vector<const unsigned char*> data(n);
    std::vector<size_t> sizes(n);
    std::vector<int64_t> dims(2 * n);
    int64_t* tab = table_host_ + (int64_t)slot_ * max_batch_ * 4;
    int64_t total = 0;
    for (int i = 0; i < n; ++i) {
      data[i] = reinterpret_cast<const unsigned char*>(ptrs[i]);
      sizes[i] = (size_t)lens[i];
      int comps = 0, ws[NVJPEG_MAX_COMPONENT] = {0}, hs[NVJPEG_MAX_COMPONENT] = {0};
      nvjpegChromaSubsampling_t sub;
      NVJ(nvjpegGetImageInfo(handle_, data[i], sizes[i], &comps, &sub, ws, hs));
      const int64_t w = ws[0], h = hs[0];
      TORCH_CHECK(w > 0 && h > 0, "decode_resize: empty image");
      const int64_t pitch = w * 3;
      tab[i * 4 + 0] = total;
      tab[i * 4 + 1] = w;
      tab[i * 4 + 2] = h;
      tab[i * 4 + 3] = pitch;
      dims[2 * i] = w;
      dims[2 * i + 1] = h;
      total += (pitch * h + 255) / 256 * 256;
    }
    if (!scratch_.defined() || scratch_.numel() < total)
      scratch_ = at::empty({total + total / 4}, at::TensorOptions().dtype(at::kByte).device(out.device()));
    uint8_t* base = scratch_.data_ptr<uint8_t>();
    std::vector<nvjpegImage_t> dst(n);
    for (int i = 0; i < n; ++i) {
      for (int c = 0; c < NVJPEG_MAX_COMPONENT; ++c) {
        dst[i].channel[c] = nullptr;
        dst[i].pitch[c] = 0;
      }
      dst[i].channel[0] = base + tab[i * 4 + 0];
      dst[i].pitch[0] = (size_t)tab[i * 4 + 3];
    }
    if (n != cur_batch_) {
      NVJ(nvjpegDecodeBatchedInitialize(handle_, state_, n, cpu_threads_, NVJPEG_OUTPUT_RGBI));
      cur_batch_ = n;
    }
    NVJ(nvjpegDecodeBatched(handle_, state_, data.data(), sizes.data(), dst.data(), stream));
    int64_t* tdev = table_dev_.data_ptr<int64_t>() + (int64_t)slot_ * max_batch_ * 4;
    if (cudaMemcpyAsync(tdev, tab, sizeof(int64_t) * 4 * n, cudaMemcpyHostToDevice, stream) != cudaSuccess)
      throw std::runtime_error("JpegDecoder: table copy failed");
    b200::resize_triangle_batched(base, tdev, out.data_ptr<uint8_t>(), n, (int)out.size(1), (int)out.size(2), stream);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("resize_triangle_batched: ") + cudaGetErrorString(e));
    slot_ = (slot_ + 1) % kTables;
    return dims;
  }

 private:
  static constexpr int kTables = 4;   // host/device size tables rotate: a table is rewritten 4 calls later at the earliest
  int max_batch_, cpu_threads_, device_;
  std::string backend_;
  nvjpegHandle_t handle_ = nullptr;
  nvjpegJpegState_t state_ = nullptr;
  int cur_batch_ = -1;
  int slot_ = 0;
  int64_t* table_host_ = nullptr;
  at::Tensor table_dev_;
  at::Tensor scratch_;
};

// plain batched resize of already decoded images (tests: the kernel against PIL without involving nvJPEG)
void resize_batched(at::Tensor src, at::Tensor table, at::Tensor out) {
  TORCH_CHECK(src.is_cuda() && src.scalar_type() == at::kByte && table.is_cuda() && table.scalar_type() == at::kLong &&
                  out.is_cuda() && out.scalar_type() == at::kByte && out.dim() == 4 && out.is_contiguous(), "resize_batched args");
  c10::cuda::CUDAGuard guard(out.device());
  b200::resize_triangle_batched(src.data_ptr<uint8_t>(), table.data_ptr<int64_t>(), out.data_ptr<uint8_t>(), (int)out.size(0),
                                (int)out.size(1), (int)out.size(2), c10::cuda::getCurrentCUDAStream(out.device().index()).stream());
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  pybind11::class_<JpegDecoder>(m, "JpegDecoder")
      .def(pybind11::init<int64_t, const std::string&, int64_t, int64_t>(), pybind11::arg("max_batch"),
           pybind11::arg("backend") = "hardware", pybind11::arg("cpu_threads") = 1, pybind11::arg("device") = 0)
      .def("backend", &JpegDecoder::backend)
      .def("hardware_info", &JpegDecoder::hardware_info)
      .def("decode_resize", &JpegDecoder::decode_resize, pybind11::call_guard<pybind11::gil_scoped_release>());
  m.def("resize_batched", &resize_batched);
}
