// Fused gradient all-reduce kernels for 2-8 H100s on one NVSwitch domain (SURVEY.md K1-K3, §5.8).
//
// The reference reaches NCCL through Horovod's DistributedOptimizer and then runs separate scale / cast kernels.
// Here ONE kernel does barrier -> reduce -> x(1/N) -> cast -> write-back -> barrier, reading and writing peer
// memory directly:
//   * one-shot  (<= ~256 KB): every rank loads all peers' values over NVLink P2P and reduces in registers;
//   * two-shot P2P           : reduce-scatter by P2P loads, all-gather by P2P stores;
//   * two-shot NVLS          : multimem.ld_reduce (reduction inside the NVSwitch) + multimem.st (multicast).
// Cross-GPU synchronisation is a flag barrier in symmetric memory (release/acquire CAS at .sys scope); flags
// toggle 0 -> 1 -> 0 so the kernels are CUDA-graph replayable without host-side epochs.
#include <cuda_bf16.h>

#include <stdexcept>
#include <string>

#include "comm_api.h"
#include "optim_rules.cuh"

namespace b200 {

// Watchdog (SURVEY.md 5.3): a peer that died or never launched its kernel would leave us spinning forever; after
// kCommTimeoutNs of wall time the kernel traps, the CUDA error kills this rank and the Runner stops the gang.
constexpr unsigned long long kCommTimeoutNs = 120ull * 1000ull * 1000ull * 1000ull;

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ void flag_signal(uint32_t* addr) {
  uint32_t old;
  unsigned long long t0 = 0;
  unsigned int spins = 0;
  do {
    asm volatile("atom.global.release.sys.cas.b32 %0, [%1], 0, 1;" : "=r"(old) : "l"(addr) : "memory");
    if (old != 0u && (++spins & 0xFFFFu) == 0u) {
      const unsigned long long now = global_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > kCommTimeoutNs) __trap();
    }
  } while (old != 0u);
}
__device__ __forceinline__ void flag_wait(uint32_t* addr) {
  uint32_t old;
  unsigned long long t0 = 0;
  unsigned int spins = 0;
  do {
    asm volatile("atom.global.acquire.sys.cas.b32 %0, [%1], 1, 0;" : "=r"(old) : "l"(addr) : "memory");
    if (old != 1u && (++spins & 0xFFFFu) == 0u) {
      const unsigned long long now = global_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > kCommTimeoutNs) __trap();
    }
  } while (old != 1u);
}

// Block-scoped barrier across all ranks: thread t < world signals peer t and waits for peer t's signal.
// flags layout per rank: [slot][block][world].
__device__ __forceinline__ void block_barrier(const CommCtx& c, int slot) {
  __syncthreads();
  if (threadIdx.x < c.world) {
    const int peer = threadIdx.x;
    const size_t base = (static_cast<size_t>(slot) * kCommMaxBlocks + blockIdx.x) * c.world;
    flag_signal(c.peer_flags[peer] + base + c.rank);
    flag_wait(c.peer_flags[c.rank] + base + peer);
  }
  __syncthreads();
}

struct f32x4 { float v[4]; };

__device__ __forceinline__ float4 ld_f4(const void* p) { return *reinterpret_cast<const float4*>(p); }

// 16 bytes of payload -> fp32 lanes (4 for f32, 8 for bf16)
template <int T> struct Vec;
template <> struct Vec<kF32> {
  static constexpr int kElems = 4;
  __device__ static void load(const void* p, float (&f)[8]) {
    float4 a = ld_f4(p);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  }
  __device__ static void store(void* p, const float (&f)[8]) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  }
};
template <> struct Vec<kBF16> {
  static constexpr int kElems = 8;
  __device__ static void load(const void* p, float (&f)[8]) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[i]);
      float2 t = __bfloat1622float2(h);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
  __device__ static void store(void* p, const float (&f)[8]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  }
};

template <int T> __device__ __forceinline__ size_t esize() { return T == kF32 ? 4 : 2; }

// ------------------------------------------------------------------------------------------------ one-shot
template <int TIN, int TOUT>
__global__ void __launch_bounds__(512) allreduce_oneshot_kernel(CommCtx c, int64_t off, int64_t n, void* dst, float scale) {
  block_barrier(c, 0);
  constexpr int E = Vec<TIN>::kElems;
  const int64_t nvec = n / E;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    // fixed rank order => bit-identical result on every rank
    for (int r = 0; r < c.world; ++r) {
      float f[8];
      Vec<TIN>::load(reinterpret_cast<const char*>(c.peer_bufs[r]) + (off + i * E) * esize<TIN>(), f);
#pragma unroll
      for (int k = 0; k < E; ++k) acc[k] += f[k];
    }
#pragma unroll
    for (int k = 0; k < E; ++k) acc[k] *= scale;
    char* o = reinterpret_cast<char*>(dst) + i * E * esize<TOUT>();
    if (TOUT == TIN) {
      Vec<TOUT>::store(o, acc);
    } else if (TIN == kF32 && TOUT == kBF16) {
      __nv_bfloat162 a = __floats2bfloat162_rn(acc[0], acc[1]);
      __nv_bfloat162 b = __floats2bfloat162_rn(acc[2], acc[3]);
      uint2 u;
      u.x = *reinterpret_cast<uint32_t*>(&a);
      u.y = *reinterpret_cast<uint32_t*>(&b);
      *reinterpret_cast<uint2*>(o) = u;
    } else {  // bf16 in, f32 out
      *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      *reinterpret_cast<float4*>(o + 16) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
  }
  block_barrier(c, 1);
}

// ------------------------------------------------------------------------------------------------ two-shot P2P
// UNROLL independent 16-byte vectors per thread per iteration: all peer loads of an iteration are issued before the
// first add, so UNROLL * world loads are in flight per thread (NVLink latency is ~3 us; bandwidth needs depth).
template <int T, int UNROLL>
__global__ void __launch_bounds__(512) allreduce_twoshot_p2p_kernel(CommCtx c, int64_t off, int64_t n, float scale) {
  constexpr int E = Vec<T>::kElems;
  const int64_t nvec = n / E;
  const int64_t per = (nvec + c.world - 1) / c.world;
  const int64_t v0 = per * c.rank;
  const int64_t v1 = (v0 + per < nvec) ? v0 + per : nvec;
  block_barrier(c, 0);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = v0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v1; i += stride * UNROLL) {
    uint4 raw[UNROLL];
    float acc[UNROLL][8];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[u][k] = 0.f;
    for (int r = 0; r < c.world; ++r) {
      const char* base = reinterpret_cast<const char*>(c.peer_bufs[r]) + off * esize<T>();
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int64_t j = i + u * stride;
        raw[u] = (j < v1) ? *reinterpret_cast<const uint4*>(base + j * 16) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        float f[8];
        Vec<T>::load(&raw[u], f);
#pragma unroll
        for (int k = 0; k < E; ++k) acc[u][k] += f[k];
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t j = i + u * stride;
      if (j >= v1) continue;
#pragma unroll
      for (int k = 0; k < E; ++k) acc[u][k] *= scale;
      uint4 outv;
      Vec<T>::store(&outv, acc[u]);
      // all-gather by P2P stores: push the reduced vector into every rank's buffer
      for (int r = 0; r < c.world; ++r)
        *reinterpret_cast<uint4*>(reinterpret_cast<char*>(c.peer_bufs[r]) + off * esize<T>() + j * 16) = outv;
    }
  }
  block_barrier(c, 1);
}

// ------------------------------------------------------------------------------------------------ two-shot NVLS
__device__ __forceinline__ void mm_ld_reduce_f32(const void* mc, float (&f)[4]) {
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(f[0]), "=f"(f[1]), "=f"(f[2]), "=f"(f[3])
               : "l"(mc)
               : "memory");
}
__device__ __forceinline__ void mm_st_f32(void* mc, const float (&f)[4]) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(f[0]), "f"(f[1]),
               "f"(f[2]), "f"(f[3])
               : "memory");
}
__device__ __forceinline__ void mm_ld_reduce_bf16(const void* mc, uint32_t (&w)[4]) {
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
               : "l"(mc)
               : "memory");
}
__device__ __forceinline__ void mm_st_b32x4(void* mc, const uint32_t (&w)[4]) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1, %2, %3, %4};" ::"l"(mc), "r"(w[0]), "r"(w[1]),
               "r"(w[2]), "r"(w[3])
               : "memory");
}

template <int T, int UNROLL>
__global__ void __launch_bounds__(512) allreduce_twoshot_nvls_kernel(CommCtx c, int64_t off, int64_t n, float scale) {
  constexpr int E = Vec<T>::kElems;
  const int64_t nvec = n / E;
  const int64_t per = (nvec + c.world - 1) / c.world;
  const int64_t v0 = per * c.rank;
  const int64_t v1 = (v0 + per < nvec) ? v0 + per : nvec;
  block_barrier(c, 0);
  char* mc = reinterpret_cast<char*>(c.mc_buf) + off * esize<T>();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = v0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v1; i += stride * UNROLL) {
    if (T == kF32) {
      float f[UNROLL][4];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int64_t j = i + u * stride;
        if (j < v1) mm_ld_reduce_f32(mc + j * 16, f[u]);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int64_t j = i + u * stride;
        if (j >= v1) continue;
#pragma unroll
        for (int k = 0; k < 4; ++k) f[u][k] *= scale;
        mm_st_f32(mc + j * 16, f[u]);
      }
    } else {
      uint32_t w[UNROLL][4];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int64_t j = i + u * stride;
        if (j < v1) mm_ld_reduce_bf16(mc + j * 16, w[u]);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int64_t j = i + u * stride;
        if (j >= v1) continue;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&w[u][k]);
          float2 t = __bfloat1622float2(h);
          h = __floats2bfloat162_rn(t.x * scale, t.y * scale);
          w[u][k] = *reinterpret_cast<uint32_t*>(&h);
        }
        mm_st_b32x4(mc + j * 16, w[u]);
      }
    }
  }
  block_barrier(c, 1);
}

// ------------------------------------------------------------------------------------------------ broadcast
template <int T>
__global__ void __launch_bounds__(512) broadcast_kernel(CommCtx c, int64_t off, int64_t n, int root) {
  constexpr int E = Vec<T>::kElems;
  const int64_t nvec = n / E;
  block_barrier(c, 0);
  if (c.rank == root) {
    const char* src = reinterpret_cast<const char*>(c.peer_bufs[root]) + off * esize<T>();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
      uint4 u = *reinterpret_cast<const uint4*>(src + i * 16);
      if (c.mc_buf != nullptr) {
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
        mm_st_b32x4(reinterpret_cast<char*>(c.mc_buf) + off * esize<T>() + i * 16, w);
      } else {
        for (int r = 0; r < c.world; ++r)
          if (r != root) *reinterpret_cast<uint4*>(reinterpret_cast<char*>(c.peer_bufs[r]) + off * esize<T>() + i * 16) = u;
      }
    }
  }
  block_barrier(c, 1);
}

// ------------------------------------------------------------------------------------------------ all-reduce + SGD
// grad: fp32 symmetric (multicast) buffer;  weight: fp32 symmetric (multicast) buffer;  momentum: local slice-owner
// state (indexed by global element);  w16_mc: optional bf16 multicast working copy.
__global__ void __launch_bounds__(512)
allreduce_sgd_nvls_kernel(CommCtx g, CommCtx w, int64_t off, int64_t n, float* __restrict__ mom, void* w16_mc,
                          float scale, const float* __restrict__ hyper) {
  const int64_t nvec = n / 4;
  const int64_t per = (nvec + g.world - 1) / g.world;
  const int64_t v0 = per * g.rank;
  const int64_t v1 = (v0 + per < nvec) ? v0 + per : nvec;
  const SgdRule<false> sgd(hyper, scale);   // the unfused update's rule, on the gradient scaled by `scale`
  block_barrier(g, 0);
  char* gmc = reinterpret_cast<char*>(g.mc_buf) + off * 4;
  char* wloc = reinterpret_cast<char*>(w.peer_bufs[w.rank]) + off * 4;
  char* wmc = reinterpret_cast<char*>(w.mc_buf) + off * 4;
  for (int64_t i = v0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < v1; i += (int64_t)gridDim.x * blockDim.x) {
    float gr[4];
    mm_ld_reduce_f32(gmc + i * 16, gr);
    float4 wv = *reinterpret_cast<const float4*>(wloc + i * 16);
    float4 mv = *reinterpret_cast<const float4*>(mom + off + i * 4);
    float* wf = &wv.x;
    float* mf = &mv.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) sgd(wf[k], gr[k], &mf[k]);
    *reinterpret_cast<float4*>(mom + off + i * 4) = mv;
    const float o[4] = {wf[0], wf[1], wf[2], wf[3]};
    mm_st_f32(wmc + i * 16, o);
    if (w16_mc != nullptr) {
      __nv_bfloat162 a = __floats2bfloat162_rn(wf[0], wf[1]);
      __nv_bfloat162 b = __floats2bfloat162_rn(wf[2], wf[3]);
      asm volatile("multimem.st.relaxed.sys.global.v2.bf16x2 [%0], {%1, %2};" ::"l"(
                       reinterpret_cast<char*>(w16_mc) + (off + i * 4) * 2),
                   "r"(*reinterpret_cast<uint32_t*>(&a)), "r"(*reinterpret_cast<uint32_t*>(&b))
                   : "memory");
    }
  }
  block_barrier(g, 1);
}

// ------------------------------------------------------------------------------------------------ host
static void check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
static int clamp_blocks(int b) { return b < 1 ? 1 : (b > kCommMaxBlocks ? kCommMaxBlocks : b); }

void allreduce_oneshot(const CommCtx& c, int64_t off, int64_t n, CommDtype in_t, void* dst, CommDtype out_t,
                       float scale, int blocks, cudaStream_t s) {
  blocks = clamp_blocks(blocks);
  if (in_t == kF32 && out_t == kF32) allreduce_oneshot_kernel<kF32, kF32><<<blocks, 512, 0, s>>>(c, off, n, dst, scale);
  else if (in_t == kF32 && out_t == kBF16) allreduce_oneshot_kernel<kF32, kBF16><<<blocks, 512, 0, s>>>(c, off, n, dst, scale);
  else if (in_t == kBF16 && out_t == kBF16) allreduce_oneshot_kernel<kBF16, kBF16><<<blocks, 512, 0, s>>>(c, off, n, dst, scale);
  else allreduce_oneshot_kernel<kBF16, kF32><<<blocks, 512, 0, s>>>(c, off, n, dst, scale);
  check_launch("allreduce_oneshot");
}
void allreduce_twoshot_p2p(const CommCtx& c, int64_t off, int64_t n, CommDtype t, float scale, int blocks,
                           cudaStream_t s) {
  blocks = clamp_blocks(blocks);
  if (c.world <= 2) {
    if (t == kF32) allreduce_twoshot_p2p_kernel<kF32, 4><<<blocks, 512, 0, s>>>(c, off, n, scale);
    else allreduce_twoshot_p2p_kernel<kBF16, 4><<<blocks, 512, 0, s>>>(c, off, n, scale);
  } else {
    if (t == kF32) allreduce_twoshot_p2p_kernel<kF32, 2><<<blocks, 512, 0, s>>>(c, off, n, scale);
    else allreduce_twoshot_p2p_kernel<kBF16, 2><<<blocks, 512, 0, s>>>(c, off, n, scale);
  }
  check_launch("allreduce_twoshot_p2p");
}
void allreduce_twoshot_nvls(const CommCtx& c, int64_t off, int64_t n, CommDtype t, float scale, int blocks,
                            cudaStream_t s) {
  if (c.mc_buf == nullptr) throw std::runtime_error("allreduce_twoshot_nvls: no multicast mapping");
  blocks = clamp_blocks(blocks);
  if (t == kF32) allreduce_twoshot_nvls_kernel<kF32, 8><<<blocks, 512, 0, s>>>(c, off, n, scale);
  else allreduce_twoshot_nvls_kernel<kBF16, 8><<<blocks, 512, 0, s>>>(c, off, n, scale);
  check_launch("allreduce_twoshot_nvls");
}
void broadcast_sym(const CommCtx& c, int64_t off, int64_t n, CommDtype t, int root, int blocks, cudaStream_t s) {
  blocks = clamp_blocks(blocks);
  if (t == kF32) broadcast_kernel<kF32><<<blocks, 512, 0, s>>>(c, off, n, root);
  else broadcast_kernel<kBF16><<<blocks, 512, 0, s>>>(c, off, n, root);
  check_launch("broadcast_sym");
}
void allreduce_sgd_nvls(const CommCtx& grad, const CommCtx& weight, int64_t off, int64_t n, float* mom_local,
                        void* w16_mc, float scale, const float* hyper, int blocks, cudaStream_t s) {
  if (grad.mc_buf == nullptr || weight.mc_buf == nullptr)
    throw std::runtime_error("allreduce_sgd_nvls: no multicast mapping");
  blocks = clamp_blocks(blocks);
  allreduce_sgd_nvls_kernel<<<blocks, 512, 0, s>>>(grad, weight, off, n, mom_local, w16_mc, scale, hyper);
  check_launch("allreduce_sgd_nvls");
}

}  // namespace b200
