// Fused optimizers over flat parameter / gradient / state buffers (SURVEY.md K16).
// One launch updates every parameter of the model: fp32 master weights and state are read and written once, the
// (all-reduced) fp32 gradient bucket is read once, and an optional bf16 working copy is emitted in the same pass.
// Hyper-parameters come from a device array so that LR warm-up / ReduceLROnPlateau never re-capture the CUDA graph.
#include <cuda_bf16.h>

#include "ops_api.h"
#include "optim_rules.cuh"

namespace b200 {

__device__ __forceinline__ void store_bf16x4(__nv_bfloat16* p16, int64_t i, float4 w) {
  __nv_bfloat162 a = __floats2bfloat162_rn(w.x, w.y);
  __nv_bfloat162 b = __floats2bfloat162_rn(w.z, w.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p16 + i) = u;
}

// One launch of a rule over the flat buffers: per float4, load p, g and the rule's states in order, apply the rule to
// each lane, store p, the states, then the optional bf16 copy.
template <int N>
struct StatePtrs {
  float* __restrict__ s[N];
};
template <class Rule>
__global__ void update_kernel(float* __restrict__ p, const float* __restrict__ g, StatePtrs<Rule::kStates> st,
                              __nv_bfloat16* __restrict__ p16, int64_t n4, const float* __restrict__ hyper) {
  constexpr int S = Rule::kStates;
  const Rule rule(hyper);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 w = reinterpret_cast<float4*>(p)[i];
    const float4 gr = reinterpret_cast<const float4*>(g)[i];
    float4 s[S];
#pragma unroll
    for (int j = 0; j < S; ++j) s[j] = reinterpret_cast<float4*>(st.s[j])[i];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float sk[S];
#pragma unroll
      for (int j = 0; j < S; ++j) sk[j] = (&s[j].x)[k];
      rule((&w.x)[k], (&gr.x)[k], sk);
#pragma unroll
      for (int j = 0; j < S; ++j) (&s[j].x)[k] = sk[j];
    }
    reinterpret_cast<float4*>(p)[i] = w;
#pragma unroll
    for (int j = 0; j < S; ++j) reinterpret_cast<float4*>(st.s[j])[i] = s[j];
    if (p16 != nullptr) store_bf16x4(p16, i * 4, w);
  }
}

// ------------------------------------------------------------------------------------------------ chunked passes
// The clip and LAMB passes work on a chunk table (kChunkFields int64 per row: lo, hi, segment): every segment (one
// parameter tensor) of the flat buffer is cut into chunks of at most kChunkMax floats, float4-aligned, and no chunk spans
// two segments.  One CTA handles one chunk, so a per-segment value (clip factor, LAMB trust ratio) is one load per CTA,
// and a chunk's sum of squares is reduced in a fixed order into one partial: no atomics, bit-reproducible.
constexpr int kChunkThreads = 256;

struct Chunk {
  int64_t lo4, hi4;
  int seg;
};
// rows outside [0, n) or not float4-aligned are skipped (the host builds and checks the table; this only keeps a bad
// row from touching memory it does not own)
__device__ __forceinline__ bool load_chunk(const int64_t* __restrict__ chunks, int64_t n, Chunk& c,
                                           int64_t nseg = INT32_MAX) {
  const int64_t* row = chunks + (int64_t)blockIdx.x * kChunkFields;
  const int64_t lo = row[0], hi = row[1];
  c.lo4 = lo >> 2;
  c.hi4 = hi >> 2;
  c.seg = (int)row[2];
  return lo >= 0 && lo <= hi && hi <= n && ((lo | hi) & 3) == 0 && hi - lo <= kChunkMax && row[2] >= 0 &&
         row[2] < nseg;
}

// fixed-order CTA sum of one value per thread (kChunkThreads threads): warp trees, then warp 0 over the warp sums
__device__ __forceinline__ float block_sum(float x, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = x;
  __syncthreads();
  x = lane < kChunkThreads / 32 ? red[lane] : 0.f;
  if (warp == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  }
  return x;   // valid in thread 0
}

// partial[chunk] = sum over the chunk of (g * hyper[kHypHostGScale])^2
__global__ void __launch_bounds__(kChunkThreads) segment_sumsq_kernel(const float* __restrict__ g, int64_t n,
                                                                      const int64_t* __restrict__ chunks,
                                                                      float* __restrict__ partial,
                                                                      const float* __restrict__ hyper) {
  __shared__ float red[kChunkThreads / 32];
  Chunk c;
  const bool ok = load_chunk(chunks, n, c);
  const float gs = hyper[kHypHostGScale];
  float acc = 0.f;
  if (ok) {
    for (int64_t i = c.lo4 + threadIdx.x; i < c.hi4; i += kChunkThreads) {
      const float4 v = reinterpret_cast<const float4*>(g)[i];
      const float x0 = v.x * gs, x1 = v.y * gs, x2 = v.z * gs, x3 = v.w * gs;
      acc = fmaf(x0, x0, acc);
      acc = fmaf(x1, x1, acc);
      acc = fmaf(x2, x2, acc);
      acc = fmaf(x3, x3, acc);
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// One CTA of 32 warps.  Segment s's partials (chunks segs[s].first .. segs[s].end) are summed by one warp: lane l adds
// chunks first + l, first + l + 32, ... in order, then a shuffle tree; the global sum is the same warp reduction over
// the segment sums in segment order.  sums[k * (nseg + 1) + s] (k = 0: partial_a, 1: partial_b), global at index nseg.
// mode kFinClipGlobal: hyper[kHypGScale] = hyper[kHypHostGScale] * c / max(norm, c) with c = hyper[kHypClip]
// mode kFinClipNorm:   factor[s] = c / max(norm_s, c)
// (the clip factor is exactly 1 when the norm does not exceed c)
// mode kFinLamb:       factor[s] = norm(p)_s / norm(r)_s, or 1 when either is 0 (partial_a: p^2, partial_b: r^2)
constexpr int kFinThreads = 1024;
// Keras's c / max(norm, c), written so that a norm within the threshold gives exactly 1 (an approximate c / c need not)
__device__ __forceinline__ float clip_factor(float sumsq, float c) {
  const float norm = sqrtf(sumsq);
  return norm > c ? c / norm : 1.f;
}
__device__ __forceinline__ float warp_sum_strided(const float* __restrict__ x, int64_t first, int64_t end) {
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  for (int64_t j = first + lane; j < end; j += 32) acc += x[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  return __shfl_sync(0xffffffffu, acc, 0);
}
__global__ void __launch_bounds__(kFinThreads) segment_finalize_kernel(const float* __restrict__ partial,
                                                                       int64_t nchunks,
                                                                       const int64_t* __restrict__ segs, int nseg,
                                                                       float* __restrict__ sums,
                                                                       float* __restrict__ factor,
                                                                       float* __restrict__ hyper, int mode) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = mode == kFinLamb ? 2 : 1;
  const float c = hyper[kHypClip];
  for (int s = warp; s < nseg; s += kFinThreads / 32) {
    const int64_t first = max(segs[2 * s], (int64_t)0), end = min(segs[2 * s + 1], nchunks);   // bad rows: no reads
    float sk[2];
    for (int k = 0; k < nk; ++k) {
      sk[k] = warp_sum_strided(partial + k * nchunks, first, end);
      if (lane == 0) sums[k * (nseg + 1) + s] = sk[k];
    }
    if (lane == 0) {
      if (mode == kFinClipNorm) {
        factor[s] = clip_factor(sk[0], c);
      } else if (mode == kFinLamb) {
        const float pn = sqrtf(sk[0]), rn = sqrtf(sk[1]);
        factor[s] = (pn > 0.f && rn > 0.f) ? pn / rn : 1.f;
      }
    }
  }
  __syncthreads();
  if (warp == 0) {
    for (int k = 0; k < nk; ++k) {
      const float tot = warp_sum_strided(sums + k * (nseg + 1), 0, nseg);
      if (lane == 0) sums[k * (nseg + 1) + nseg] = tot;
      if (k == 0 && lane == 0 && mode == kFinClipGlobal)
        hyper[kHypGScale] = hyper[kHypHostGScale] * clip_factor(tot, c);
    }
  }
}

// clipnorm (factor != nullptr): g = g * gs * factor[segment]; clipvalue: g = clamp(g * gs, -c, c)
__global__ void __launch_bounds__(kChunkThreads) clip_apply_kernel(float* __restrict__ g, int64_t n,
                                                                   const int64_t* __restrict__ chunks,
                                                                   const float* __restrict__ factor, int nseg,
                                                                   const float* __restrict__ hyper) {
  Chunk c;
  if (!load_chunk(chunks, n, c, factor != nullptr ? nseg : INT32_MAX)) return;
  const float gs = hyper[kHypHostGScale], lim = hyper[kHypClip];
  const float f = factor != nullptr ? gs * factor[c.seg] : gs;
  for (int64_t i = c.lo4 + threadIdx.x; i < c.hi4; i += kChunkThreads) {
    float4 v = reinterpret_cast<float4*>(g)[i];
    float* vf = &v.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) vf[k] = factor != nullptr ? vf[k] * f : fminf(fmaxf(vf[k] * f, -lim), lim);
    reinterpret_cast<float4*>(g)[i] = v;
  }
}

// LAMB (You et al. 2019) direction r = m_hat / (sqrt(v_hat) + eps) + wd p, written with explicit intrinsics so that
// pass 1 (norms) and pass 3 (update) evaluate the same instruction sequence on the same stored m, v, p.
__device__ __forceinline__ float lamb_dir(float m, float v, float w, float inv_bc1, float inv_sqrt_bc2, float eps,
                                          float wd) {
  const float denom = __fmaf_rn(sqrtf(v), inv_sqrt_bc2, eps);
  return __fmaf_rn(wd, w, __fdividef(__fmul_rn(m, inv_bc1), denom));
}
struct LambHyper {
  float b1, b2, eps, wd, gs, inv_bc1, inv_sqrt_bc2;
  __device__ explicit LambHyper(const float* __restrict__ h)
      : b1(h[kHypMom]), b2(h[kHypBeta2]), eps(h[kHypEps]), wd(h[kHypWd]), gs(h[kHypGScale]), inv_bc1(1.f / h[kHypBc1]),
        inv_sqrt_bc2(rsqrtf(h[kHypBc2])) {}
};

// pass 1: m, v update; partial[chunk] = sum p^2, partial[nchunks + chunk] = sum r^2
__global__ void __launch_bounds__(kChunkThreads) lamb_moments_kernel(const float* __restrict__ p,
                                                                     const float* __restrict__ g, float* __restrict__ m1,
                                                                     float* __restrict__ v1, int64_t n,
                                                                     const int64_t* __restrict__ chunks,
                                                                     int64_t nchunks, float* __restrict__ partial,
                                                                     const float* __restrict__ hyper) {
  __shared__ float red[kChunkThreads / 32];
  Chunk c;
  const bool ok = load_chunk(chunks, n, c);
  const LambHyper h(hyper);
  float pp = 0.f, rr = 0.f;
  if (ok) {
    for (int64_t i = c.lo4 + threadIdx.x; i < c.hi4; i += kChunkThreads) {
      const float4 w = reinterpret_cast<const float4*>(p)[i];
      const float4 gr = reinterpret_cast<const float4*>(g)[i];
      float4 m = reinterpret_cast<float4*>(m1)[i];
      float4 v = reinterpret_cast<float4*>(v1)[i];
      const float* wf = &w.x; const float* gf = &gr.x; float* mf = &m.x; float* vf = &v.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float d = gf[k] * h.gs;
        mf[k] = fmaf(h.b1, mf[k], (1.f - h.b1) * d);
        vf[k] = fmaf(h.b2, vf[k], (1.f - h.b2) * d * d);
        const float r = lamb_dir(mf[k], vf[k], wf[k], h.inv_bc1, h.inv_sqrt_bc2, h.eps, h.wd);
        pp = fmaf(wf[k], wf[k], pp);
        rr = fmaf(r, r, rr);
      }
      reinterpret_cast<float4*>(m1)[i] = m;
      reinterpret_cast<float4*>(v1)[i] = v;
    }
  }
  pp = block_sum(pp, red);
  __syncthreads();   // red is reused
  rr = block_sum(rr, red);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = pp;
    partial[nchunks + blockIdx.x] = rr;
  }
}

// pass 3: p -= lr * phi[segment] * r, bf16 copy in the same pass
__global__ void __launch_bounds__(kChunkThreads) lamb_apply_kernel(float* __restrict__ p,
                                                                   const float* __restrict__ m1,
                                                                   const float* __restrict__ v1,
                                                                   __nv_bfloat16* __restrict__ p16, int64_t n,
                                                                   const int64_t* __restrict__ chunks,
                                                                   const float* __restrict__ phi, int nseg,
                                                                   const float* __restrict__ hyper) {
  Chunk c;
  if (!load_chunk(chunks, n, c, nseg)) return;
  const LambHyper h(hyper);
  const float step = -hyper[kHypLr] * phi[c.seg];
  for (int64_t i = c.lo4 + threadIdx.x; i < c.hi4; i += kChunkThreads) {
    float4 w = reinterpret_cast<float4*>(p)[i];
    const float4 m = reinterpret_cast<const float4*>(m1)[i];
    const float4 v = reinterpret_cast<const float4*>(v1)[i];
    float* wf = &w.x; const float* mf = &m.x; const float* vf = &v.x;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wf[k] = fmaf(step, lamb_dir(mf[k], vf[k], wf[k], h.inv_bc1, h.inv_sqrt_bc2, h.eps, h.wd), wf[k]);
    reinterpret_cast<float4*>(p)[i] = w;
    if (p16 != nullptr) store_bf16x4(p16, i * 4, w);
  }
}

// ------------------------------------------------------------------------------------ accumulation and weight EMA
// IEEE intrinsics throughout (the build uses --use_fast_math): both kernels equal the torch path bit for bit.
// ACCUMULATE (mode 0): accum += g.  COMBINE (mode 1): g = (accum + g) / n, accum = 0.
template <bool COMBINE>
__global__ void grad_accumulate_kernel(float* __restrict__ g, float* __restrict__ accum, int64_t n4, float n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 gr = reinterpret_cast<float4*>(g)[i];
    float4 a = reinterpret_cast<float4*>(accum)[i];
    float* gf = &gr.x; float* af = &a.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if constexpr (COMBINE) {
        gf[k] = __fdiv_rn(__fadd_rn(af[k], gf[k]), n);
        af[k] = 0.f;
      } else {
        af[k] = __fadd_rn(af[k], gf[k]);
      }
    }
    if (COMBINE) reinterpret_cast<float4*>(g)[i] = gr;
    reinterpret_cast<float4*>(accum)[i] = a;
  }
}

// ema = d * ema + (1 - d) * p with d = hyper[kHypEmaDecay], 1 - d = hyper[kHypEmaRest]; when hyper[kHypEmaOverwrite]
// is set, p = ema and the bf16 copy is rewritten in the same pass.
__global__ void ema_update_kernel(float* __restrict__ p, float* __restrict__ ema, __nv_bfloat16* __restrict__ p16,
                                  int64_t n4, const float* __restrict__ hyper) {
  const float d = hyper[kHypEmaDecay], d1 = hyper[kHypEmaRest];
  const bool overwrite = hyper[kHypEmaOverwrite] != 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 w = reinterpret_cast<const float4*>(p)[i];
    float4 e = reinterpret_cast<float4*>(ema)[i];
    const float* wf = &w.x; float* ef = &e.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) ef[k] = __fadd_rn(__fmul_rn(d, ef[k]), __fmul_rn(d1, wf[k]));
    reinterpret_cast<float4*>(ema)[i] = e;
    if (overwrite) {
      reinterpret_cast<float4*>(p)[i] = e;
      if (p16 != nullptr) store_bf16x4(p16, i * 4, e);
    }
  }
}

__global__ void cast_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, int64_t n4) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
    store_bf16x4(out, i * 4, reinterpret_cast<const float4*>(x)[i]);
}

static inline int blocks_for(int64_t n4) {
  int64_t b = (n4 + 255) / 256;
  if (b > 132 * 8) b = 132 * 8;
  if (b < 1) b = 1;
  return (int)b;
}

template <class Rule>
static void launch_update(float* p, const float* g, float* const* state, void* p16, int64_t n4, const float* hyper,
                          cudaStream_t s) {
  StatePtrs<Rule::kStates> st;
  for (int j = 0; j < Rule::kStates; ++j) st.s[j] = state[j];
  update_kernel<Rule><<<blocks_for(n4), 256, 0, s>>>(p, g, st, (__nv_bfloat16*)p16, n4, hyper);
}
struct RuleEntry {
  void (*launch)(float*, const float*, float* const*, void*, int64_t, const float*, cudaStream_t);
  int states;
};
template <class Rule>
constexpr RuleEntry entry() { return {launch_update<Rule>, Rule::kStates}; }
constexpr RuleEntry kRules[] = {
    entry<SgdRule<false>>(),            // kRuleSgd
    entry<SgdRule<true>>(),             // kRuleSgdNesterov
    entry<AdamRule<false>>(),           // kRuleAdam
    entry<AdamRule<true>>(),            // kRuleAdamW
    entry<AdadeltaRule>(),              // kRuleAdadelta
    entry<RmspropRule<false, false>>(), // kRuleRmsprop
    entry<RmspropRule<false, true>>(),  // kRuleRmspropMomentum
    entry<RmspropRule<true, false>>(),  // kRuleRmspropCentered
    entry<RmspropRule<true, true>>(),   // kRuleRmspropCenteredMomentum
    entry<AdagradRule>(),               // kRuleAdagrad
    entry<AdamaxRule>(),                // kRuleAdamax
};
static_assert(sizeof(kRules) / sizeof(kRules[0]) == kNumOptimRules, "one entry per OptimRule");

int optim_rule_states(OptimRule rule) { return kRules[rule].states; }
// n must be a multiple of 4 (flat buffers are padded by the caller).
void optim_step(OptimRule rule, float* p, const float* g, float* const* state, void* p16, int64_t n,
                const float* hyper, cudaStream_t s) {
  kRules[rule].launch(p, g, state, p16, n / 4, hyper, s);
}
void segment_sumsq(const float* g, int64_t n, const int64_t* chunks, int64_t nchunks, float* partial,
                   const float* hyper, cudaStream_t s) {
  segment_sumsq_kernel<<<(unsigned)nchunks, kChunkThreads, 0, s>>>(g, n, chunks, partial, hyper);
}
void segment_finalize(const float* partial, int64_t nchunks, const int64_t* segs, int nseg, float* sums,
                      float* factor, float* hyper, int mode, cudaStream_t s) {
  segment_finalize_kernel<<<1, kFinThreads, 0, s>>>(partial, nchunks, segs, nseg, sums, factor, hyper, mode);
}
void clip_apply(float* g, int64_t n, const int64_t* chunks, int64_t nchunks, const float* factor, int nseg,
                const float* hyper, cudaStream_t s) {
  clip_apply_kernel<<<(unsigned)nchunks, kChunkThreads, 0, s>>>(g, n, chunks, factor, nseg, hyper);
}
void lamb_moments(const float* p, const float* g, float* m, float* v, int64_t n, const int64_t* chunks,
                  int64_t nchunks, float* partial, const float* hyper, cudaStream_t s) {
  lamb_moments_kernel<<<(unsigned)nchunks, kChunkThreads, 0, s>>>(p, g, m, v, n, chunks, nchunks, partial, hyper);
}
void lamb_apply(float* p, const float* m, const float* v, void* p16, int64_t n, const int64_t* chunks,
                int64_t nchunks, const float* phi, int nseg, const float* hyper, cudaStream_t s) {
  lamb_apply_kernel<<<(unsigned)nchunks, kChunkThreads, 0, s>>>(p, m, v, (__nv_bfloat16*)p16, n, chunks, phi, nseg,
                                                                hyper);
}
void grad_accumulate(float* g, float* accum, int64_t n, int steps, bool combine, cudaStream_t s) {
  const int64_t n4 = n / 4;
  if (combine)
    grad_accumulate_kernel<true><<<blocks_for(n4), 256, 0, s>>>(g, accum, n4, (float)steps);
  else
    grad_accumulate_kernel<false><<<blocks_for(n4), 256, 0, s>>>(g, accum, n4, (float)steps);
}
void ema_update(float* p, float* ema, void* p16, int64_t n, const float* hyper, cudaStream_t s) {
  const int64_t n4 = n / 4;
  ema_update_kernel<<<blocks_for(n4), 256, 0, s>>>(p, ema, (__nv_bfloat16*)p16, n4, hyper);
}
void cast_f32_to_bf16(const float* x, void* out, int64_t n, cudaStream_t s) {
  cast_kernel<<<blocks_for(n / 4), 256, 0, s>>>(x, (__nv_bfloat16*)out, n / 4);
}

}  // namespace b200
