// Classifier-head and stem-tail kernels (SURVEY.md K11, K14, K15): the bandwidth-bound glue around the two GEMM-shaped
// ends of the network.  The FC layer itself runs on the wgmma implicit-GEMM kernels (a 1x1 "convolution" over a 1x1
// image, csrc/conv_igemm.cuh / conv_wgrad.cu); what lives here is everything the reference's Dense + softmax head
// (P1/02:175) and MaxPool backward need besides the GEMMs:
//   * softmax_ce_head: bf16 logits + fp32 bias -> loss, accuracy, bf16 dlogits (padded columns zero) in one pass;
//   * fc_bias_grad: column sums of dlogits;
//   * stem_pool_bn_bwd: 3x3/2 max-pool backward (argmax scatter) fused with the stem BatchNorm+ReLU backward - the
//     112x112x64 pooled-gradient tensor is never written: pass 0 reduces sum(dz), sum(dz*y), pass 1 writes dy;
//     both rebuild the pooled gradient of a 16x16-pixel tile in shared memory (conflict-free colour-class scatter);
//   * pack_stem_weight: fp32 [49, 64, 3] master -> bf16 [64, 192] GEMM operand.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops_api.h"

namespace b200 {

namespace {

struct alignas(16) bf8 {
  __nv_bfloat162 v[4];
};
__device__ __forceinline__ void unpack8h(const bf8& p, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf8 pack8h(const float (&f)[8]) {
  bf8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16(x)); }

// Per-row loss weight of the weighted head kernels (Keras's class_weight / sample_weight): the batch's row weight
// rw[row] when rw is given, else the class table cw at the row's target class.  The unweighted instantiation is 1 and
// weigh() returns its argument untouched, so those kernels compile to the unweighted code.  The weighted product is a
// correctly rounded, uncontracted __fmul_rn: w = 1 gives the unweighted bits, a power of two scales them exactly.
template <bool kWeighted>
__device__ __forceinline__ float row_weight(const float* __restrict__ cw, const float* __restrict__ rw, int row,
                                            int target) {
  if (!kWeighted) return 1.f;
  return rw != nullptr ? rw[row] : cw[target];
}
template <bool kWeighted>
__device__ __forceinline__ float weigh(float v, float w) {
  return kWeighted ? __fmul_rn(v, w) : v;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ softmax CE head
// One warp per row.  logit[k] = bf16 logits16[row, k] + bias[k] for k < K (row pitch ld >= K, padded columns ignored).
// kWeighted: the row's loss, loss stat and dlogits are scaled by w = rw[row] (rw != nullptr) or cw[label]
// (row_weight); the unweighted instantiation reads neither pointer.
template <bool kWeighted>
__global__ void softmax_ce_head_kernel(const __nv_bfloat16* __restrict__ logits16, int ld,
                                       const float* __restrict__ bias, const int64_t* __restrict__ labels,
                                       float* __restrict__ logits32, __nv_bfloat16* __restrict__ dlogits16,
                                       float* __restrict__ loss_rows, float* __restrict__ stats, int B, int K,
                                       float grad_scale, const float* __restrict__ cw, const float* __restrict__ rw) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= B) return;
  const __nv_bfloat16* row = logits16 + (int64_t)warp * ld;
  const int label = (int)labels[warp];
  const float w = row_weight<kWeighted>(cw, rw, warp, label);
  float mx = -3.0e38f;
  int amax = 0;
  for (int k = lane; k < K; k += 32) {
    const float v = __bfloat162float(row[k]) + bias[k];
    if (logits32 != nullptr) logits32[(int64_t)warp * K + k] = v;
    if (v > mx) { mx = v; amax = k; }
  }
  for (int o = 16; o; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
    if (om > mx || (om == mx && oa < amax)) { mx = om; amax = oa; }
  }
  float se = 0.f;
  for (int k = lane; k < K; k += 32) se += __expf(__bfloat162float(row[k]) + bias[k] - mx);
  for (int o = 16; o; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  const float lse = mx + __logf(se);
  const float inv = 1.f / se;
  if (dlogits16 != nullptr) {
    __nv_bfloat16* drow = dlogits16 + (int64_t)warp * ld;
    for (int k = lane; k < ld; k += 32) {
      float d = 0.f;
      if (k < K) {
        const float pk = __expf(__bfloat162float(row[k]) + bias[k] - mx) * inv;
        d = weigh<kWeighted>((pk - (k == label ? 1.f : 0.f)) * grad_scale, w);
      }
      drow[k] = __float2bfloat16(d);
    }
  }
  if (lane == 0) {
    const float l = weigh<kWeighted>(lse - (__bfloat162float(row[label]) + bias[label]), w);
    if (loss_rows != nullptr) loss_rows[warp] = l;
    atomicAdd(stats, l);
    atomicAdd(stats + 1, amax == label ? 1.f : 0.f);
  }
}
void softmax_ce_head(const void* logits16, int ld, const float* bias, const int64_t* labels, float* logits32,
                     void* dlogits16, float* loss_rows, float* stats, int B, int K, float grad_scale, const float* cw,
                     const float* rw, cudaStream_t s) {
  const int threads = 128;
  const int blocks = (B * 32 + threads - 1) / threads;
  const auto kernel = cw != nullptr || rw != nullptr ? softmax_ce_head_kernel<true> : softmax_ce_head_kernel<false>;
  kernel<<<blocks, threads, 0, s>>>(
    (const __nv_bfloat16*)logits16, ld, bias, labels, logits32, (__nv_bfloat16*)dlogits16, loss_rows, stats, B, K,
    grad_scale, cw, rw);
}

// softmax_ce_head against a soft target, for MixUp / CutMix and label smoothing (eps):
//   target_k = (1 - eps) (lambda [k = y] + mu [k = y_partner]) + eps / K,   lambda = 1 - mu,  mu = num / den (mix row)
//   loss     = sum_k target_k (lse - logit_k) = (1 - eps) (lambda (lse - l_y) + mu (lse - l_p)) + eps / K sum_k (lse - l_k)
//   dlogits  = (p_k - target_k) * grad_scale;   correct: argmax(logits) == argmax of the unsmoothed target
//   lambda [k = y] + mu [k = y_partner], lowest index on ties (Keras smooths inside the loss; its accuracy metric sees
//   the mixed labels without smoothing).
// sum_k (lse - l_k) is accumulated as sum_k (max - l_k) + K (lse - max): every term is >= 0.  mu is a correctly rounded
// division (__fdiv_rn, also under --use_fast_math).  With mu = 0 and eps = 0 every product by lambda, 1 - eps, mu or
// eps / K is by 1 or 0, so each output is bit for bit softmax_ce_head's.  That argmax is decided on the integers: y when
// 2 num < den, y_partner when 2 num > den, the lower of the two on a tie.
// kWeighted: the class table cw is read at that argmax (the row's target class).
template <bool kWeighted>
__global__ void softmax_ce_soft_head_kernel(const __nv_bfloat16* __restrict__ logits16, int ld,
                                            const float* __restrict__ bias, const int64_t* __restrict__ labels,
                                            const int4* __restrict__ mix, float eps, float* __restrict__ logits32,
                                            __nv_bfloat16* __restrict__ dlogits16, float* __restrict__ loss_rows,
                                            float* __restrict__ stats, int B, int K, float grad_scale,
                                            const float* __restrict__ cw, const float* __restrict__ rw) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= B) return;
  const __nv_bfloat16* row = logits16 + (int64_t)warp * ld;
  const int label = (int)labels[warp];
  int plabel = label, target = label;
  float mu = 0.f;
  if (mix != nullptr) {
    const int4 m0 = mix[2 * warp], m1 = mix[2 * warp + 1];
    plabel = (int)labels[(unsigned)m0.x < (unsigned)B ? m0.x : warp];
    mu = __fdiv_rn((float)m1.z, (float)m1.w);
    if (plabel != label) {
      const int64_t twice = 2 * (int64_t)m1.z;
      target = twice < m1.w ? label : twice > m1.w ? plabel : min(label, plabel);
    }
  }
  const float w = row_weight<kWeighted>(cw, rw, warp, target);
  const float lam = 1.f - mu, keep = 1.f - eps, epsk = __fdiv_rn(eps, (float)K);
  float mx = -3.0e38f;
  int amax = 0;
  for (int k = lane; k < K; k += 32) {
    const float v = __bfloat162float(row[k]) + bias[k];
    if (logits32 != nullptr) logits32[(int64_t)warp * K + k] = v;
    if (v > mx) { mx = v; amax = k; }
  }
  for (int o = 16; o; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
    if (om > mx || (om == mx && oa < amax)) { mx = om; amax = oa; }
  }
  float se = 0.f, sd = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float v = __bfloat162float(row[k]) + bias[k];
    se += __expf(v - mx);
    sd += mx - v;
  }
  for (int o = 16; o; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sd += __shfl_xor_sync(0xffffffffu, sd, o);
  }
  const float lse = mx + __logf(se);   // as softmax_ce_head writes it (the compiler fuses the log's scale and the add)
  const float inv = 1.f / se;
  if (dlogits16 != nullptr) {
    __nv_bfloat16* drow = dlogits16 + (int64_t)warp * ld;
    for (int k = lane; k < ld; k += 32) {
      float d = 0.f;
      if (k < K) {
        const float pk = __expf(__bfloat162float(row[k]) + bias[k] - mx) * inv;
        const float tk = keep * ((k == label ? lam : 0.f) + (k == plabel ? mu : 0.f)) + epsk;
        d = weigh<kWeighted>((pk - tk) * grad_scale, w);
      }
      drow[k] = __float2bfloat16(d);
    }
  }
  if (lane == 0) {
    const float ly = __bfloat162float(row[label]) + bias[label];
    const float lp = __bfloat162float(row[plabel]) + bias[plabel];
    const float l = weigh<kWeighted>(keep * (lam * (lse - ly) + mu * (lse - lp)) + epsk * (sd + (float)K * (lse - mx)),
                                     w);
    if (loss_rows != nullptr) loss_rows[warp] = l;
    atomicAdd(stats, l);
    atomicAdd(stats + 1, amax == target ? 1.f : 0.f);
  }
}
void softmax_ce_soft_head(const void* logits16, int ld, const float* bias, const int64_t* labels, const int32_t* mix,
                          float eps, float* logits32, void* dlogits16, float* loss_rows, float* stats, int B, int K,
                          float grad_scale, const float* cw, const float* rw, cudaStream_t s) {
  const int threads = 128;
  const int blocks = (B * 32 + threads - 1) / threads;
  const auto kernel =
      cw != nullptr || rw != nullptr ? softmax_ce_soft_head_kernel<true> : softmax_ce_soft_head_kernel<false>;
  kernel<<<blocks, threads, 0, s>>>(
    (const __nv_bfloat16*)logits16, ld, bias, labels, (const int4*)mix, eps, logits32, (__nv_bfloat16*)dlogits16,
    loss_rows, stats, B, K, grad_scale, cw, rw);
}

// softmax_ce_soft_head plus knowledge distillation from a teacher's logits t (bf16 tlogits16 [B, tld] + tbias), at
// weight alpha and temperature T; s = the student's logits (bias included):
//   loss    = alpha * ce + (1 - alpha) * kd,   ce = softmax_ce_soft_head's loss,   kd = T^2 KL(r || q)
//   KL      = sum_k r_k (log r_k - log q_k),   r = softmax(t / T), q = softmax(s / T)   (the two log-softmaxes, no clipping)
//   dlogits = (alpha (p_k - target_k) + (1 - alpha) T (q_k - r_k)) * grad_scale
//   stats   = [sum loss, correct, sum ce, sum kd]
// The student part is softmax_ce_soft_head's code, then scaled by alpha and added to the distillation part scaled by
// 1 - alpha with correctly rounded, uncontracted operations: at alpha = 1 that is a product by 1 plus a product by 0, so
// loss, dlogits and loss_rows are bit for bit softmax_ce_soft_head's (and softmax_ce_head's at eps = 0 without mix
// rows).  The teacher's row is only read: its max, then exp((t - tmax) / T) twice.
// kWeighted: as softmax_ce_soft_head's, with the two term stats weighted too.
template <bool kWeighted>
__global__ void softmax_kd_head_kernel(const __nv_bfloat16* __restrict__ logits16, int ld,
                                       const float* __restrict__ bias, const __nv_bfloat16* __restrict__ tlogits16,
                                       int tld, const float* __restrict__ tbias, const int64_t* __restrict__ labels,
                                       const int4* __restrict__ mix, float eps, float alpha, float T,
                                       float* __restrict__ logits32, __nv_bfloat16* __restrict__ dlogits16,
                                       float* __restrict__ loss_rows, float* __restrict__ stats, int B, int K,
                                       float grad_scale, const float* __restrict__ cw, const float* __restrict__ rw) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= B) return;
  const __nv_bfloat16* row = logits16 + (int64_t)warp * ld;
  const __nv_bfloat16* trow = tlogits16 + (int64_t)warp * tld;
  const int label = (int)labels[warp];
  int plabel = label, target = label;
  float mu = 0.f;
  if (mix != nullptr) {
    const int4 m0 = mix[2 * warp], m1 = mix[2 * warp + 1];
    plabel = (int)labels[(unsigned)m0.x < (unsigned)B ? m0.x : warp];
    mu = __fdiv_rn((float)m1.z, (float)m1.w);
    if (plabel != label) {
      const int64_t twice = 2 * (int64_t)m1.z;
      target = twice < m1.w ? label : twice > m1.w ? plabel : min(label, plabel);
    }
  }
  const float w = row_weight<kWeighted>(cw, rw, warp, target);
  const float lam = 1.f - mu, keep = 1.f - eps, epsk = __fdiv_rn(eps, (float)K);
  const float beta = 1.f - alpha, invT = __fdiv_rn(1.f, T);
  float mx = -3.0e38f, tmx = -3.0e38f;
  int amax = 0;
  for (int k = lane; k < K; k += 32) {
    const float v = __bfloat162float(row[k]) + bias[k];
    if (logits32 != nullptr) logits32[(int64_t)warp * K + k] = v;
    if (v > mx) { mx = v; amax = k; }
    tmx = fmaxf(tmx, __bfloat162float(trow[k]) + tbias[k]);
  }
  for (int o = 16; o; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oa = __shfl_xor_sync(0xffffffffu, amax, o);
    if (om > mx || (om == mx && oa < amax)) { mx = om; amax = oa; }
    tmx = fmaxf(tmx, __shfl_xor_sync(0xffffffffu, tmx, o));
  }
  // the max of s / T and t / T is max / T (T > 0): (v - max) / T <= 0 in every exponent
  float se = 0.f, sd = 0.f, seT = 0.f, teT = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float v = __bfloat162float(row[k]) + bias[k];
    se += __expf(v - mx);
    sd += mx - v;
    seT += __expf((v - mx) * invT);
    teT += __expf((__bfloat162float(trow[k]) + tbias[k] - tmx) * invT);
  }
  for (int o = 16; o; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sd += __shfl_xor_sync(0xffffffffu, sd, o);
    seT += __shfl_xor_sync(0xffffffffu, seT, o);
    teT += __shfl_xor_sync(0xffffffffu, teT, o);
  }
  const float lse = mx + __logf(se);
  const float inv = 1.f / se;
  const float lseT = __logf(seT), lteT = __logf(teT);   // log-normalisers of (s - max) / T and (t - tmax) / T
  const float invS = 1.f / seT, invTe = 1.f / teT;
  float kl = 0.f;
  __nv_bfloat16* drow = dlogits16 != nullptr ? dlogits16 + (int64_t)warp * ld : nullptr;
  for (int k = lane; k < (drow != nullptr ? ld : K); k += 32) {
    float d = 0.f;
    if (k < K) {
      const float v = __bfloat162float(row[k]) + bias[k];
      const float zs = (v - mx) * invT;
      const float zt = (__bfloat162float(trow[k]) + tbias[k] - tmx) * invT;
      const float rk = __expf(zt) * invTe;
      kl += rk * ((zt - lteT) - (zs - lseT));
      if (drow != nullptr) {
        const float pk = __expf(v - mx) * inv;
        const float tk = keep * ((k == label ? lam : 0.f) + (k == plabel ? mu : 0.f)) + epsk;
        const float qk = __expf(zs) * invS;
        const float ds = (pk - tk) * grad_scale;   // softmax_ce_soft_head's dlogit
        d = weigh<kWeighted>(__fadd_rn(__fmul_rn(alpha, ds), __fmul_rn(beta, T * (qk - rk) * grad_scale)), w);
      }
    }
    if (drow != nullptr) drow[k] = __float2bfloat16(d);
  }
  for (int o = 16; o; o >>= 1) kl += __shfl_xor_sync(0xffffffffu, kl, o);
  if (lane == 0) {
    const float ly = __bfloat162float(row[label]) + bias[label];
    const float lp = __bfloat162float(row[plabel]) + bias[plabel];
    const float ce = keep * (lam * (lse - ly) + mu * (lse - lp)) + epsk * (sd + (float)K * (lse - mx));
    const float kd = T * T * kl;
    // no contraction: alpha = 1 gives ce
    const float l = weigh<kWeighted>(__fadd_rn(__fmul_rn(alpha, ce), __fmul_rn(beta, kd)), w);
    if (loss_rows != nullptr) loss_rows[warp] = l;
    atomicAdd(stats, l);
    atomicAdd(stats + 1, amax == target ? 1.f : 0.f);
    atomicAdd(stats + 2, weigh<kWeighted>(ce, w));
    atomicAdd(stats + 3, weigh<kWeighted>(kd, w));
  }
}
void softmax_kd_head(const void* logits16, int ld, const float* bias, const void* tlogits16, int tld,
                     const float* tbias, const int64_t* labels, const int32_t* mix, float eps, float alpha, float T,
                     float* logits32, void* dlogits16, float* loss_rows, float* stats, int B, int K, float grad_scale,
                     const float* cw, const float* rw, cudaStream_t s) {
  const int threads = 128;
  const int blocks = (B * 32 + threads - 1) / threads;
  const auto kernel = cw != nullptr || rw != nullptr ? softmax_kd_head_kernel<true> : softmax_kd_head_kernel<false>;
  kernel<<<blocks, threads, 0, s>>>(
    (const __nv_bfloat16*)logits16, ld, bias, (const __nv_bfloat16*)tlogits16, tld, tbias, labels, (const int4*)mix,
    eps, alpha, T, logits32, (__nv_bfloat16*)dlogits16, loss_rows, stats, B, K, grad_scale, cw, rw);
}

// dbias[k] = sum_b dlogits16[b, k]   (thread per column: coalesced across k for every row)
__global__ void fc_bias_grad_kernel(const __nv_bfloat16* __restrict__ dl, int ld, float* __restrict__ dbias, int B, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int b = 0;
  for (; b + 4 <= B; b += 4) {
    a0 += __bfloat162float(dl[(int64_t)(b + 0) * ld + k]);
    a1 += __bfloat162float(dl[(int64_t)(b + 1) * ld + k]);
    a2 += __bfloat162float(dl[(int64_t)(b + 2) * ld + k]);
    a3 += __bfloat162float(dl[(int64_t)(b + 3) * ld + k]);
  }
  for (; b < B; ++b) a0 += __bfloat162float(dl[(int64_t)b * ld + k]);
  dbias[k] = (a0 + a1) + (a2 + a3);
}
void fc_bias_grad(const void* dlogits16, int ld, float* dbias, int B, int K, cudaStream_t s) {
  fc_bias_grad_kernel<<<(K + 127) / 128, 128, 0, s>>>((const __nv_bfloat16*)dlogits16, ld, dbias, B, K);
}

// ------------------------------------------------------------------------------------------------ stem weight pack
// fp32 [49, 64, 3] (tap, co, c) -> bf16 [64, 192] with k = tap*3 + c (columns 147.. are zero)
__global__ void pack_stem_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * 192) return;
  const int co = i / 192, k = i - co * 192;
  float v = 0.f;
  if (k < 147) v = w[((k / 3) * 64 + co) * 3 + (k % 3)];
  out[i] = __float2bfloat16(v);
}
void pack_stem_weight(const float* w, void* out, cudaStream_t s) {
  pack_stem_weight_kernel<<<(64 * 192 + 255) / 256, 256, 0, s>>>(w, (__nv_bfloat16*)out);
}

// ------------------------------------------------------------------------------------------------ stem tail backward
// Backward of  p = maxpool3x3/2( relu( y*scale + shift ) )  for the 64-channel stem, without materialising the pooled
// gradient on the 2Ho x 2Wo grid:
//   da[h, w]  = sum over the <= 4 windows containing (h, w) whose saved argmax is this position of (g1 + g2)[ho, wo]
//   dz        = da * [y*scale + shift > 0]
//   PASS 0:   sum_dz += dz, sum_dzy += dz * y          (per channel; one flush of atomics per CTA)
//   PASS 1:   dy = cA*dz + cB*y + cC
// v1 of this kernel GATHERED per input pixel (compare the saved argmax of up to four windows, per channel) and was
// instruction-bound - slower than the three-kernel path it replaced.  v2 SCATTERS: every window contributes its gradient to exactly ONE pixel (its argmax), so
// a CTA builds the da tile of 16x16 pixels x 64 channels in shared memory (fp32, 64 KB) by read-modify-write:
//   * a warp handles (window, 32-channel half); lane = channel, so the smem bank is the lane whatever pixel is hit;
//   * windows are processed in four colour classes (row parity x column parity): windows of one class have disjoint 3x3
//     footprints, so plain (non-atomic) updates are race-free inside a class; __syncthreads between classes
//     (a shared-memory fp32 atomicAdd per element would serialise colliding lanes and dominate);
//   * then the pixel phase reads da from smem, y from global, and reduces / applies.
constexpr int kPoolTile = 8;
constexpr int kPoolWin = kPoolTile + 1;
constexpr int kStemDaBytes = 16 * 16 * 64 * 4;

template <int PASS>
__global__ void __launch_bounds__(256, 3)
stem_pool_bn_bwd_kernel(const uint8_t* __restrict__ idx, const __nv_bfloat16* __restrict__ g1,
                        const __nv_bfloat16* __restrict__ g2, const __nv_bfloat16* __restrict__ y,
                        const float* __restrict__ scale, const float* __restrict__ shift,
                        const float* __restrict__ cA, const float* __restrict__ cB, const float* __restrict__ cC,
                        __nv_bfloat16* __restrict__ dy, float* __restrict__ sum_dz, float* __restrict__ sum_dzy, int N,
                        int Ho, int Wo) {
  constexpr int C = 64;
  extern __shared__ __align__(16) float da[];  // [256 pixels][64 channels]
  __shared__ float red[2][8][C];
  const int H = 2 * Ho, W = 2 * Wo;
  const int tiles_h = Ho / kPoolTile, tiles_w = Wo / kPoolTile;
  const int num_tiles = N * tiles_h * tiles_w;
  const int t = threadIdx.x;
  const int warp = t >> 5, lane = t & 31;
  const int cv = t & 7;
  const int pl = t >> 3;  // 0..31: pixel lane; pixels p = pl + 32*i
  float sc[8], sh[8], A[8], B[8], Cc[8], t0[8], t1[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sc[k] = scale[cv * 8 + k];
    sh[k] = shift[cv * 8 + k];
    t0[k] = t1[k] = 0.f;
    if (PASS == 1) {
      A[k] = cA[cv * 8 + k];
      B[k] = cB[cv * 8 + k];
      Cc[k] = cC[cv * 8 + k];
    }
  }
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int tb = tile % tiles_w;
    const int rest = tile / tiles_w;
    const int ta = rest % tiles_h;
    const int n = rest / tiles_h;
    const int a0 = ta * kPoolTile, b0 = tb * kPoolTile;
    __syncthreads();  // the previous tile's pixel phase is done with da
    for (int i = t; i < 16 * 16 * C / 4; i += 256) reinterpret_cast<float4*>(da)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
#pragma unroll 1
    for (int cls = 0; cls < 4; ++cls) {
      const int ci = cls >> 1, cj = cls & 1;
      const int nwj = (kPoolWin - 1 - cj) / 2 + 1;
      const int items = ((kPoolWin - 1 - ci) / 2 + 1) * nwj * 2;
      // A warp owns at most kMaxIt = 7 (window, half) items of a class (<= 25 windows x 2 halves over 8 warps): ALL their
      // global loads are issued before the first read-modify-write, so ~7 x 5 bytes per lane are in flight instead of one
      // item's (v2a: ncu 58 % long-scoreboard stalls in this loop, 16 % DRAM throughput).
      constexpr int kMaxIt = 7;
      int a_[kMaxIt];   // bits 0-7 argmax position, 8-15 wi, 16-23 wj, bit 30 = item present
      float g_[kMaxIt];
      const int ch = (warp & 1) * 32 + lane;  // it = warp + 8q: the channel half of all of a warp's items is warp & 1
#pragma unroll
      for (int q = 0; q < kMaxIt; ++q) {
        const int it = warp + 8 * q;
        a_[q] = 0;
        g_[q] = 0.f;
        if (it < items) {
          const int w = it >> 1;
          const int wi = ci + 2 * (w / nwj), wj = cj + 2 * (w % nwj);
          const int ho = a0 + wi, wo = b0 + wj;
          if (ho < Ho && wo < Wo) {  // warp-uniform
            const int64_t o = ((((int64_t)n * Ho + ho) * Wo + wo) * C) + ch;
            a_[q] = static_cast<int>(idx[o]) | (wi << 8) | (wj << 16) | (1 << 30);
            g_[q] = __bfloat162float(g1[o]);
            if (g2 != nullptr) g_[q] += __bfloat162float(g2[o]);
          }
        }
      }
#pragma unroll
      for (int q = 0; q < kMaxIt; ++q) {
        if (a_[q] != 0) {
          const int a = a_[q] & 0xFF, wi = (a_[q] >> 8) & 0xFF, wj = (a_[q] >> 16) & 0xFF;
          const int r = (a * 11) >> 5;  // a / 3 for a in 0..8
          const int row = 2 * wi - 1 + r, col = 2 * wj - 1 + (a - 3 * r);
          if (static_cast<unsigned>(row) < 16u && static_cast<unsigned>(col) < 16u) da[(row * 16 + col) * C + ch] += g_[q];
        }
      }
      __syncthreads();
    }
    const int pw = pl & 15;
#pragma unroll 2
    for (int i = 0; i < 8; ++i) {
      const int ph = (pl >> 4) + 2 * i;
      const int h = 2 * a0 + ph, w = 2 * b0 + pw;
      const float4 d0 = *reinterpret_cast<const float4*>(&da[(ph * 16 + pw) * C + cv * 8]);
      const float4 d1 = *reinterpret_cast<const float4*>(&da[(ph * 16 + pw) * C + cv * 8 + 4]);
      const float acc[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
      const int64_t off = ((((int64_t)n * H + h) * W + w) * C) + cv * 8;
      float yy[8];
      unpack8h(*reinterpret_cast<const bf8*>(y + off), yy);
      float dz[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        // bf16 rounding of the pooled gradient: same values as the materialised path (maxpool_bwd -> bf16 tensor)
        const float a = bf16_round(acc[k]);
        dz[k] = fmaf(yy[k], sc[k], sh[k]) > 0.f ? a : 0.f;
      }
      if (PASS == 0) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          t0[k] += dz[k];
          t1[k] = fmaf(dz[k], yy[k], t1[k]);
        }
      } else {
        float o8[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) o8[k] = fmaf(A[k], dz[k], fmaf(B[k], yy[k], Cc[k]));
        *reinterpret_cast<bf8*>(dy + off) = pack8h(o8);
      }
    }
  }
  if (PASS == 0) {
    // lanes with equal (lane & 7) own the same 8 channels: fold the 4 pixel lanes of a warp, then the 8 warps
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      t0[k] += __shfl_xor_sync(0xffffffffu, t0[k], 8);
      t0[k] += __shfl_xor_sync(0xffffffffu, t0[k], 16);
      t1[k] += __shfl_xor_sync(0xffffffffu, t1[k], 8);
      t1[k] += __shfl_xor_sync(0xffffffffu, t1[k], 16);
    }
    __syncthreads();
    if (lane < 8) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        red[0][warp][lane * 8 + k] = t0[k];
        red[1][warp][lane * 8 + k] = t1[k];
      }
    }
    __syncthreads();
    if (t < 2 * C) {
      const int which = t / C, c = t % C;
      float a = 0.f;
#pragma unroll
      for (int wv = 0; wv < 8; ++wv) a += red[which][wv][c];
      atomicAdd((which == 0 ? sum_dz : sum_dzy) + c, a);
    }
  }
}

// pass 0: reduce (sum_dz, sum_dzy accumulate);  pass 1: apply (dy written)
void stem_pool_bn_bwd(int pass, const void* idx, const void* g1, const void* g2, const void* y, const float* scale,
                      const float* shift, const float* cA, const float* cB, const float* cC, void* dy, float* sum_dz,
                      float* sum_dzy, int N, int Ho, int Wo, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(stem_pool_bn_bwd_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStemDaBytes);
    cudaFuncSetAttribute(stem_pool_bn_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStemDaBytes);
    attr_set = true;
  }
  const int tiles = N * (Ho / kPoolTile) * (Wo / kPoolTile);
  int grid = 132 * 3;
  if (grid > tiles) grid = tiles;
  if (pass == 0)
    stem_pool_bn_bwd_kernel<0><<<grid, 256, kStemDaBytes, s>>>((const uint8_t*)idx, (const __nv_bfloat16*)g1,
                                                               (const __nv_bfloat16*)g2, (const __nv_bfloat16*)y, scale,
                                                               shift, cA, cB, cC, (__nv_bfloat16*)dy, sum_dz, sum_dzy, N, Ho, Wo);
  else
    stem_pool_bn_bwd_kernel<1><<<grid, 256, kStemDaBytes, s>>>((const uint8_t*)idx, (const __nv_bfloat16*)g1,
                                                               (const __nv_bfloat16*)g2, (const __nv_bfloat16*)y, scale,
                                                               shift, cA, cB, cC, (__nv_bfloat16*)dy, sum_dz, sum_dzy, N, Ho, Wo);
}

}  // namespace b200
