// Plain (torch-free) launch interface of the bandwidth-bound kernels and fused optimizers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

// Optional in-kernel BatchNorm coefficient computation (replaces a separate bn_finalize / bn_bwd_coeffs launch on the
// critical path).  sum == nullptr / sum_dz == nullptr selects the unfused behaviour (coefficients read from arrays).
struct BnFwdFuse {
  const float* sum;      // per-channel sum(y), sum(y^2) accumulated by the conv epilogue (zeroed once per step by the engine)
  const float* sqsum;
  const float* gamma;
  const float* beta;
  float* running_mean;   // updated by the first row-block
  float* running_var;
  float* mean;           // written by the first row-block for the backward pass
  float* invstd;
  float* scale;
  float* shift;
  float inv_count, unbias, momentum, eps;
};
struct BnBwdFuse {
  const float* sum_dz;   // per-channel sum(dz), sum(dz*y) (zeroed once per step by the engine)
  const float* sum_dzy;
  const float* gamma;
  const float* mean;
  const float* invstd;
  float* dgamma;         // written by the first row-block
  float* dbeta;
  float inv_count;
};
void bn_apply_fused(const void* y, const BnFwdFuse& f, const void* res, const BnFwdFuse* res_f, void* out, void* mask,
                    int64_t M, int C, bool relu, cudaStream_t s);
void bn_bwd_apply_fused(const void* g, const void* y, const float* scale, const float* shift, const BnBwdFuse& f, void* dy,
                        int64_t M, int C, cudaStream_t s);
void bn_finalize(float* sum, float* sqsum, double count, const float* gamma, const float* beta, float* running_mean,
                 float* running_var, float momentum, float eps, float* mean, float* invstd, float* scale,
                 float* shift, int C, bool training, cudaStream_t s);
// rows per loop iteration of the BatchNorm apply / backward-apply kernels: 1 (default), 2 or 4 - bit-identical results
void set_bn_rows_unroll(int u);
int get_bn_rows_unroll();
void bn_apply(const void* y, const float* scale, const float* shift, const void* res, const float* res_scale,
              const float* res_shift, void* out, void* mask, int64_t M, int C, int act, cudaStream_t s);
void channel_stats(const void* y, float* sum, float* sqsum, int64_t M, int C, cudaStream_t s);
void bn_bwd_reduce(int mode, const void* g1, const void* g2, const void* outp, const void* y, const float* scale,
                   const float* shift, void* dz_out, float* sum_dz, float* sum_dzy, int64_t M, int C, cudaStream_t s);
void bn_bwd_coeffs(float* sum_dz, float* sum_dzy, const float* gamma, const float* mean, const float* invstd,
                   double count, float* dgamma, float* dbeta, float* cA, float* cB, float* cC, int C, bool inference,
                   cudaStream_t s);
void bn_bwd_apply(const void* g, const void* y, const float* scale, const float* shift, const float* cA,
                  const float* cB, const float* cC, void* dy, int64_t M, int C, cudaStream_t s);
void maxpool_fwd(const void* x, void* out, void* idx, int N, int H, int W, int C, cudaStream_t s);
void bn_relu_maxpool_fwd(const void* y, const float* scale, const float* shift, void* out, void* idx, int N, int H,
                         int W, int C, cudaStream_t s);
void maxpool_bwd(const void* idx, const void* g1, const void* g2, void* dx, int N, int H, int W, int C,
                 cudaStream_t s);
void gap_fwd(const void* x, void* out, int N, int HW, int C, float drop_p, uint64_t seed, cudaStream_t s);
void gap_bwd(const void* dout, void* dx, int N, int HW, int C, float drop_p, uint64_t seed, cudaStream_t s);
void softmax_ce(const float* logits, const int64_t* labels, float* dlogits, float* loss_rows, float* stats, int B,
                int K, float grad_scale, cudaStream_t s);
// The three heads take an optional per-row loss weight (Keras class_weight / sample_weight): cw = fp32 [K] class table
// read at the row's target class, or rw = fp32 [B] row weights, at most one of them; both nullptr launch the unweighted
// kernel.  Weighted: loss_rows, the loss stat(s) and dlogits are scaled by the row's weight; the correct count is not.
void softmax_ce_head(const void* logits16, int ld, const float* bias, const int64_t* labels, float* logits32,
                     void* dlogits16, float* loss_rows, float* stats, int B, int K, float grad_scale, const float* cw,
                     const float* rw, cudaStream_t s);
void fc_bias_grad(const void* dlogits16, int ld, float* dbias, int B, int K, cudaStream_t s);
void pack_stem_weight(const float* w, void* out, cudaStream_t s);
void stem_pool_bn_bwd(int pass, const void* idx, const void* g1, const void* g2, const void* y, const float* scale,
                      const float* shift, const float* cA, const float* cB, const float* cC, void* dy, float* sum_dz,
                      float* sum_dzy, int N, int Ho, int Wo, cudaStream_t s);
void mbv2_stem(const uint8_t* x, const float* w, const float* scale, const float* shift, void* out, int N, int H, int W,
               int ldc, float mul, float add, cudaStream_t s);
void dwconv3x3(const void* x, const float* w, const float* scale, const float* shift, void* out, int N, int H, int W, int C,
               int stride, int tile_w, cudaStream_t s);
// Training-mode BatchNorm variants: c = conv(x) stored as bf16, no affine / clamp, and sum[c] += sum(c), sqsum[c] +=
// sum(c^2) of the stored (bf16) values (zeroed by the caller).  mbv2_stem_stats writes and sums the 32 real channels.
void mbv2_stem_stats(const uint8_t* x, const float* w, void* out, float* sum, float* sqsum, int N, int H, int W, int ldc,
                     float mul, float add, cudaStream_t s);
void dwconv3x3_stats(const void* x, const float* w, void* out, float* sum, float* sqsum, int N, int H, int W, int C,
                     int stride, int tile_w, cudaStream_t s);
void preprocess_u8(const uint8_t* x, void* out, int64_t npix, int cpad, float mul, float add, cudaStream_t s);
void resize_bilinear_u8(const uint8_t* x, uint8_t* out, int N, int H, int W, int OH, int OW, bool planar, cudaStream_t s);
void weight_prep(const float* w, void* wf, void* wd, int taps, int cout, int cin, cudaStream_t s);
void weight_prep_batched(const float* params, void* wd, const int64_t* table, int layers, int64_t total,
                         cudaStream_t s);

// Fused flat-buffer optimizers.  `hyper` is a DEVICE array (so LR schedules do not invalidate CUDA graphs):
//   [0] lr  [1] momentum/beta1  [2] beta2/rho  [3] eps  [4] weight_decay  [5] grad_scale  [6] bias_corr1  [7] bias_corr2
//   [8] clip threshold  [9] the host's grad_scale
//   [10] EMA decay d  [11] 1 - d  [12] EMA overwrite flag (nonzero: p = ema after the average)  [13..15] unused
// The update kernels read slots 0-7 only (their binding accepts >= kHyperLen); the clip, LAMB and EMA passes need all
// kHyperSlots.  The global-norm clip writes [5] = [9] * factor, so repeating a step never compounds the factor.
constexpr int kHyperLen = 8;
constexpr int kHyperSlots = 16;
enum : int {
  kHypLr, kHypMom, kHypBeta2, kHypEps, kHypWd, kHypGScale, kHypBc1, kHypBc2,
  kHypClip, kHypHostGScale, kHypEmaDecay, kHypEmaRest, kHypEmaOverwrite
};
// Elementwise update rules (csrc/optim_rules.cuh), one per kernel instantiation.
enum OptimRule : int {
  kRuleSgd, kRuleSgdNesterov, kRuleAdam, kRuleAdamW, kRuleAdadelta, kRuleRmsprop, kRuleRmspropMomentum,
  kRuleRmspropCentered, kRuleRmspropCenteredMomentum, kRuleAdagrad, kRuleAdamax, kNumOptimRules
};
// number of state buffers the rule reads and writes
int optim_rule_states(OptimRule rule);
// state: optim_rule_states(rule) fp32 buffers of n elements, in the rule's order; p16 may be nullptr
void optim_step(OptimRule rule, float* p, const float* g, float* const* state, void* p16, int64_t n,
                const float* hyper, cudaStream_t s);
// Chunk table: int64 [nchunks, kChunkFields] = (lo, hi, segment), lo / hi multiples of 4, hi - lo <= kChunkMax.
// Segment table: int64 [nseg, 2] = (first chunk, end chunk).  partial: fp32 [nchunks] (x2 for LAMB);
// sums: fp32 [2, nseg + 1] (per-segment sums of squares, then the total); factor: fp32 [nseg].
constexpr int kChunkFields = 3;
constexpr int64_t kChunkMax = 8192;
constexpr int kMaxSegments = 1 << 20;
enum : int { kFinSums = 0, kFinClipGlobal = 1, kFinClipNorm = 2, kFinLamb = 3 };
void segment_sumsq(const float* g, int64_t n, const int64_t* chunks, int64_t nchunks, float* partial,
                   const float* hyper, cudaStream_t s);
void segment_finalize(const float* partial, int64_t nchunks, const int64_t* segs, int nseg, float* sums,
                      float* factor, float* hyper, int mode, cudaStream_t s);
// factor != nullptr: clipnorm (g *= grad_scale * factor[segment]); nullptr: clipvalue (clamp(g * grad_scale, -c, c))
void clip_apply(float* g, int64_t n, const int64_t* chunks, int64_t nchunks, const float* factor, int nseg,
                const float* hyper, cudaStream_t s);
void lamb_moments(const float* p, const float* g, float* m, float* v, int64_t n, const int64_t* chunks,
                  int64_t nchunks, float* partial, const float* hyper, cudaStream_t s);
void lamb_apply(float* p, const float* m, const float* v, void* p16, int64_t n, const int64_t* chunks,
                int64_t nchunks, const float* phi, int nseg, const float* hyper, cudaStream_t s);
// Gradient accumulation (Keras gradient_accumulation_steps): combine = false: accum += g; combine = true:
// g = (accum + g) / steps, accum = 0.
void grad_accumulate(float* g, float* accum, int64_t n, int steps, bool combine, cudaStream_t s);
// Weight EMA after an update, from hyper slots kHypEmaDecay..kHypEmaOverwrite; p16 may be nullptr.
void ema_update(float* p, float* ema, void* p16, int64_t n, const float* hyper, cudaStream_t s);
void cast_f32_to_bf16(const float* x, void* out, int64_t n, cudaStream_t s);

// MobileNetV2 fine-tuning backward (csrc/mobilenet_bwd.cu).  relu6_mask_reduce: with c (training-mode BatchNorm, the
// conv output before normalisation) it also accumulates sum_dzc[ch] += sum(dz * c).
void relu6_mask_reduce(const void* g1, const void* g2, const void* y, void* dz, float* sum, const void* c, float* sum_dzc,
                       int64_t M, int C, bool relu6, cudaStream_t s);
void dw_dgrad(const void* dz, const float* w, const float* scale, void* dx, int N, int H, int W, int C, int stride,
              cudaStream_t s);
void dw_wgrad(const void* dz, const void* x, float* G, int N, int H, int W, int C, int stride, cudaStream_t s);
void mbv2_stem_wgrad(const uint8_t* x, const void* dz, float* G, int N, int H, int W, int ldc, float mul, float add,
                     cudaStream_t s);
// finalize table row (int64): c_real, count, cstride, jstride, w_is_bf16, G off, W off, dgamma off, dbeta off (offsets
// into the flat buffers), then device pointers scale, invstd, mean, sum_dz
constexpr int kFtFinalizeFields = 13;
void mbv2_ft_finalize(const float* params, const void* w16, float* grads, const int64_t* table, int layers, cudaStream_t s);
// refresh table row (int64): c_real, cp, cin_p (0: no dgrad filter), gamma off, beta off, W off (flat params), then
// device pointers invstd, mean, scale, shift, wd (bf16 [cin_p, cp] or 0)
constexpr int kFtRefreshFields = 11;
void mbv2_ft_refresh(const float* params, const int64_t* table, int layers, cudaStream_t s);

// Random augmentation of the uint8 NHWC training batch (csrc/augment.cu).  params: int32 [N, 8] per image =
// Q16.16 a00 a01 b0 a10 a11 b1, flip bits, 0;  rot_table: int32 [2^kAugRotBits][2] Q16.16 (cos, sin);  step: one int32 in
// device memory;  zq / txq / tyq: Q16.16 zoom half-range and translation half-ranges in pixels.  H, W <= kAugMaxSide keeps
// every source coordinate inside int32.
constexpr int kAugParamFields = 8;
constexpr int kAugRotBits = 12;
constexpr int kAugMaxSide = 2048;
constexpr int kAugWarpMaxBlocks = 132 * 8;   // upper bound of the warp's grid (it launches one wave of resident blocks)
void augment_params(int32_t* params, const int32_t* step, const int32_t* rot_table, int N, int H, int W, uint32_t key,
                    int flip_mode, int32_t zq, int32_t txq, int32_t tyq, cudaStream_t s);
void augment_warp(const uint8_t* x, uint8_t* out, const int32_t* params, int N, int H, int W, bool reflect, int fill,
                  cudaStream_t s);
// MixUp / CutMix on top of the geometric warp.  mix: int32 [N, 8] per image = partner, MixUp own weight w (0..256),
// CutMix box x0 y0 x1 y1 (half-open), then the partner's label weight mu = num / den;  lam_table: int32
// [2^kAugLamBits][2] = Q16 lambda and Q16 sqrt(1 - lambda) at the Beta(alpha, alpha) quantiles (i + 0.5) / 2^kAugLamBits.
constexpr int kAugMixFields = 8;
constexpr int kAugLamBits = 12;
enum AugMix : int { kMixNone = 0, kMixUp = 1, kCutMix = 2 };
void augment_mix_params(int32_t* params, int32_t* mix, const int32_t* step, const int32_t* rot_table,
                        const int32_t* lam_table, int N, int H, int W, uint32_t key, int flip_mode, int32_t zq,
                        int32_t txq, int32_t tyq, int mode, cudaStream_t s);
void augment_mix_warp(const uint8_t* x, uint8_t* out, const int32_t* params, const int32_t* mix, int N, int H, int W,
                      int mode, bool reflect, int fill, cudaStream_t s);
// Color augmentation on top of the warp (or of the raw batch), in place or not: brightness, contrast, saturation, hue,
// grayscale in that order, in Q8 fixed point.  Half-ranges: bq Q8 levels (<= 255 * 256), cq / sq Q16 (<= 65536),
// hq Q16 sixths of a turn (<= 3 * 65536), pq Q16 grayscale probability (<= 65536); 0 skips the stage.  ckey: the
// color draw key.  cluster: CTAs per image (1, 2, 4 or 8; 0 = chosen from N and the SM count); the bytes do not
// depend on it.  Returns the cluster size launched.
constexpr int kAugColorMaxCluster = 8;
int augment_color(const uint8_t* src, uint8_t* dst, const int32_t* step, int N, int H, int W, uint32_t ckey, int32_t bq,
                  int32_t cq, int32_t sq, int32_t hq, int32_t pq, int cluster, cudaStream_t s);
// softmax_ce_head against the soft target (1 - eps) (lambda [k = y_n] + mu [k = y_partner]) + eps / K; mix may be
// nullptr (mu = 0: label smoothing alone)
void softmax_ce_soft_head(const void* logits16, int ld, const float* bias, const int64_t* labels, const int32_t* mix,
                          float eps, float* logits32, void* dlogits16, float* loss_rows, float* stats, int B, int K,
                          float grad_scale, const float* cw, const float* rw, cudaStream_t s);
// softmax_ce_soft_head's loss at weight alpha plus (1 - alpha) T^2 KL(softmax(t / T) || softmax(s / T)), t = the
// teacher's bf16 logits [B, tld] + tbias; stats = [sum loss, correct, sum soft-target loss, sum T^2 KL]
void softmax_kd_head(const void* logits16, int ld, const float* bias, const void* tlogits16, int tld,
                     const float* tbias, const int64_t* labels, const int32_t* mix, float eps, float alpha, float T,
                     float* logits32, void* dlogits16, float* loss_rows, float* stats, int B, int K, float grad_scale,
                     const float* cw, const float* rw, cudaStream_t s);

}  // namespace b200
