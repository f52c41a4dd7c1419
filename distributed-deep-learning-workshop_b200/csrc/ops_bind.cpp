// pybind layer for the bandwidth-bound kernels and fused optimizers (tensor checks + raw-pointer dispatch).
#include <ATen/cuda/CUDAContext.h>
#include <torch/extension.h>

#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "ops_api.h"

namespace {

using at::Tensor;
using OptT = c10::optional<at::Tensor>;

int64_t g_launches = 0;  // number of kernels of ours launched through this module (bench.py reports it)

inline cudaStream_t cur() { return at::cuda::getCurrentCUDAStream(); }
inline void chk(const Tensor& t, at::ScalarType ty, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be CUDA");
  TORCH_CHECK(t.scalar_type() == ty, name, " has wrong dtype");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}
// The kernels move 16 bytes (8 bf16 / 4 fp32) per access, or 8 bytes for the uint8 argmax / bf16x4 stores.
// Check messages are strings only: formatting an integer into a TORCH_CHECK message crashes this extension when
// its libstdc++ differs from the one torch was built with.
inline void aligned(const Tensor& t, int bytes, const char* name) {
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % bytes == 0, name,
              " is not aligned for the kernel's vector accesses");
}
// contiguous CUDA tensor of dtype `ty` with n elements, `align`-byte aligned (1: the kernel reads it element-wise)
inline void vec(const Tensor& t, at::ScalarType ty, int64_t n, const char* name, int align = 16) {
  chk(t, ty, name);
  TORCH_CHECK(t.numel() == n, name, " has the wrong number of elements");
  aligned(t, align, name);
}
// bf16 NHWC / [M, C] activation: C % 8 == 0 and 16-byte aligned
inline int act_channels(const Tensor& t, const char* name) {
  chk(t, at::kBFloat16, name);
  TORCH_CHECK(t.dim() >= 1 && t.size(-1) % 8 == 0 && t.size(-1) > 0, name, ": channel count must be a positive multiple of 8");
  aligned(t, 16, name);
  return (int)t.size(-1);
}
inline const float* fp(const OptT& t) { return t.has_value() ? t->data_ptr<float>() : nullptr; }
inline const void* vp(const OptT& t) { return t.has_value() ? t->data_ptr() : nullptr; }
inline void after() {
  ++g_launches;
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void bn_finalize(Tensor sum, Tensor sqsum, double count, Tensor gamma, Tensor beta, Tensor rmean, Tensor rvar,
                 double momentum, double eps, Tensor mean, Tensor invstd, Tensor scale, Tensor shift, bool training) {
  const int C = (int)gamma.numel();
  for (auto* t : {&sum, &sqsum, &gamma, &beta, &rmean, &rvar, &mean, &invstd, &scale, &shift}) chk(*t, at::kFloat, "bn tensor");
  b200::bn_finalize(sum.data_ptr<float>(), sqsum.data_ptr<float>(), count, gamma.data_ptr<float>(),
                    beta.data_ptr<float>(), rmean.data_ptr<float>(), rvar.data_ptr<float>(), (float)momentum,
                    (float)eps, mean.data_ptr<float>(), invstd.data_ptr<float>(), scale.data_ptr<float>(),
                    shift.data_ptr<float>(), C, training, cur());
  after();
}

// a bf16 tensor with the same element count as the activation `like`, 16-byte aligned
inline void same_act(const Tensor& t, const Tensor& like, const char* name) {
  chk(t, at::kBFloat16, name);
  TORCH_CHECK(t.numel() == like.numel(), name, " must have as many elements as the activation");
  aligned(t, 16, name);
}

// relu6: cap the ReLU at 6 (needs relu; no ReLU bitmask, no BatchNorm on the residual)
void bn_apply(Tensor y, Tensor scale, Tensor shift, OptT res, OptT res_scale, OptT res_shift, Tensor out, bool relu,
              OptT mask, bool relu6) {
  TORCH_CHECK(!relu6 || (relu && !mask.has_value() && !res_scale.has_value()),
              "relu6 caps the ReLU: it needs relu=True, and takes no mask and no res_scale / res_shift");
  const int C = act_channels(y, "y");
  const int64_t M = y.numel() / C;
  same_act(out, y, "out");
  vec(scale, at::kFloat, C, "scale");
  vec(shift, at::kFloat, C, "shift");
  if (res.has_value()) same_act(*res, y, "res");
  TORCH_CHECK(res_scale.has_value() == res_shift.has_value() && (!res_scale.has_value() || res.has_value()),
              "res_scale and res_shift go together, and need res");
  if (res_scale.has_value()) { vec(*res_scale, at::kFloat, C, "res_scale"); vec(*res_shift, at::kFloat, C, "res_shift"); }
  if (mask.has_value()) { chk(*mask, at::kByte, "mask"); TORCH_CHECK(mask->numel() * 8 == y.numel()); }
  b200::bn_apply(y.data_ptr(), scale.data_ptr<float>(), shift.data_ptr<float>(), vp(res), fp(res_scale),
                 fp(res_shift), out.data_ptr(), mask.has_value() ? mask->data_ptr() : nullptr, M, C,
                 relu6 ? 2 : (relu ? 1 : 0), cur());
  after();
}

void channel_stats(Tensor y, Tensor sum, Tensor sqsum) {
  const int C = act_channels(y, "y");
  TORCH_CHECK(C <= 2048, "channel_stats: at most 2048 channels");
  vec(sum, at::kFloat, C, "sum", 1);
  vec(sqsum, at::kFloat, C, "sqsum", 1);
  b200::channel_stats(y.data_ptr(), sum.data_ptr<float>(), sqsum.data_ptr<float>(), y.numel() / C, C, cur());
  after();
}

// mode: 1 = ReLU mask from `outp` (g2 / dz_out optional), 2 = mask from y*scale+shift, 3 = no mask
void bn_bwd_reduce(int64_t mode, Tensor g1, OptT g2, OptT outp, Tensor y, OptT scale, OptT shift, OptT dz_out,
                   Tensor sum_dz, Tensor sum_dzy) {
  const int C = act_channels(y, "y");
  TORCH_CHECK(C <= 2048, "bn_bwd_reduce: at most 2048 channels");
  same_act(g1, y, "g1");
  TORCH_CHECK(mode >= 1 && mode <= 4);
  TORCH_CHECK((mode != 1 && mode != 4) || outp.has_value(), "modes 1/4 need the activation output / bitmask");
  TORCH_CHECK(mode != 2 || (scale.has_value() && shift.has_value()), "mode 2 needs scale/shift");
  // operands a mode does not read must be absent, so that a call never silently ignores one
  TORCH_CHECK(mode == 1 || mode == 4 || (!g2.has_value() && !outp.has_value() && !dz_out.has_value()),
              "g2 / outp / dz_out are used by modes 1 and 4 only");
  TORCH_CHECK(mode == 2 || (!scale.has_value() && !shift.has_value()), "scale / shift are used by mode 2 only");
  if (g2.has_value()) same_act(*g2, y, "g2");
  if (dz_out.has_value()) same_act(*dz_out, y, "dz_out");
  if (mode == 1) same_act(*outp, y, "outp");
  if (mode == 4) vec(*outp, at::kByte, y.numel() / 8, "outp (bitmask)", 1);
  if (mode == 2) { vec(*scale, at::kFloat, C, "scale"); vec(*shift, at::kFloat, C, "shift"); }
  vec(sum_dz, at::kFloat, C, "sum_dz", 1);
  vec(sum_dzy, at::kFloat, C, "sum_dzy", 1);
  b200::bn_bwd_reduce((int)mode, g1.data_ptr(), vp(g2), vp(outp), y.data_ptr(), fp(scale), fp(shift),
                      dz_out.has_value() ? dz_out->data_ptr() : nullptr, sum_dz.data_ptr<float>(),
                      sum_dzy.data_ptr<float>(), y.numel() / C, C, cur());
  after();
}

// inference: the BatchNorm normalised with its running statistics (mean / invstd): B = C = 0, dy = A * dz
void bn_bwd_coeffs(Tensor sum_dz, Tensor sum_dzy, Tensor gamma, Tensor mean, Tensor invstd, double count,
                   Tensor dgamma, Tensor dbeta, Tensor cA, Tensor cB, Tensor cC, bool inference) {
  const int C = (int)gamma.numel();
  for (const auto& [t, name] : {std::pair<const Tensor*, const char*>{&sum_dz, "sum_dz"}, {&sum_dzy, "sum_dzy"},
                                {&gamma, "gamma"}, {&mean, "mean"}, {&invstd, "invstd"}, {&dgamma, "dgamma"},
                                {&dbeta, "dbeta"}, {&cA, "cA"}, {&cB, "cB"}, {&cC, "cC"}})
    vec(*t, at::kFloat, C, name, 1);
  b200::bn_bwd_coeffs(sum_dz.data_ptr<float>(), sum_dzy.data_ptr<float>(), gamma.data_ptr<float>(),
                      mean.data_ptr<float>(), invstd.data_ptr<float>(), count, dgamma.data_ptr<float>(),
                      dbeta.data_ptr<float>(), cA.data_ptr<float>(), cB.data_ptr<float>(), cC.data_ptr<float>(), C,
                      inference, cur());
  after();
}

// dz = g, or g * (y*scale + shift > 0) when scale / shift are given: both or neither, C fp32 values each
static void bn_bwd_apply_operands(const Tensor& g, const Tensor& y, const OptT& scale, const OptT& shift, const Tensor& dy,
                                  int C) {
  same_act(g, y, "g");
  same_act(dy, y, "dy");
  TORCH_CHECK(scale.has_value() == shift.has_value(), "scale and shift go together");
  if (scale.has_value()) { vec(*scale, at::kFloat, C, "scale"); vec(*shift, at::kFloat, C, "shift"); }
}

void bn_bwd_apply(Tensor g, Tensor y, OptT scale, OptT shift, Tensor cA, Tensor cB, Tensor cC, Tensor dy) {
  const int C = act_channels(y, "y");
  bn_bwd_apply_operands(g, y, scale, shift, dy, C);
  vec(cA, at::kFloat, C, "cA");
  vec(cB, at::kFloat, C, "cB");
  vec(cC, at::kFloat, C, "cC");
  b200::bn_bwd_apply(g.data_ptr(), y.data_ptr(), fp(scale), fp(shift), cA.data_ptr<float>(), cB.data_ptr<float>(),
                     cC.data_ptr<float>(), dy.data_ptr(), y.numel() / C, C, cur());
  after();
}

// ---- fused variants: the BatchNorm coefficients are computed inside the consumer kernel (no bn_finalize / bn_bwd_coeffs
// launch on the critical path); the caller zeroes the sum accumulators once per step.
static b200::BnFwdFuse fwd_fuse(const Tensor& sum, const Tensor& sqsum, const Tensor& gamma, const Tensor& beta,
                                const Tensor& rmean, const Tensor& rvar, const Tensor& mean, const Tensor& invstd,
                                const Tensor& scale, const Tensor& shift, double count, double momentum, double eps, int C) {
  for (const Tensor* t : {&sum, &sqsum, &gamma, &beta, &rmean, &rvar, &mean, &invstd, &scale, &shift}) {
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kFloat && t->numel() == C && t->is_contiguous(),
                "fused BN parameter must be a contiguous fp32 CUDA vector of C elements");
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "fused BN parameter must be 16-byte aligned");
  }
  b200::BnFwdFuse f;
  f.sum = sum.data_ptr<float>(); f.sqsum = sqsum.data_ptr<float>();
  f.gamma = gamma.data_ptr<float>(); f.beta = beta.data_ptr<float>();
  f.running_mean = rmean.data_ptr<float>(); f.running_var = rvar.data_ptr<float>();
  f.mean = mean.data_ptr<float>(); f.invstd = invstd.data_ptr<float>();
  f.scale = scale.data_ptr<float>(); f.shift = shift.data_ptr<float>();
  f.inv_count = (float)(1.0 / count);
  f.unbias = count > 1 ? (float)(count / (count - 1.0)) : 1.f;
  f.momentum = (float)momentum;
  f.eps = (float)eps;
  return f;
}

// pack order (main BN and `res_pack`): sum, sqsum, gamma, beta, running_mean, running_var, mean, invstd, scale, shift
void bn_apply_fused(Tensor y, std::vector<Tensor> pack, double count, double momentum, double eps, OptT res,
                    c10::optional<std::vector<Tensor>> res_pack, Tensor out, bool relu, OptT mask) {
  const int C = act_channels(y, "y");
  const int64_t M = y.numel() / C;
  same_act(out, y, "out");
  TORCH_CHECK(pack.size() == 10);
  if (res.has_value()) same_act(*res, y, "res");
  if (mask.has_value()) { chk(*mask, at::kByte, "mask"); TORCH_CHECK(mask->numel() * 8 == y.numel()); }
  TORCH_CHECK(!res_pack.has_value() || res.has_value(), "res_pack needs res");
  b200::BnFwdFuse f = fwd_fuse(pack[0], pack[1], pack[2], pack[3], pack[4], pack[5], pack[6], pack[7], pack[8], pack[9],
                               count, momentum, eps, C);
  b200::BnFwdFuse rf;
  if (res_pack.has_value()) {
    const auto& q = *res_pack;
    TORCH_CHECK(q.size() == 10);
    rf = fwd_fuse(q[0], q[1], q[2], q[3], q[4], q[5], q[6], q[7], q[8], q[9], count, momentum, eps, C);
  }
  b200::bn_apply_fused(y.data_ptr(), f, vp(res), res_pack.has_value() ? &rf : nullptr, out.data_ptr(),
                       mask.has_value() ? mask->data_ptr() : nullptr, M, C, relu, cur());
  after();
}

// dy = A*dz + B*y + C with A, B, C computed in the kernel from sum_dz, sum_dzy; dgamma / dbeta written by the kernel.
void bn_bwd_apply_fused(Tensor g, Tensor y, OptT scale, OptT shift, Tensor sum_dz, Tensor sum_dzy, Tensor gamma,
                        Tensor mean, Tensor invstd, double count, Tensor dgamma, Tensor dbeta, Tensor dy) {
  const int C = act_channels(y, "y");
  bn_bwd_apply_operands(g, y, scale, shift, dy, C);
  for (const Tensor* t : {&sum_dz, &sum_dzy, &gamma, &mean, &invstd, &dgamma, &dbeta}) {
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kFloat && t->numel() == C && t->is_contiguous());
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0, "fused BN parameter must be 16-byte aligned");
  }
  b200::BnBwdFuse f;
  f.sum_dz = sum_dz.data_ptr<float>(); f.sum_dzy = sum_dzy.data_ptr<float>();
  f.gamma = gamma.data_ptr<float>(); f.mean = mean.data_ptr<float>(); f.invstd = invstd.data_ptr<float>();
  f.dgamma = dgamma.data_ptr<float>(); f.dbeta = dbeta.data_ptr<float>();
  f.inv_count = (float)(1.0 / count);
  b200::bn_bwd_apply_fused(g.data_ptr(), y.data_ptr(), fp(scale), fp(shift), f, dy.data_ptr(), y.numel() / C, C, cur());
  after();
}

// 3x3/2 pad-1 max pool: x bf16 NHWC [N, H, W, C], pooled [N, Ho, Wo, C] bf16 and its uint8 argmax of the same shape
static void pool_shapes(const Tensor& x, const Tensor& pooled, const char* pname, const OptT& idx) {
  TORCH_CHECK(x.dim() == 4, "max pool: NHWC input");
  const int C = act_channels(x, "pool input");
  chk(pooled, at::kBFloat16, pname);
  aligned(pooled, 16, pname);
  const int64_t Ho = (x.size(1) - 1) / 2 + 1, Wo = (x.size(2) - 1) / 2 + 1;
  TORCH_CHECK(pooled.dim() == 4 && pooled.size(0) == x.size(0) && pooled.size(1) == Ho && pooled.size(2) == Wo &&
              pooled.size(3) == C, pname, " must be [N, (H+1)/2, (W+1)/2, C]");
  if (idx.has_value()) vec(*idx, at::kByte, pooled.numel(), "idx", 8);
}

void maxpool_fwd(Tensor x, Tensor out, OptT idx) {
  pool_shapes(x, out, "out", idx);
  b200::maxpool_fwd(x.data_ptr(), out.data_ptr(), idx.has_value() ? idx->data_ptr() : nullptr, (int)x.size(0),
                    (int)x.size(1), (int)x.size(2), (int)x.size(3), cur());
  after();
}
void bn_relu_maxpool_fwd(Tensor y, Tensor scale, Tensor shift, Tensor out, OptT idx) {
  pool_shapes(y, out, "out", idx);
  vec(scale, at::kFloat, y.size(3), "scale");
  vec(shift, at::kFloat, y.size(3), "shift");
  b200::bn_relu_maxpool_fwd(y.data_ptr(), scale.data_ptr<float>(), shift.data_ptr<float>(), out.data_ptr(),
                            idx.has_value() ? idx->data_ptr() : nullptr, (int)y.size(0), (int)y.size(1),
                            (int)y.size(2), (int)y.size(3), cur());
  after();
}
void maxpool_bwd(Tensor idx, Tensor g1, OptT g2, Tensor dx) {
  pool_shapes(dx, g1, "g1", idx);
  if (g2.has_value()) same_act(*g2, g1, "g2");
  b200::maxpool_bwd(idx.data_ptr(), g1.data_ptr(), vp(g2), dx.data_ptr(), (int)dx.size(0), (int)dx.size(1),
                    (int)dx.size(2), (int)dx.size(3), cur());
  after();
}
// global average pool: x bf16 [N, ..., C] (HW = the middle extent), pooled bf16 [N, C]
static int gap_shapes(const Tensor& x, const Tensor& pooled, double drop_p) {
  TORCH_CHECK(x.dim() >= 2 && x.size(0) > 0, "global average pool: [N, ..., C] input");
  const int C = act_channels(x, "pool input");
  TORCH_CHECK(x.numel() / x.size(0) / C > 0, "global average pool: empty spatial extent");
  chk(pooled, at::kBFloat16, "pooled");
  aligned(pooled, 16, "pooled");
  TORCH_CHECK(pooled.numel() == x.size(0) * C, "pooled must have N * C elements");
  TORCH_CHECK(drop_p >= 0.0 && drop_p < 1.0, "dropout probability must be in [0, 1)");
  return C;
}

void gap_fwd(Tensor x, Tensor out, double drop_p, int64_t seed) {
  const int N = (int)x.size(0), C = gap_shapes(x, out, drop_p);
  b200::gap_fwd(x.data_ptr(), out.data_ptr(), N, (int)(x.numel() / N / C), C, (float)drop_p, (uint64_t)seed, cur());
  after();
}
void gap_bwd(Tensor dout, Tensor dx, double drop_p, int64_t seed) {
  const int N = (int)dx.size(0), C = gap_shapes(dx, dout, drop_p);
  b200::gap_bwd(dout.data_ptr(), dx.data_ptr(), N, (int)(dx.numel() / N / C), C, (float)drop_p, (uint64_t)seed, cur());
  after();
}
void softmax_ce(Tensor logits, Tensor labels, OptT dlogits, OptT loss_rows, Tensor stats, double grad_scale) {
  chk(logits, at::kFloat, "logits");
  chk(labels, at::kLong, "labels");
  chk(stats, at::kFloat, "stats");
  b200::softmax_ce(logits.data_ptr<float>(), labels.data_ptr<int64_t>(),
                   dlogits.has_value() ? dlogits->data_ptr<float>() : nullptr,
                   loss_rows.has_value() ? loss_rows->data_ptr<float>() : nullptr, stats.data_ptr<float>(),
                   (int)logits.size(0), (int)logits.size(1), (float)grad_scale, cur());
  after();
}
// Optional per-row loss weights of the three heads: class_weight fp32 [K] (read at the row's target class) or
// row_weight fp32 [B], at most one; neither launches the unweighted kernel.
static void head_weights(const OptT& class_weight, const OptT& row_weight, const Tensor& logits16, int64_t B,
                         int64_t K) {
  TORCH_CHECK(!(class_weight.has_value() && row_weight.has_value()), "pass class_weight or row_weight, not both");
  if (class_weight.has_value()) {
    vec(*class_weight, at::kFloat, K, "class_weight", 4);
    TORCH_CHECK(class_weight->device() == logits16.device(), "class_weight must be on the device of logits16");
  }
  if (row_weight.has_value()) {
    vec(*row_weight, at::kFloat, B, "row_weight", 4);
    TORCH_CHECK(row_weight->device() == logits16.device(), "row_weight must be on the device of logits16");
  }
}
// classifier head: bf16 logits [B, ld] (first K columns real) + fp32 bias -> loss / accuracy / bf16 dlogits [B, ld]
void softmax_ce_head(Tensor logits16, Tensor bias, Tensor labels, OptT logits32, OptT dlogits16, OptT loss_rows,
                     Tensor stats, double grad_scale, OptT class_weight, OptT row_weight) {
  chk(logits16, at::kBFloat16, "logits16");
  chk(bias, at::kFloat, "bias");
  chk(labels, at::kLong, "labels");
  chk(stats, at::kFloat, "stats");
  TORCH_CHECK(logits16.dim() == 2 && bias.numel() <= logits16.size(1) && labels.numel() == logits16.size(0));
  const int B = (int)logits16.size(0), ld = (int)logits16.size(1), K = (int)bias.numel();
  head_weights(class_weight, row_weight, logits16, B, K);
  if (logits32.has_value()) { chk(*logits32, at::kFloat, "logits32"); TORCH_CHECK(logits32->numel() == (int64_t)B * K); }
  if (dlogits16.has_value()) { chk(*dlogits16, at::kBFloat16, "dlogits16"); TORCH_CHECK(dlogits16->numel() == logits16.numel()); }
  b200::softmax_ce_head(logits16.data_ptr(), ld, bias.data_ptr<float>(), labels.data_ptr<int64_t>(),
                        logits32.has_value() ? logits32->data_ptr<float>() : nullptr,
                        dlogits16.has_value() ? dlogits16->data_ptr() : nullptr,
                        loss_rows.has_value() ? loss_rows->data_ptr<float>() : nullptr, stats.data_ptr<float>(), B, K,
                        (float)grad_scale, fp(class_weight), fp(row_weight), cur());
  after();
}
// softmax_ce_head against the soft target of label smoothing `eps` and, with `mix` (int32 [B, 8] mix rows of
// augment_mix_params), the partner's label at weight num / den; see csrc/head_stem.cu
void softmax_ce_soft_head(Tensor logits16, Tensor bias, Tensor labels, OptT mix, double eps, OptT logits32,
                          OptT dlogits16, OptT loss_rows, Tensor stats, double grad_scale, OptT class_weight,
                          OptT row_weight) {
  chk(logits16, at::kBFloat16, "logits16");
  chk(bias, at::kFloat, "bias");
  chk(labels, at::kLong, "labels");
  chk(stats, at::kFloat, "stats");
  TORCH_CHECK(logits16.dim() == 2 && logits16.size(0) >= 1 && bias.numel() >= 1 && bias.numel() <= logits16.size(1) &&
                  labels.numel() == logits16.size(0),
              "logits16 must be bf16 [B, ld] with ld >= K = bias.numel() and B = labels.numel() >= 1");
  TORCH_CHECK(stats.numel() >= 2, "stats must hold [sum loss, correct]");
  TORCH_CHECK(eps >= 0.0 && eps <= 1.0, "label smoothing must be in [0, 1]");
  const int B = (int)logits16.size(0), ld = (int)logits16.size(1), K = (int)bias.numel();
  for (const Tensor* t : {&bias, &labels, &stats})
    TORCH_CHECK(t->device() == logits16.device(), "bias, labels and stats must be on the device of logits16");
  head_weights(class_weight, row_weight, logits16, B, K);
  if (mix.has_value()) {
    chk(*mix, at::kInt, "mix");
    TORCH_CHECK(mix->dim() == 2 && mix->size(0) == B && mix->size(1) == b200::kAugMixFields,
                "mix must be int32 [B, 8] for the batch's B rows");
    TORCH_CHECK(mix->device() == logits16.device(), "mix must be on the device of logits16");
    aligned(*mix, 16, "mix");
  }
  if (logits32.has_value()) {
    chk(*logits32, at::kFloat, "logits32");
    TORCH_CHECK(logits32->numel() == (int64_t)B * K, "logits32 must hold B x K values");
  }
  if (dlogits16.has_value()) {
    chk(*dlogits16, at::kBFloat16, "dlogits16");
    TORCH_CHECK(dlogits16->numel() == logits16.numel(), "dlogits16 must have the shape of logits16");
    TORCH_CHECK(dlogits16->data_ptr() != logits16.data_ptr(), "dlogits16 cannot overwrite logits16");
  }
  if (loss_rows.has_value()) {
    chk(*loss_rows, at::kFloat, "loss_rows");
    TORCH_CHECK(loss_rows->numel() == B, "loss_rows must hold B values");
  }
  for (const OptT* t : {&logits32, &dlogits16, &loss_rows})
    if (t->has_value()) TORCH_CHECK((*t)->device() == logits16.device(), "outputs must be on the device of logits16");
  b200::softmax_ce_soft_head(logits16.data_ptr(), ld, bias.data_ptr<float>(), labels.data_ptr<int64_t>(),
                             mix.has_value() ? mix->data_ptr<int32_t>() : nullptr, (float)eps,
                             logits32.has_value() ? logits32->data_ptr<float>() : nullptr,
                             dlogits16.has_value() ? dlogits16->data_ptr() : nullptr,
                             loss_rows.has_value() ? loss_rows->data_ptr<float>() : nullptr, stats.data_ptr<float>(), B,
                             K, (float)grad_scale, fp(class_weight), fp(row_weight), cur());
  after();
}
// softmax_ce_soft_head plus distillation from the teacher's bf16 logits [B, tld] + tbias (tld >= K = bias.numel()) at
// weight 1 - alpha and temperature T; stats: [sum loss, correct, sum student loss, sum distillation loss]
void softmax_kd_head(Tensor logits16, Tensor bias, Tensor tlogits16, Tensor tbias, Tensor labels, OptT mix, double eps,
                     double alpha, double temperature, OptT logits32, OptT dlogits16, OptT loss_rows, Tensor stats,
                     double grad_scale, OptT class_weight, OptT row_weight) {
  chk(logits16, at::kBFloat16, "logits16");
  chk(bias, at::kFloat, "bias");
  chk(tlogits16, at::kBFloat16, "tlogits16");
  chk(tbias, at::kFloat, "tbias");
  chk(labels, at::kLong, "labels");
  chk(stats, at::kFloat, "stats");
  TORCH_CHECK(logits16.dim() == 2 && logits16.size(0) >= 1 && bias.numel() >= 1 && bias.numel() <= logits16.size(1) &&
                  labels.numel() == logits16.size(0),
              "logits16 must be bf16 [B, ld] with ld >= K = bias.numel() and B = labels.numel() >= 1");
  TORCH_CHECK(tlogits16.dim() == 2 && tlogits16.size(0) == logits16.size(0) && tbias.numel() == bias.numel() &&
                  tlogits16.size(1) >= bias.numel(),
              "tlogits16 must be bf16 [B, tld] with tld >= K and tbias must hold K values");
  TORCH_CHECK(stats.numel() >= 4, "stats must hold [sum loss, correct, sum student loss, sum distillation loss]");
  TORCH_CHECK(eps >= 0.0 && eps <= 1.0, "label smoothing must be in [0, 1]");
  TORCH_CHECK(alpha >= 0.0 && alpha <= 1.0, "alpha must be in [0, 1]");
  TORCH_CHECK(temperature > 0.0 && temperature < 1e30, "temperature must be finite and > 0");
  const int B = (int)logits16.size(0), ld = (int)logits16.size(1), tld = (int)tlogits16.size(1), K = (int)bias.numel();
  for (const Tensor* t : {&bias, &tlogits16, &tbias, &labels, &stats})
    TORCH_CHECK(t->device() == logits16.device(), "bias, the teacher's tensors, labels and stats must be on the device "
                "of logits16");
  head_weights(class_weight, row_weight, logits16, B, K);
  if (mix.has_value()) {
    chk(*mix, at::kInt, "mix");
    TORCH_CHECK(mix->dim() == 2 && mix->size(0) == B && mix->size(1) == b200::kAugMixFields,
                "mix must be int32 [B, 8] for the batch's B rows");
    TORCH_CHECK(mix->device() == logits16.device(), "mix must be on the device of logits16");
    aligned(*mix, 16, "mix");
  }
  if (logits32.has_value()) {
    chk(*logits32, at::kFloat, "logits32");
    TORCH_CHECK(logits32->numel() == (int64_t)B * K, "logits32 must hold B x K values");
  }
  if (dlogits16.has_value()) {
    chk(*dlogits16, at::kBFloat16, "dlogits16");
    TORCH_CHECK(dlogits16->numel() == logits16.numel(), "dlogits16 must have the shape of logits16");
    TORCH_CHECK(dlogits16->data_ptr() != logits16.data_ptr() && dlogits16->data_ptr() != tlogits16.data_ptr(),
                "dlogits16 cannot overwrite logits16 or tlogits16");
  }
  if (loss_rows.has_value()) {
    chk(*loss_rows, at::kFloat, "loss_rows");
    TORCH_CHECK(loss_rows->numel() == B, "loss_rows must hold B values");
  }
  for (const OptT* t : {&logits32, &dlogits16, &loss_rows})
    if (t->has_value()) TORCH_CHECK((*t)->device() == logits16.device(), "outputs must be on the device of logits16");
  b200::softmax_kd_head(logits16.data_ptr(), ld, bias.data_ptr<float>(), tlogits16.data_ptr(), tld,
                        tbias.data_ptr<float>(), labels.data_ptr<int64_t>(),
                        mix.has_value() ? mix->data_ptr<int32_t>() : nullptr, (float)eps, (float)alpha,
                        (float)temperature, logits32.has_value() ? logits32->data_ptr<float>() : nullptr,
                        dlogits16.has_value() ? dlogits16->data_ptr() : nullptr,
                        loss_rows.has_value() ? loss_rows->data_ptr<float>() : nullptr, stats.data_ptr<float>(), B, K,
                        (float)grad_scale, fp(class_weight), fp(row_weight), cur());
  after();
}
void fc_bias_grad(Tensor dlogits16, Tensor dbias) {
  chk(dlogits16, at::kBFloat16, "dlogits16");
  chk(dbias, at::kFloat, "dbias");
  TORCH_CHECK(dlogits16.dim() == 2 && dbias.numel() <= dlogits16.size(1));
  b200::fc_bias_grad(dlogits16.data_ptr(), (int)dlogits16.size(1), dbias.data_ptr<float>(), (int)dlogits16.size(0),
                     (int)dbias.numel(), cur());
  after();
}
void pack_stem_weight(Tensor w, Tensor out) {
  chk(w, at::kFloat, "w");
  chk(out, at::kBFloat16, "out");
  TORCH_CHECK(w.numel() == 49 * 64 * 3 && out.numel() == 64 * 192);
  b200::pack_stem_weight(w.data_ptr<float>(), out.data_ptr(), cur());
  after();
}
// max-pool 3x3/2 backward fused with the stem BN+ReLU backward; pass 0 = reduce, pass 1 = apply (see head_stem.cu)
void stem_pool_bn_bwd(int64_t pass, Tensor idx, Tensor g1, OptT g2, Tensor y, Tensor scale, Tensor shift, OptT cA, OptT cB,
                      OptT cC, OptT dy, Tensor sum_dz, Tensor sum_dzy) {
  chk(idx, at::kByte, "idx");
  chk(g1, at::kBFloat16, "g1");
  chk(y, at::kBFloat16, "y");
  chk(scale, at::kFloat, "scale");
  chk(shift, at::kFloat, "shift");
  TORCH_CHECK(y.dim() == 4 && y.size(3) == 64 && g1.dim() == 4 && g1.size(3) == 64, "stem tail: 64 channels, NHWC");
  const int N = (int)g1.size(0), Ho = (int)g1.size(1), Wo = (int)g1.size(2);
  TORCH_CHECK(y.size(0) == N && y.size(1) == 2 * Ho && y.size(2) == 2 * Wo && idx.numel() == g1.numel());
  TORCH_CHECK(Ho % 8 == 0 && Wo % 8 == 0, "stem tail: pooled grid must tile by 8");
  if (g2.has_value()) { chk(*g2, at::kBFloat16, "g2"); TORCH_CHECK(g2->numel() == g1.numel()); }
  TORCH_CHECK(pass == 0 || (cA.has_value() && cB.has_value() && cC.has_value() && dy.has_value()));
  if (dy.has_value()) same_act(*dy, y, "dy");
  aligned(y, 16, "y");
  for (const auto& [t, name] : {std::pair<const OptT, const char*>{scale, "scale"}, {shift, "shift"}, {cA, "cA"}, {cB, "cB"},
                                {cC, "cC"}, {sum_dz, "sum_dz"}, {sum_dzy, "sum_dzy"}})
    if (t.has_value()) vec(*t, at::kFloat, 64, name, 1);
  b200::stem_pool_bn_bwd((int)pass, idx.data_ptr(), g1.data_ptr(), vp(g2), y.data_ptr(), scale.data_ptr<float>(),
                         shift.data_ptr<float>(), fp(cA), fp(cB), fp(cC), dy.has_value() ? dy->data_ptr() : nullptr,
                         sum_dz.data_ptr<float>(), sum_dzy.data_ptr<float>(), N, Ho, Wo, cur());
  after();
}
// cudaMemsetAsync on the current stream (a memset node under graph capture, not a kernel)
void zero_(Tensor t) {
  TORCH_CHECK(t.is_cuda() && t.is_contiguous());
  C10_CUDA_CHECK(cudaMemsetAsync(t.data_ptr(), 0, t.numel() * t.element_size(), cur()));
}
// MobileNetV2 stem: uint8 [N,H,W,3] -> bf16 [N,H/2,W/2,ldc] (32 real channels), relu6(conv3x3/2(x*mul+add) * scale + shift)
void mbv2_stem(Tensor x, Tensor w, Tensor scale, Tensor shift, Tensor out, double mul, double add) {
  chk(x, at::kByte, "x");
  chk(w, at::kFloat, "w");
  chk(scale, at::kFloat, "scale");
  chk(shift, at::kFloat, "shift");
  chk(out, at::kBFloat16, "out");
  TORCH_CHECK(x.dim() == 4 && x.size(3) == 3 && x.size(1) % 2 == 0 && x.size(2) % 2 == 0, "stem input: uint8 [N, H, W, 3], even H / W");
  TORCH_CHECK(w.numel() == 27 * 32 && scale.numel() >= 32 && shift.numel() >= 32);
  TORCH_CHECK(out.dim() == 4 && out.size(0) == x.size(0) && out.size(1) == x.size(1) / 2 && out.size(2) == x.size(2) / 2 &&
              out.size(3) >= 32 && out.size(3) % 8 == 0);
  aligned(out, 16, "out");
  b200::mbv2_stem(x.data_ptr<uint8_t>(), w.data_ptr<float>(), scale.data_ptr<float>(), shift.data_ptr<float>(), out.data_ptr(),
                  (int)x.size(0), (int)x.size(1), (int)x.size(2), (int)out.size(3), (float)mul, (float)add, cur());
  after();
}
// depthwise 3x3 (pad 1, stride 1 / 2) + folded BatchNorm + ReLU6;  x bf16 [N,H,W,C], w fp32 [9, C], out bf16 [N,Ho,Wo,C]
void dwconv3x3(Tensor x, Tensor w, Tensor scale, Tensor shift, Tensor out, int64_t stride, int64_t tile_w) {
  chk(x, at::kBFloat16, "x");
  chk(w, at::kFloat, "w");
  chk(scale, at::kFloat, "scale");
  chk(shift, at::kFloat, "shift");
  chk(out, at::kBFloat16, "out");
  TORCH_CHECK((stride == 1 || stride == 2) && (tile_w == 1 || tile_w == 4));
  const int C = (int)x.size(3), H = (int)x.size(1), W = (int)x.size(2);
  TORCH_CHECK(x.dim() == 4 && C % 8 == 0 && w.numel() == 9 * C && scale.numel() == C && shift.numel() == C);
  TORCH_CHECK(out.dim() == 4 && out.size(0) == x.size(0) && out.size(3) == C && out.size(1) == (H - 1) / stride + 1 &&
              out.size(2) == (W - 1) / stride + 1, "dwconv3x3 output shape");
  for (const Tensor* t : {&x, &w, &scale, &shift, &out}) aligned(*t, 16, "dwconv3x3 operand");
  b200::dwconv3x3(x.data_ptr(), w.data_ptr<float>(), scale.data_ptr<float>(), shift.data_ptr<float>(), out.data_ptr(),
                  (int)x.size(0), H, W, C, (int)stride, (int)tile_w, cur());
  after();
}
// NHWC bf16 pair of a depthwise 3x3 (pad 1) layer: input grid x, output grid (H-1)/stride+1; returns C
static int dw_pair(const Tensor& x, const Tensor& dz, int64_t stride, const char* xname) {
  TORCH_CHECK(stride == 1 || stride == 2, "stride must be 1 or 2");
  TORCH_CHECK(x.dim() == 4 && dz.dim() == 4, "depthwise operands are NHWC");
  const int C = act_channels(x, xname);
  act_channels(dz, "dz");
  TORCH_CHECK(dz.size(0) == x.size(0) && dz.size(3) == C && dz.size(1) == (x.size(1) - 1) / stride + 1 &&
              dz.size(2) == (x.size(2) - 1) / stride + 1, "dz shape does not match the input grid and stride");
  return C;
}
// training-mode BatchNorm variants: c = conv (bf16, no affine / clamp) and sum / sqsum += per-channel sum(c), sum(c^2)
// of the stored values (zeroed by the caller)
void mbv2_stem_stats(Tensor x, Tensor w, Tensor out, Tensor sum, Tensor sqsum, double mul, double add) {
  chk(x, at::kByte, "x");
  TORCH_CHECK(x.dim() == 4 && x.size(3) == 3 && x.size(1) % 2 == 0 && x.size(2) % 2 == 0,
              "stem input: uint8 [N, H, W, 3], even H / W");
  vec(w, at::kFloat, 27 * 32, "w", 4);
  const int ldc = act_channels(out, "out");
  TORCH_CHECK(out.dim() == 4 && out.size(0) == x.size(0) && out.size(1) == x.size(1) / 2 && out.size(2) == x.size(2) / 2 &&
              ldc >= 32, "out: bf16 [N, H/2, W/2, ldc >= 32]");
  vec(sum, at::kFloat, 32, "sum", 1);
  vec(sqsum, at::kFloat, 32, "sqsum", 1);
  b200::mbv2_stem_stats(x.data_ptr<uint8_t>(), w.data_ptr<float>(), out.data_ptr(), sum.data_ptr<float>(),
                        sqsum.data_ptr<float>(), (int)x.size(0), (int)x.size(1), (int)x.size(2), ldc, (float)mul,
                        (float)add, cur());
  after();
}
void dwconv3x3_stats(Tensor x, Tensor w, Tensor out, Tensor sum, Tensor sqsum, int64_t stride, int64_t tile_w) {
  TORCH_CHECK(tile_w == 1 || tile_w == 4, "tile_w must be 1 or 4");
  const int C = dw_pair(x, out, stride, "x");
  vec(w, at::kFloat, 9 * (int64_t)C, "w");
  vec(sum, at::kFloat, C, "sum", 1);
  vec(sqsum, at::kFloat, C, "sqsum", 1);
  b200::dwconv3x3_stats(x.data_ptr(), w.data_ptr<float>(), out.data_ptr(), sum.data_ptr<float>(), sqsum.data_ptr<float>(),
                        (int)x.size(0), (int)x.size(1), (int)x.size(2), C, (int)stride, (int)tile_w, cur());
  after();
}
void preprocess_u8(Tensor x, Tensor out, double mul, double add) {
  chk(x, at::kByte, "x");
  chk(out, at::kBFloat16, "out");
  TORCH_CHECK(x.size(-1) == 3);
  b200::preprocess_u8(x.data_ptr<uint8_t>(), out.data_ptr(), x.numel() / 3, (int)out.size(-1), (float)mul, (float)add, cur());
  after();
}
// x: uint8 [N, H, W, 3] (planar = false) or [N, 3, H, W] (planar = true, the nvJPEG layout);  out: uint8 [N, OH, OW, 3]
void resize_bilinear_u8(Tensor x, Tensor out, bool planar) {
  chk(x, at::kByte, "x");
  chk(out, at::kByte, "out");
  TORCH_CHECK(x.dim() == 4 && out.dim() == 4 && out.size(3) == 3 && x.size(0) == out.size(0));
  TORCH_CHECK(planar ? x.size(1) == 3 : x.size(3) == 3, "resize_bilinear_u8: 3-channel images");
  const int H = (int)(planar ? x.size(2) : x.size(1)), W = (int)(planar ? x.size(3) : x.size(2));
  b200::resize_bilinear_u8(x.data_ptr<uint8_t>(), out.data_ptr<uint8_t>(), (int)x.size(0), H, W, (int)out.size(1),
                           (int)out.size(2), planar, cur());
  after();
}
void weight_prep(Tensor w, OptT wf, OptT wd, int64_t taps, int64_t cout, int64_t cin) {
  chk(w, at::kFloat, "w");
  TORCH_CHECK(w.numel() == taps * cout * cin);
  if (wf.has_value()) vec(*wf, at::kBFloat16, w.numel(), "wf", 1);
  if (wd.has_value()) vec(*wd, at::kBFloat16, w.numel(), "wd", 1);
  b200::weight_prep(w.data_ptr<float>(), wf.has_value() ? wf->data_ptr() : nullptr,
                    wd.has_value() ? wd->data_ptr() : nullptr, (int)taps, (int)cout, (int)cin, cur());
  after();
}
// table: int64 [layers, 6] on the device = (src_off, dst_off, taps, cout, cin, first_tile_index); a tile = 64 co x 32 ci
void weight_prep_batched(Tensor params, Tensor wd, Tensor table, int64_t total) {
  chk(params, at::kFloat, "params");
  chk(wd, at::kBFloat16, "wd");
  chk(table, at::kLong, "table");
  TORCH_CHECK(table.dim() == 2 && table.size(1) == 6 && table.size(0) <= 128);
  b200::weight_prep_batched(params.data_ptr<float>(), wd.data_ptr(), table.data_ptr<int64_t>(), (int)table.size(0),
                            total, cur());
  after();
}
// One elementwise optimizer update (csrc/optim_rules.cuh): rule name -> kernel instantiation; `state` holds the rule's
// state buffers in its order.  Flat fp32 buffers are read as float4, the bf16 working copy written 8 bytes at a time.
const std::pair<const char*, b200::OptimRule> kOptimRules[] = {
    {"sgd", b200::kRuleSgd},
    {"sgd_nesterov", b200::kRuleSgdNesterov},
    {"adam", b200::kRuleAdam},
    {"adamw", b200::kRuleAdamW},
    {"adadelta", b200::kRuleAdadelta},
    {"rmsprop", b200::kRuleRmsprop},
    {"rmsprop_momentum", b200::kRuleRmspropMomentum},
    {"rmsprop_centered", b200::kRuleRmspropCentered},
    {"rmsprop_centered_momentum", b200::kRuleRmspropCenteredMomentum},
    {"adagrad", b200::kRuleAdagrad},
    {"adamax", b200::kRuleAdamax},
};
void optim_step(const std::string& rule, Tensor p, Tensor g, std::vector<Tensor> state, OptT p16, Tensor hyper) {
  const auto* it = std::find_if(std::begin(kOptimRules), std::end(kOptimRules),
                                [&](const auto& r) { return rule == r.first; });
  TORCH_CHECK(it != std::end(kOptimRules), "optim_step: unknown rule");
  TORCH_CHECK((int64_t)state.size() == b200::optim_rule_states(it->second),
              "optim_step: the state list does not hold the rule's state buffers");
  chk(p, at::kFloat, "p");
  TORCH_CHECK(p.numel() % 4 == 0, "p: element count must be a multiple of 4");
  aligned(p, 16, "p");
  vec(g, at::kFloat, p.numel(), "g");
  std::vector<float*> sp;
  for (const Tensor& t : state) {
    vec(t, at::kFloat, p.numel(), "state");
    sp.push_back(t.data_ptr<float>());
  }
  if (p16.has_value()) vec(*p16, at::kBFloat16, p.numel(), "p16", 8);
  vec(hyper, at::kFloat, hyper.numel(), "hyper", 1);
  TORCH_CHECK(hyper.numel() >= b200::kHyperLen, "hyper must hold 8 values");
  b200::optim_step(it->second, p.data_ptr<float>(), g.data_ptr<float>(), sp.data(),
                   p16.has_value() ? p16->data_ptr() : nullptr, p.numel(), hyper.data_ptr<float>(), cur());
  after();
}

// ---- chunked clip / LAMB passes: flat buffer x (fp32, n % 4 == 0, 16-byte aligned), chunk table, 16-slot hyper array
static int64_t chunk_operands(const Tensor& x, const Tensor& chunks, const Tensor& hyper) {
  chk(x, at::kFloat, "flat buffer");
  TORCH_CHECK(x.numel() % 4 == 0, "flat buffer: element count must be a multiple of 4");
  aligned(x, 16, "flat buffer");
  chk(chunks, at::kLong, "chunks");
  TORCH_CHECK(chunks.dim() == 2 && chunks.size(1) == b200::kChunkFields && chunks.size(0) >= 1 &&
              chunks.size(0) < (int64_t(1) << 31), "chunks: int64 [nchunks (1 .. 2^31 - 1), 3] = (lo, hi, segment)");
  vec(hyper, at::kFloat, hyper.numel(), "hyper", 4);
  TORCH_CHECK(hyper.numel() >= b200::kHyperSlots, "hyper must hold 16 values for the clip and LAMB passes");
  TORCH_CHECK(chunks.device() == x.device() && hyper.device() == x.device(),
              "chunks and hyper must be on the device of the flat buffer");
  return chunks.size(0);
}
static void partial_operand(const Tensor& partial, int64_t rows, int64_t nchunks, const Tensor& like) {
  vec(partial, at::kFloat, rows * nchunks, "partial", 4);
  TORCH_CHECK(partial.dim() == (rows == 1 ? 1 : 2), "partial: fp32 [nchunks], or [2, nchunks] for LAMB");
  TORCH_CHECK(partial.device() == like.device(), "partial must be on the device of the flat buffer");
}
void segment_sumsq(Tensor g, Tensor chunks, Tensor partial, Tensor hyper) {
  const int64_t nc = chunk_operands(g, chunks, hyper);
  partial_operand(partial, 1, nc, g);
  b200::segment_sumsq(g.data_ptr<float>(), g.numel(), chunks.data_ptr<int64_t>(), nc, partial.data_ptr<float>(),
                      hyper.data_ptr<float>(), cur());
  after();
}
void segment_finalize(Tensor partial, Tensor segs, Tensor sums, Tensor factor, Tensor hyper, int64_t mode) {
  TORCH_CHECK(mode >= b200::kFinSums && mode <= b200::kFinLamb, "mode: 0 sums, 1 global clip, 2 per-segment clip, 3 LAMB");
  const int64_t rows = mode == b200::kFinLamb ? 2 : 1;
  TORCH_CHECK(partial.dim() == (rows == 1 ? 1 : 2) && (rows == 1 || partial.size(0) == 2),
              "partial: fp32 [nchunks], or [2, nchunks] for LAMB");
  const int64_t nc = partial.size(-1);
  partial_operand(partial, rows, nc, partial);
  chk(segs, at::kLong, "segs");
  TORCH_CHECK(segs.dim() == 2 && segs.size(1) == 2 && segs.size(0) >= 1 && segs.size(0) <= b200::kMaxSegments,
              "segs: int64 [nseg (1 .. 2^20), 2] = (first chunk, end chunk)");
  const int64_t ns = segs.size(0);
  vec(sums, at::kFloat, 2 * (ns + 1), "sums", 4);
  vec(factor, at::kFloat, ns, "factor", 4);
  vec(hyper, at::kFloat, hyper.numel(), "hyper", 4);
  TORCH_CHECK(hyper.numel() >= b200::kHyperSlots, "hyper must hold 16 values for the clip and LAMB passes");
  for (const Tensor* t : {&segs, &sums, &factor, &hyper})
    TORCH_CHECK(t->device() == partial.device(), "segs, sums, factor and hyper must be on the device of partial");
  b200::segment_finalize(partial.data_ptr<float>(), nc, segs.data_ptr<int64_t>(), (int)ns, sums.data_ptr<float>(),
                         factor.data_ptr<float>(), hyper.data_ptr<float>(), (int)mode, cur());
  after();
}
void clip_apply(Tensor g, Tensor chunks, OptT factor, Tensor hyper) {
  const int64_t nc = chunk_operands(g, chunks, hyper);
  if (factor.has_value()) {
    chk(*factor, at::kFloat, "factor");
    TORCH_CHECK(factor->dim() == 1 && factor->numel() >= 1 && factor->numel() <= b200::kMaxSegments &&
                factor->device() == g.device(),
                "factor: fp32 [nseg] on the device of g");
  }
  b200::clip_apply(g.data_ptr<float>(), g.numel(), chunks.data_ptr<int64_t>(), nc, fp(factor),
                   factor.has_value() ? (int)factor->numel() : 0, hyper.data_ptr<float>(), cur());
  after();
}
void lamb_moments(Tensor p, Tensor g, Tensor m, Tensor v, Tensor chunks, Tensor partial, Tensor hyper) {
  const int64_t nc = chunk_operands(p, chunks, hyper);
  for (const auto& [t, name] : {std::pair<const Tensor*, const char*>{&g, "g"}, {&m, "m"}, {&v, "v"}}) {
    vec(*t, at::kFloat, p.numel(), name);
    TORCH_CHECK(t->device() == p.device(), name, " must be on the device of p");
  }
  partial_operand(partial, 2, nc, p);
  b200::lamb_moments(p.data_ptr<float>(), g.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), p.numel(),
                     chunks.data_ptr<int64_t>(), nc, partial.data_ptr<float>(), hyper.data_ptr<float>(), cur());
  after();
}
void lamb_apply(Tensor p, Tensor m, Tensor v, OptT p16, Tensor chunks, Tensor phi, Tensor hyper) {
  const int64_t nc = chunk_operands(p, chunks, hyper);
  for (const auto& [t, name] : {std::pair<const Tensor*, const char*>{&m, "m"}, {&v, "v"}}) {
    vec(*t, at::kFloat, p.numel(), name);
    TORCH_CHECK(t->device() == p.device(), name, " must be on the device of p");
  }
  if (p16.has_value()) vec(*p16, at::kBFloat16, p.numel(), "p16", 8);
  chk(phi, at::kFloat, "phi");
  TORCH_CHECK(phi.dim() == 1 && phi.numel() >= 1 && phi.numel() <= b200::kMaxSegments && phi.device() == p.device(),
              "phi: fp32 [nseg] on the device of p");
  b200::lamb_apply(p.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                   p16.has_value() ? p16->data_ptr() : nullptr, p.numel(), chunks.data_ptr<int64_t>(), nc,
                   phi.data_ptr<float>(), (int)phi.numel(), hyper.data_ptr<float>(), cur());
  after();
}
// ---- gradient accumulation and weight EMA: flat fp32 buffers of one size on one device, none overlapping another
static void disjoint(std::initializer_list<std::pair<const Tensor*, const char*>> ts) {
  for (auto a = ts.begin(); a != ts.end(); ++a)
    for (auto b = a + 1; b != ts.end(); ++b) {
      const auto lo_a = reinterpret_cast<uintptr_t>(a->first->data_ptr()), lo_b = reinterpret_cast<uintptr_t>(b->first->data_ptr());
      const auto hi_a = lo_a + a->first->nbytes(), hi_b = lo_b + b->first->nbytes();
      TORCH_CHECK(hi_a <= lo_b || hi_b <= lo_a, a->second, " and ", b->second, " must not overlap");
    }
}
void grad_accumulate(Tensor g, Tensor accum, int64_t steps, int64_t mode) {
  TORCH_CHECK(mode == 0 || mode == 1, "grad_accumulate: mode 0 (accum += g) or 1 (g = (accum + g) / steps, accum = 0)");
  TORCH_CHECK(steps >= 1 && steps < (int64_t(1) << 24), "grad_accumulate: steps must be in [1, 2^24)");
  chk(g, at::kFloat, "g");
  TORCH_CHECK(g.numel() % 4 == 0, "g: element count must be a multiple of 4");
  aligned(g, 16, "g");
  vec(accum, at::kFloat, g.numel(), "accum");
  TORCH_CHECK(accum.device() == g.device(), "accum must be on the device of g");
  disjoint({{&g, "g"}, {&accum, "accum"}});
  b200::grad_accumulate(g.data_ptr<float>(), accum.data_ptr<float>(), g.numel(), (int)steps, mode == 1, cur());
  after();
}
void ema_update(Tensor p, Tensor ema, OptT p16, Tensor hyper) {
  chk(p, at::kFloat, "p");
  TORCH_CHECK(p.numel() % 4 == 0, "p: element count must be a multiple of 4");
  aligned(p, 16, "p");
  vec(ema, at::kFloat, p.numel(), "ema");
  vec(hyper, at::kFloat, hyper.numel(), "hyper", 4);
  TORCH_CHECK(hyper.numel() >= b200::kHyperSlots, "hyper must hold 16 values for the EMA pass");
  TORCH_CHECK(ema.device() == p.device() && hyper.device() == p.device(), "ema and hyper must be on the device of p");
  if (p16.has_value()) {
    vec(*p16, at::kBFloat16, p.numel(), "p16", 8);
    TORCH_CHECK(p16->device() == p.device(), "p16 must be on the device of p");
    disjoint({{&p, "p"}, {&ema, "ema"}, {&*p16, "p16"}, {&hyper, "hyper"}});
  } else {
    disjoint({{&p, "p"}, {&ema, "ema"}, {&hyper, "hyper"}});
  }
  b200::ema_update(p.data_ptr<float>(), ema.data_ptr<float>(), p16.has_value() ? p16->data_ptr() : nullptr, p.numel(),
                   hyper.data_ptr<float>(), cur());
  after();
}
void cast_bf16(Tensor x, Tensor out) {
  chk(x, at::kFloat, "x");
  TORCH_CHECK(x.numel() % 4 == 0, "x: element count must be a multiple of 4");
  aligned(x, 16, "x");
  vec(out, at::kBFloat16, x.numel(), "out", 8);
  b200::cast_f32_to_bf16(x.data_ptr<float>(), out.data_ptr(), x.numel(), cur());
  after();
}

// ------------------------------------------------------------------------------------------------ MobileNetV2 fine-tuning
// dz = g1 [+ g2], masked by 0 < y < 6 when relu6; sum[c] += sum_rows dz (sum must be zeroed by the caller).  dz may be g1.
// With c (bf16, y's shape; training-mode BatchNorm) also sum_dzc[ch] += sum_rows dz * c; c and sum_dzc go together.
void relu6_mask_reduce(Tensor g1, OptT g2, Tensor y, Tensor dz, Tensor sum, bool relu6, OptT c, OptT sum_dzc) {
  const int C = act_channels(y, "y");
  same_act(g1, y, "g1");
  same_act(dz, y, "dz");
  if (g2.has_value()) same_act(*g2, y, "g2");
  vec(sum, at::kFloat, C, "sum", 1);
  TORCH_CHECK(c.has_value() == sum_dzc.has_value(), "c and sum_dzc go together");
  if (c.has_value()) {
    same_act(*c, y, "c");
    vec(*sum_dzc, at::kFloat, C, "sum_dzc", 1);
    TORCH_CHECK(c->data_ptr() != dz.data_ptr(), "dz must not overwrite c");
  }
  b200::relu6_mask_reduce(g1.data_ptr(), vp(g2), y.data_ptr(), dz.data_ptr(), sum.data_ptr<float>(), vp(c),
                          sum_dzc.has_value() ? sum_dzc->data_ptr<float>() : nullptr, y.numel() / C, C, relu6, cur());
  after();
}
// dx = conv_transpose(dz, scale (.) w) of a depthwise 3x3;  w fp32 [9, C], scale fp32 [C]
void dw_dgrad(Tensor dz, Tensor w, Tensor scale, Tensor dx, int64_t stride) {
  const int C = dw_pair(dx, dz, stride, "dx");
  vec(w, at::kFloat, 9 * (int64_t)C, "w");
  vec(scale, at::kFloat, C, "scale");
  b200::dw_dgrad(dz.data_ptr(), w.data_ptr<float>(), scale.data_ptr<float>(), dx.data_ptr(), (int)dx.size(0),
                 (int)dx.size(1), (int)dx.size(2), C, (int)stride, cur());
  after();
}
// G[9, C] += depthwise 3x3 weight gradient of dz over input x (G zeroed by the caller)
void dw_wgrad(Tensor dz, Tensor x, Tensor G, int64_t stride) {
  const int C = dw_pair(x, dz, stride, "x");
  vec(G, at::kFloat, 9 * (int64_t)C, "G", 4);
  b200::dw_wgrad(dz.data_ptr(), x.data_ptr(), G.data_ptr<float>(), (int)x.size(0), (int)x.size(1), (int)x.size(2), C,
                 (int)stride, cur());
  after();
}
// G[27, 32] += weight gradient of the 3x3/2 stem (mbv2_stem) from the uint8 batch and dz bf16 [N, H/2, W/2, ldc]
void mbv2_stem_wgrad(Tensor x, Tensor dz, Tensor G, double mul, double add) {
  chk(x, at::kByte, "x");
  TORCH_CHECK(x.dim() == 4 && x.size(3) == 3 && x.size(1) % 2 == 0 && x.size(2) % 2 == 0,
              "stem input: uint8 [N, H, W, 3], even H / W");
  const int ldc = act_channels(dz, "dz");
  TORCH_CHECK(dz.dim() == 4 && dz.size(0) == x.size(0) && dz.size(1) == x.size(1) / 2 && dz.size(2) == x.size(2) / 2 &&
              ldc >= 32, "dz: bf16 [N, H/2, W/2, ldc >= 32]");
  vec(G, at::kFloat, 27 * 32, "G", 4);
  b200::mbv2_stem_wgrad(x.data_ptr<uint8_t>(), dz.data_ptr(), G.data_ptr<float>(), (int)x.size(0), (int)x.size(1),
                        (int)x.size(2), ldc, (float)mul, (float)add, cur());
  after();
}
// device table: int64 [layers, fields] on the same device as the flat buffers
static void ft_table(const Tensor& table, const Tensor& like, int fields) {
  chk(table, at::kLong, "table");
  TORCH_CHECK(table.dim() == 2 && table.size(1) == fields && table.size(0) >= 1 && table.size(0) <= 128,
              "table: int64 [layers (1..128), fields]");
  TORCH_CHECK(table.device() == like.device(), "table must be on the device of the flat buffers");
}
void mbv2_ft_finalize(Tensor params, Tensor w16, Tensor grads, Tensor table) {
  chk(params, at::kFloat, "params");
  vec(w16, at::kBFloat16, params.numel(), "w16", 1);
  vec(grads, at::kFloat, params.numel(), "grads", 1);
  ft_table(table, params, b200::kFtFinalizeFields);
  b200::mbv2_ft_finalize(params.data_ptr<float>(), w16.data_ptr(), grads.data_ptr<float>(), table.data_ptr<int64_t>(),
                         (int)table.size(0), cur());
  after();
}
void mbv2_ft_refresh(Tensor params, Tensor table) {
  chk(params, at::kFloat, "params");
  ft_table(table, params, b200::kFtRefreshFields);
  b200::mbv2_ft_refresh(params.data_ptr<float>(), table.data_ptr<int64_t>(), (int)table.size(0), cur());
  after();
}

// ------------------------------------------------------------------------------------------------ augmentation
// params int32 [N, 8] (16-byte aligned rows) of a batch of N images of H x W
static void aug_params_table(const Tensor& params, int64_t N, const char* name) {
  chk(params, at::kInt, name);
  TORCH_CHECK(params.dim() == 2 && params.size(1) == b200::kAugParamFields && params.size(0) == N,
              name, " must be int32 [N, 8] for the batch's N images");
  aligned(params, 16, name);
}
static void aug_side(int64_t H, int64_t W) {
  TORCH_CHECK(H >= 1 && W >= 1 && H <= b200::kAugMaxSide && W <= b200::kAugMaxSide,
              "augmentation: image sides must be in 1..2048");
}
// params[n] = transform of image n for the step held in `step` (int32 [1] on the device); see csrc/augment.cu
void augment_params(Tensor params, Tensor step, Tensor rot_table, int64_t H, int64_t W, int64_t key, int64_t flip_mode,
                    int64_t zq, int64_t txq, int64_t tyq) {
  TORCH_CHECK(params.dim() == 2 && params.size(0) >= 1, "params must be int32 [N, 8] with N >= 1");
  aug_params_table(params, params.size(0), "params");
  vec(step, at::kInt, 1, "step", 4);
  vec(rot_table, at::kInt, 2 << b200::kAugRotBits, "rot_table", 8);
  TORCH_CHECK(step.device() == params.device() && rot_table.device() == params.device(),
              "step and rot_table must be on the device of params");
  aug_side(H, W);
  TORCH_CHECK(key >= 0 && key <= 0xFFFFFFFFLL, "key must be a uint32");
  TORCH_CHECK(flip_mode >= 0 && flip_mode <= 3, "flip_mode: bit 0 horizontal, bit 1 vertical");
  TORCH_CHECK(zq >= 0 && zq < 65536, "zq: Q16.16 zoom factor in [0, 1)");
  TORCH_CHECK(txq >= 0 && txq <= W * 65536 && tyq >= 0 && tyq <= H * 65536,
              "txq / tyq: Q16.16 translation in [0, W] / [0, H] pixels");
  b200::augment_params(params.data_ptr<int32_t>(), step.data_ptr<int32_t>(), rot_table.data_ptr<int32_t>(),
                       (int)params.size(0), (int)H, (int)W, (uint32_t)key, (int)flip_mode, (int32_t)zq, (int32_t)txq,
                       (int32_t)tyq, cur());
  after();
}
// out = bilinear warp of x (uint8 [N, H, W, 3]) by the per-image maps in params; fill_mode "reflect" or "constant"
void augment_warp(Tensor x, Tensor out, Tensor params, std::string fill_mode, int64_t fill_value) {
  chk(x, at::kByte, "x");
  chk(out, at::kByte, "out");
  TORCH_CHECK(x.dim() == 4 && x.size(3) == 3 && x.size(0) >= 1, "x must be uint8 [N, H, W, 3]");
  TORCH_CHECK(out.sizes() == x.sizes(), "out must have the shape of x");
  TORCH_CHECK(out.device() == x.device() && params.device() == x.device(), "x, out and params must share a device");
  TORCH_CHECK(out.data_ptr() != x.data_ptr(), "augment_warp cannot run in place");
  aligned(out, 16, "out");
  aug_side(x.size(1), x.size(2));
  aug_params_table(params, x.size(0), "params");
  TORCH_CHECK(fill_mode == "reflect" || fill_mode == "constant", "fill_mode must be 'reflect' or 'constant'");
  TORCH_CHECK(fill_value >= 0 && fill_value <= 255, "fill_value must be a uint8");
  b200::augment_warp(x.data_ptr<uint8_t>(), out.data_ptr<uint8_t>(), params.data_ptr<int32_t>(), (int)x.size(0),
                     (int)x.size(1), (int)x.size(2), fill_mode == "reflect", (int)fill_value, cur());
  after();
}

// augment_params plus the mix rows (int32 [N, 8]) of MixUp (mode 1) or CutMix (mode 2) in the same launch
void augment_mix_params(Tensor params, Tensor mix, Tensor step, Tensor rot_table, Tensor lam_table, int64_t H, int64_t W,
                        int64_t key, int64_t flip_mode, int64_t zq, int64_t txq, int64_t tyq, int64_t mode) {
  TORCH_CHECK(params.dim() == 2 && params.size(0) >= 1, "params must be int32 [N, 8] with N >= 1");
  aug_params_table(params, params.size(0), "params");
  aug_params_table(mix, params.size(0), "mix");
  TORCH_CHECK(mix.data_ptr() != params.data_ptr(), "mix and params must be separate buffers");
  vec(step, at::kInt, 1, "step", 4);
  vec(rot_table, at::kInt, 2 << b200::kAugRotBits, "rot_table", 8);
  vec(lam_table, at::kInt, 2 << b200::kAugLamBits, "lam_table", 8);
  for (const Tensor* t : {&mix, &step, &rot_table, &lam_table})
    TORCH_CHECK(t->device() == params.device(), "mix, step, rot_table and lam_table must be on the device of params");
  aug_side(H, W);
  TORCH_CHECK(key >= 0 && key <= 0xFFFFFFFFLL, "key must be a uint32");
  TORCH_CHECK(flip_mode >= 0 && flip_mode <= 3, "flip_mode: bit 0 horizontal, bit 1 vertical");
  TORCH_CHECK(zq >= 0 && zq < 65536, "zq: Q16.16 zoom factor in [0, 1)");
  TORCH_CHECK(txq >= 0 && txq <= W * 65536 && tyq >= 0 && tyq <= H * 65536,
              "txq / tyq: Q16.16 translation in [0, W] / [0, H] pixels");
  TORCH_CHECK(mode == b200::kMixUp || mode == b200::kCutMix, "mode: 1 MixUp, 2 CutMix");
  b200::augment_mix_params(params.data_ptr<int32_t>(), mix.data_ptr<int32_t>(), step.data_ptr<int32_t>(),
                           rot_table.data_ptr<int32_t>(), lam_table.data_ptr<int32_t>(), (int)params.size(0), (int)H,
                           (int)W, (uint32_t)key, (int)flip_mode, (int32_t)zq, (int32_t)txq, (int32_t)tyq, (int)mode,
                           cur());
  after();
}
// out = augment_warp of x mixed with each image's partner by its mix row (mode 1 MixUp, 2 CutMix)
void augment_mix_warp(Tensor x, Tensor out, Tensor params, Tensor mix, int64_t mode, std::string fill_mode,
                      int64_t fill_value) {
  chk(x, at::kByte, "x");
  chk(out, at::kByte, "out");
  TORCH_CHECK(x.dim() == 4 && x.size(3) == 3 && x.size(0) >= 1, "x must be uint8 [N, H, W, 3]");
  TORCH_CHECK(out.sizes() == x.sizes(), "out must have the shape of x");
  TORCH_CHECK(out.device() == x.device() && params.device() == x.device() && mix.device() == x.device(),
              "x, out, params and mix must share a device");
  TORCH_CHECK(out.data_ptr() != x.data_ptr(), "augment_mix_warp cannot run in place");
  aligned(out, 16, "out");
  aug_side(x.size(1), x.size(2));
  aug_params_table(params, x.size(0), "params");
  aug_params_table(mix, x.size(0), "mix");
  TORCH_CHECK(mode == b200::kMixUp || mode == b200::kCutMix, "mode: 1 MixUp, 2 CutMix");
  TORCH_CHECK(fill_mode == "reflect" || fill_mode == "constant", "fill_mode must be 'reflect' or 'constant'");
  TORCH_CHECK(fill_value >= 0 && fill_value <= 255, "fill_value must be a uint8");
  b200::augment_mix_warp(x.data_ptr<uint8_t>(), out.data_ptr<uint8_t>(), params.data_ptr<int32_t>(),
                         mix.data_ptr<int32_t>(), (int)x.size(0), (int)x.size(1), (int)x.size(2), (int)mode,
                         fill_mode == "reflect", (int)fill_value, cur());
  after();
}

// dst = color augmentation of src (uint8 [N, H, W, 3]; dst may be src) for the step held in `step`; returns the number
// of CTAs per image launched (`cluster`: 1, 2, 4 or 8, or 0 to let the launch choose; the bytes do not depend on it)
int64_t augment_color(Tensor src, Tensor dst, Tensor step, int64_t H, int64_t W, int64_t ckey, int64_t bq, int64_t cq,
                      int64_t sq, int64_t hq, int64_t pq, int64_t cluster) {
  chk(src, at::kByte, "src");
  chk(dst, at::kByte, "dst");
  TORCH_CHECK(src.dim() == 4 && src.size(3) == 3 && src.size(0) >= 1, "src must be uint8 [N, H, W, 3]");
  TORCH_CHECK(src.size(1) == H && src.size(2) == W, "src must be [N, H, W, 3] for the given H and W");
  TORCH_CHECK(dst.sizes() == src.sizes(), "dst must have the shape of src");
  aug_side(H, W);
  TORCH_CHECK(src.size(0) * b200::kAugColorMaxCluster < (1LL << 31), "augment_color: batch too large");
  aligned(src, 16, "src");
  aligned(dst, 16, "dst");
  const bool same = src.data_ptr() == dst.data_ptr();
  if (!same) {   // in place is allowed; a partial overlap is not
    const auto s0 = reinterpret_cast<uintptr_t>(src.data_ptr()), d0 = reinterpret_cast<uintptr_t>(dst.data_ptr());
    const auto nb = (uintptr_t)src.numel();
    TORCH_CHECK(s0 + nb <= d0 || d0 + nb <= s0, "augment_color: src and dst overlap without being the same buffer");
  }
  vec(step, at::kInt, 1, "step", 4);
  TORCH_CHECK(dst.device() == src.device() && step.device() == src.device(), "src, dst and step must share a device");
  TORCH_CHECK(ckey >= 0 && ckey <= 0xFFFFFFFFLL, "ckey must be a uint32");
  TORCH_CHECK(bq >= 0 && bq <= 255 * 256, "bq: Q8 brightness half-range in [0, 255 * 256]");
  TORCH_CHECK(cq >= 0 && cq <= 65536, "cq: Q16 contrast half-range in [0, 1]");
  TORCH_CHECK(sq >= 0 && sq <= 65536, "sq: Q16 saturation half-range in [0, 1]");
  TORCH_CHECK(hq >= 0 && hq <= 3 * 65536, "hq: Q16 hue half-range in [0, 3] sixths of a turn");
  TORCH_CHECK(pq >= 0 && pq <= 65536, "pq: Q16 grayscale probability in [0, 1]");
  TORCH_CHECK(cluster == 0 || cluster == 1 || cluster == 2 || cluster == 4 || cluster == 8,
              "cluster must be 0 (chosen by the launch), 1, 2, 4 or 8");
  const int G = b200::augment_color(src.data_ptr<uint8_t>(), dst.data_ptr<uint8_t>(), step.data_ptr<int32_t>(),
                                    (int)src.size(0), (int)H, (int)W, (uint32_t)ckey, (int32_t)bq, (int32_t)cq,
                                    (int32_t)sq, (int32_t)hq, (int32_t)pq, (int)cluster, cur());
  after();
  TORCH_CHECK(G > 0, "augment_color: the cluster launch failed");
  return G;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  namespace py = pybind11;
  m.doc() = "b200ddl bandwidth-bound sm_90a kernels and fused optimizers";
  m.def("bn_finalize", &bn_finalize);
  m.def("bn_apply", &bn_apply, py::arg("y"), py::arg("scale"), py::arg("shift"), py::arg("res") = c10::nullopt,
        py::arg("res_scale") = c10::nullopt, py::arg("res_shift") = c10::nullopt, py::arg("out"), py::arg("relu") = true,
        py::arg("mask") = c10::nullopt, py::arg("relu6") = false);
  m.def("channel_stats", &channel_stats);
  m.def("bn_bwd_reduce", &bn_bwd_reduce);
  m.def("bn_bwd_coeffs", &bn_bwd_coeffs, py::arg("sum_dz"), py::arg("sum_dzy"), py::arg("gamma"), py::arg("mean"),
        py::arg("invstd"), py::arg("count"), py::arg("dgamma"), py::arg("dbeta"), py::arg("cA"), py::arg("cB"),
        py::arg("cC"), py::arg("inference") = false);
  m.def("bn_bwd_apply", &bn_bwd_apply);
  m.def("bn_apply_fused", &bn_apply_fused, py::arg("y"), py::arg("pack"), py::arg("count"), py::arg("momentum"),
        py::arg("eps"), py::arg("res") = c10::nullopt, py::arg("res_pack") = c10::nullopt, py::arg("out"),
        py::arg("relu") = true, py::arg("mask") = c10::nullopt);
  m.def("bn_bwd_apply_fused", &bn_bwd_apply_fused);
  m.def("maxpool_fwd", &maxpool_fwd);
  m.def("maxpool_bwd", &maxpool_bwd);
  m.def("bn_relu_maxpool_fwd", &bn_relu_maxpool_fwd);
  m.def("gap_fwd", &gap_fwd);
  m.def("gap_bwd", &gap_bwd);
  m.def("softmax_ce", &softmax_ce);
  m.def("softmax_ce_head", &softmax_ce_head, py::arg("logits16"), py::arg("bias"), py::arg("labels"),
        py::arg("logits32") = c10::nullopt, py::arg("dlogits16") = c10::nullopt, py::arg("loss_rows") = c10::nullopt,
        py::arg("stats"), py::arg("grad_scale") = 1.0,
        py::arg("class_weight") = c10::nullopt, py::arg("row_weight") = c10::nullopt);
  m.def("softmax_ce_soft_head", &softmax_ce_soft_head, py::arg("logits16"), py::arg("bias"), py::arg("labels"),
        py::arg("mix") = c10::nullopt, py::arg("label_smoothing") = 0.0, py::arg("logits32") = c10::nullopt,
        py::arg("dlogits16") = c10::nullopt, py::arg("loss_rows") = c10::nullopt, py::arg("stats"),
        py::arg("grad_scale") = 1.0,
        py::arg("class_weight") = c10::nullopt, py::arg("row_weight") = c10::nullopt);
  m.def("softmax_kd_head", &softmax_kd_head, py::arg("logits16"), py::arg("bias"), py::arg("tlogits16"),
        py::arg("tbias"), py::arg("labels"), py::arg("mix") = c10::nullopt, py::arg("label_smoothing") = 0.0,
        py::arg("alpha") = 0.1, py::arg("temperature") = 3.0, py::arg("logits32") = c10::nullopt,
        py::arg("dlogits16") = c10::nullopt, py::arg("loss_rows") = c10::nullopt, py::arg("stats"),
        py::arg("grad_scale") = 1.0,
        py::arg("class_weight") = c10::nullopt, py::arg("row_weight") = c10::nullopt);
  m.def("fc_bias_grad", &fc_bias_grad);
  m.def("pack_stem_weight", &pack_stem_weight);
  m.def("stem_pool_bn_bwd", &stem_pool_bn_bwd, py::arg("pass_"), py::arg("idx"), py::arg("g1"), py::arg("g2"), py::arg("y"),
        py::arg("scale"), py::arg("shift"), py::arg("cA") = c10::nullopt, py::arg("cB") = c10::nullopt,
        py::arg("cC") = c10::nullopt, py::arg("dy") = c10::nullopt, py::arg("sum_dz"), py::arg("sum_dzy"));
  m.def("zero_", &zero_);
  m.def("set_bn_rows_unroll", [](int64_t u) { b200::set_bn_rows_unroll((int)u); });
  m.def("get_bn_rows_unroll", []() { return (int64_t)b200::get_bn_rows_unroll(); });
  m.def("mbv2_stem", &mbv2_stem);
  m.def("dwconv3x3", &dwconv3x3, pybind11::arg("x"), pybind11::arg("w"), pybind11::arg("scale"), pybind11::arg("shift"),
        pybind11::arg("out"), pybind11::arg("stride"), pybind11::arg("tile_w") = 4);
  m.def("mbv2_stem_stats", &mbv2_stem_stats, py::arg("x"), py::arg("w"), py::arg("out"), py::arg("sum"), py::arg("sqsum"),
        py::arg("mul"), py::arg("add"));
  m.def("dwconv3x3_stats", &dwconv3x3_stats, py::arg("x"), py::arg("w"), py::arg("out"), py::arg("sum"), py::arg("sqsum"),
        py::arg("stride"), py::arg("tile_w") = 4);
  m.def("preprocess_u8", &preprocess_u8);
  m.def("resize_bilinear_u8", &resize_bilinear_u8, py::arg("x"), py::arg("out"), py::arg("planar") = false);
  m.def("weight_prep", &weight_prep);
  m.def("weight_prep_batched", &weight_prep_batched);
  m.def("optim_step", &optim_step, py::arg("rule"), py::arg("p"), py::arg("g"), py::arg("state"), py::arg("p16"),
        py::arg("hyper"));
  m.def("segment_sumsq", &segment_sumsq);
  m.def("segment_finalize", &segment_finalize);
  m.def("clip_apply", &clip_apply);
  m.def("lamb_moments", &lamb_moments);
  m.def("lamb_apply", &lamb_apply);
  m.def("grad_accumulate", &grad_accumulate);
  m.def("ema_update", &ema_update);
  m.def("cast_bf16", &cast_bf16);
  m.def("launch_count", [] { return g_launches; });
  m.def("reset_launch_count", [] { g_launches = 0; });
  m.def("relu6_mask_reduce", &relu6_mask_reduce, py::arg("g1"), py::arg("g2"), py::arg("y"), py::arg("dz"), py::arg("sum"),
        py::arg("relu6") = true, py::arg("c") = c10::nullopt, py::arg("sum_dzc") = c10::nullopt);
  m.def("dw_dgrad", &dw_dgrad);
  m.def("dw_wgrad", &dw_wgrad);
  m.def("mbv2_stem_wgrad", &mbv2_stem_wgrad);
  m.def("mbv2_ft_finalize", &mbv2_ft_finalize);
  m.def("mbv2_ft_refresh", &mbv2_ft_refresh);
  m.def("augment_params", &augment_params, py::arg("params"), py::arg("step"), py::arg("rot_table"), py::arg("H"),
        py::arg("W"), py::arg("key"), py::arg("flip_mode"), py::arg("zq"), py::arg("txq"), py::arg("tyq"));
  m.def("augment_warp", &augment_warp, py::arg("x"), py::arg("out"), py::arg("params"), py::arg("fill_mode"),
        py::arg("fill_value"));
  m.def("augment_mix_params", &augment_mix_params, py::arg("params"), py::arg("mix"), py::arg("step"),
        py::arg("rot_table"), py::arg("lam_table"), py::arg("H"), py::arg("W"), py::arg("key"), py::arg("flip_mode"),
        py::arg("zq"), py::arg("txq"), py::arg("tyq"), py::arg("mode"));
  m.def("augment_mix_warp", &augment_mix_warp, py::arg("x"), py::arg("out"), py::arg("params"), py::arg("mix"),
        py::arg("mode"), py::arg("fill_mode"), py::arg("fill_value"));
  m.def("augment_color", &augment_color, py::arg("src"), py::arg("dst"), py::arg("step"), py::arg("H"), py::arg("W"),
        py::arg("ckey"), py::arg("bq"), py::arg("cq"), py::arg("sq"), py::arg("hq"), py::arg("pq"),
        py::arg("cluster") = 0);
}
