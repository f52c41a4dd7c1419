"""Every layer of the ResNet-50 training step (and of the inference build) against a float64 oracle fed the engine's own
tensors.

End-to-end comparisons of a bf16 network have to be loose (rounding differences grow through 50 layers), so they cannot
see a wrong buffer, a swapped tap part or a gradient off by a few percent in one layer.  Here each layer's float64
reference is evaluated on the engine's own inputs to that layer (forward activations, BatchNorm statistics and the
backward gradients captured as the step runs), so the only admissible difference is that layer's own rounding:

* a bf16 output may be off by half a bf16 ulp of its value (`exact_util.bf16_bound`) plus the error of the fp32
  arithmetic behind it;
* an fp32 sum of terms is off by at most ``depth * u * sum|terms|``, where ``depth`` is the longest chain of additions
  a term goes through, taken from the kernel's plan (register partials, tiles, atomics).  Tensor-core GEMMs are charged
  2u per addition because their accumulators may truncate instead of rounding to nearest;
* ``bn_finalize`` computes ``var = E[y^2] - E[y]^2`` in fp32: the error of E[y^2] is carried through the cancellation
  to ``invstd`` and the running variance.

Every check also asserts ``||bound|| / ||ref|| <= 1/16``, so no off-by-a-factor, wrong-tensor or wrong-channel error can
hide inside a bound.  The network's structure (strides, paddings, downsample placement, eps, momentum) comes from
torchvision's ResNet-50, loaded with the engine's weights, not from the engine's own block table.
"""
from __future__ import annotations

import math
from typing import List

import pytest
import torch
import torch.nn.functional as F

from exact_util import DEV, U, bf16_bound

pytestmark = pytest.mark.gpu

UM = 2.0 ** -23      # per addition of a tensor-core accumulator (round-toward-zero allowed)
TEETH = 1.0 / 16     # largest admissible ||bound|| / ||ref||
N_BATCH, CLASSES, SIZE = 8, 10, 224

PATHS = {
    "default": ({}, {}),
    "no_block_grad": ({"fuse_block_grad": False}, {}),
    "fuse_bn_coeffs": ({"fuse_bn_coeffs": True}, {}),
    "tails": ({}, {"B200DDL_TAILS": "1"}),
    "fuse_stem_bwd": ({"fuse_stem_bwd": True}, {}),
    "no_overlap_wgrad": ({"overlap_wgrad": False}, {}),
    "torch_stem": ({"native_stem": False}, {}),
}
TORCH_STEM_EXEMPT = {
    "conv1 y": "the stem convolution is torch's bf16 conv2d; cuDNN's accumulation order cannot be derived",
    "conv1.weight wgrad": "the stem weight gradient is torch's bf16 conv2d_weight; cuDNN's accumulation order cannot be derived",
}
# bounds that are asserted but may exceed ||ref|| / 16: the reduction itself cancels (printed ratios measured on an H100)
TEETH_EXEMPT = {
    "bn1 dbeta": "sum of dz over 100,352 stem pixels cancels; through up to 1,091 fp32 additions (1,056 per-block "
                 "atomics when the pooled gradient is materialised) the bound is 0.067-0.082 of ||ref||",
    "layer1.0.bn1 dgamma": "sum dz*y - mean * sum dz over 25,088 pixels cancels; the bound is 0.063-0.074 of ||ref||",
}


# ------------------------------------------------------------------------------------------------ report
class Report:
    """Collects one row per checked tensor and the failures; `failures` names the layer of each."""

    def __init__(self, exempt=None):
        self.exempt = dict(exempt or {})
        self.failures: List[str] = []
        self.rows: List[tuple] = []
        self.params = set()

    def bounded(self, key, got, ref, bound, teeth_ref=None, param=None):
        got, ref, bound = got.double(), ref.double(), bound.double()
        assert got.shape == ref.shape == bound.shape, (key, got.shape, ref.shape, bound.shape)
        err = (got - ref).abs()
        bad = ~(err <= bound)
        worst = float(torch.where(bound > 0, err / bound, torch.where(err > 0, math.inf, 0.0)).max())
        tr = (ref if teeth_ref is None else teeth_ref).double()
        ratio = float(bound.norm() / tr.norm()) if float(tr.norm()) > 0 else math.inf
        if param is not None:
            self.params.add(param)
        note = self.exempt.get(key)
        loose = TEETH_EXEMPT.get(key) if ratio > TEETH else None
        self.rows.append((key, worst, ratio, note or loose))
        if note is not None:
            return
        if bool(bad.any()):
            ix = tuple(bad.nonzero()[0].tolist())
            self.failures.append(f"{key}: {int(bad.sum())} of {bad.numel()} elements outside the bound; at {ix} got "
                                 f"{got[ix].item():.6g} want {ref[ix].item():.6g} (bound {bound[ix].item():.3g}), "
                                 f"worst err/bound {worst:.3g}")
        if ratio > TEETH and loose is None:
            self.failures.append(f"{key}: bound too loose, ||bound||/||ref|| = {ratio:.3g} > 1/16")

    def equal(self, key, ok, detail=""):
        self.rows.append((key, 0.0 if ok else math.inf, 0.0, None))
        if not ok:
            self.failures.append(f"{key}: {detail}")

    def print(self, title):
        print(f"\n== {title}: {len(self.rows)} tensors checked")
        for key, worst, ratio, note in self.rows:
            tail = f"  EXEMPT: {note}" if note else ""
            print(f"  {key:<44} max err/bound {worst:9.3g}   ||bound||/||ref|| {ratio:9.3g}{tail}")


# ------------------------------------------------------------------------------------------------ float64 references
def nchw(t):
    return t.double().permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def conv_fwd(x, conv):
    """(ref, sum|terms|) of conv(x) for an NHWC input and a torch Conv2d (float64 weights)."""
    a = dict(stride=conv.stride, padding=conv.padding)
    return (nhwc(F.conv2d(nchw(x), conv.weight, **a)), nhwc(F.conv2d(nchw(x).abs(), conv.weight.abs(), **a)))


def conv_dgrad(dy, conv, x_shape):
    N, H, W, Cin = x_shape
    a = dict(stride=conv.stride, padding=conv.padding)
    g = torch.nn.grad.conv2d_input
    return (nhwc(g((N, Cin, H, W), conv.weight, nchw(dy), **a)),
            nhwc(g((N, Cin, H, W), conv.weight.abs(), nchw(dy).abs(), **a)))


def conv_wgrad(x, dy, conv):
    a = dict(stride=conv.stride, padding=conv.padding)
    g = torch.nn.grad.conv2d_weight
    return (g(nchw(x), conv.weight.shape, nchw(dy), **a), g(nchw(x).abs(), conv.weight.shape, nchw(dy).abs(), **a))


def gemm_depth(K):
    """Additions on a term's path in one tensor-core reduction of length K: one per k16 MMA, <= 16 inside it."""
    return -(-K // 16) + 16


def kernel_grad(rec, name):
    """Engine gradient of a conv filter in torch's OIHW layout (the flat buffer holds [R*S, Cout, Cin])."""
    from b200ddl.ops import conv as C

    g = rec["grads"][name]
    k = int(round(math.sqrt(g.shape[0])))
    return C.weight_from_kernel_layout(g.double(), k, k)


def flat(t):
    return t.double().reshape(-1, t.shape[-1])


def unpack_mask(m, shape):
    bits = (m.view(-1, 1).to(torch.int32) >> torch.arange(8, device=m.device, dtype=torch.int32)) & 1
    return bits.view(shape).bool()


def stats_ref(y, depth):
    """Float64 batch statistics of the engine's bf16 ``y`` and bounds on what fp32 ``bn_finalize`` may produce from
    fp32 sums of depth ``depth``: mean, biased variance, and their bounds."""
    y = flat(y)
    M = y.shape[0]
    mean = y.mean(0)
    e2 = (y * y).mean(0)
    var = e2 - mean * mean
    d_mean = depth * U * y.abs().mean(0) + 3 * U * mean.abs()
    d_e2 = (depth + 3) * U * e2
    am = mean.abs() + d_mean
    # E[y^2] - mean^2: the E[y^2] error passes the cancellation unchanged; then mean^2 and the subtraction round
    d_var = d_e2 + (2 * mean.abs() + d_mean) * d_mean + U * am * am + U * (e2 + d_e2 + am * am)
    return M, mean, var, d_mean, d_var


def invstd_bound(var, d_var, eps):
    """|rsqrtf(max(v, 0) + eps) - 1/sqrt(var + eps)| for |v - var| <= d_var (rsqrtf: 2 ulp, eps add: one rounding)."""
    d = d_var + U * (var.abs() + d_var + eps) + U * eps
    lo = torch.clamp(var + eps - d, min=eps * (1 - U))
    hi = var + eps + d
    ref = (var + eps).rsqrt()
    return ref, torch.maximum(lo.rsqrt() - ref, ref - hi.rsqrt()) + 4 * U * lo.rsqrt()


def bn_bwd_ref(dz_sum, dz_apply, y, mean, invstd, gamma, depth, dz_err=0.0):
    """BatchNorm backward from the engine's incoming gradient: dbeta = sum dz, dgamma = invstd (sum dz*y - mean sum dz),
    dy = A dz + B y + C with the engine's fp32 mean / invstd.  ``dz_sum``: the values the kernel reduces; ``dz_apply``:
    the values its apply pass reads (they differ where an fp32 sum is reduced before its bf16 store).  ``dz_err``:
    per-element bound on how far the kernel's own dz may be from them.  Returns refs and bounds."""
    dz_sum, dz_apply, y = flat(dz_sum), flat(dz_apply), flat(y)
    if torch.is_tensor(dz_err):
        dz_err = flat(dz_err)
    M = y.shape[0]
    m, s, g = mean.double(), invstd.double(), gamma.double()
    s1 = dz_sum.sum(0)
    s2 = (dz_sum * y).sum(0)
    e1 = depth * U * dz_sum.abs().sum(0) + (dz_err + 0 * y).sum(0)
    e2 = depth * U * (dz_sum * y).abs().sum(0) + (dz_err * y.abs()).sum(0)
    inner = s2 - m * s1
    d_inner = e2 + m.abs() * e1 + U * m.abs() * (s1.abs() + e1) + U * (inner.abs() + e2 + m.abs() * e1)
    dg = s * inner
    d_dg = s * d_inner * (1 + U) + U * dg.abs()
    A = g * s
    B = -A * s * dg / M
    Cc = -A * s1 / M - B * m
    dA = U * A.abs()
    dB = (A * s / M).abs() * d_dg + 5 * U * B.abs()
    dC = (A / M).abs() * e1 + m.abs() * dB + 5 * U * ((A * s1 / M).abs() + (B * m).abs())
    dy = A * dz_apply + B * y + Cc
    e = dz_apply.abs() * dA + A.abs() * dz_err + y.abs() * dB + dC + U * ((B * y + Cc).abs() + dy.abs())
    return dict(dbeta=s1, d_dbeta=e1, dgamma=dg, d_dgamma=d_dg, dy=dy, d_dy=bf16_bound(dy, e))


def check_bn_bwd(rep, rec, bn, dz_sum, dz_apply, y, dz_err=0.0):
    w = rec["bnw"][bn]
    r = bn_bwd_ref(dz_sum, dz_apply, y, w["mean"], w["invstd"], rec["gamma"][bn], rec["depth"]["bwd"][bn], dz_err)
    rep.bounded(f"{bn} dbeta", rec["grads"][bn + ".bias"], r["dbeta"], r["d_dbeta"], param=bn + ".bias")
    rep.bounded(f"{bn} dgamma", rec["grads"][bn + ".weight"], r["dgamma"], r["d_dgamma"], param=bn + ".weight")
    rep.bounded(f"{bn} dy", flat(rec["bwd"][bn]["dy"] if bn != "bn1" else rec["dy0"]), r["dy"], r["d_dy"])


def check_stats(rep, rec, bn, y, bnmod):
    """Batch mean / invstd in ``bnw`` and the running-statistics update of one BatchNorm (training)."""
    M, mean, var, d_mean, d_var = stats_ref(y, rec["depth"]["fwd"][bn])
    w = rec["bnw"][bn]
    rep.bounded(f"{bn} mean", w["mean"], mean, d_mean)
    ref_is, d_is = invstd_bound(var, d_var, bnmod.eps)
    rep.bounded(f"{bn} invstd", w["invstd"], ref_is, d_is)
    mom = bnmod.momentum
    rm0, rv0 = (t.double() for t in rec["run_before"][bn])
    rm1, rv1 = rec["run_after"][bn]
    unb = M / (M - 1.0)
    rep.bounded(f"{bn} running_mean", rm1, (1 - mom) * rm0 + mom * mean,
                mom * d_mean + 4 * U * (rm0.abs() + mean.abs()), teeth_ref=mom * mean)
    rep.bounded(f"{bn} running_var", rv1, (1 - mom) * rv0 + mom * var * unb,
                mom * unb * d_var + 6 * U * (rv0.abs() + var.abs() * unb), teeth_ref=mom * var * unb)


def check_affine(rep, rec, bn):
    """scale = gamma * invstd and shift = beta - mean * scale, as the apply kernels read them."""
    w = rec["bnw"][bn]
    g, b = rec["gamma"][bn].double(), rec["beta"][bn].double()
    sc_ref = g * w["invstd"].double()
    rep.bounded(f"{bn} scale", w["scale"], sc_ref, U * sc_ref.abs())
    sh_ref = b - w["mean"].double() * w["scale"].double()
    rep.bounded(f"{bn} shift", w["shift"], sh_ref, 2 * U * (b.abs() + (w["mean"].double() * w["scale"].double()).abs()))


def bn_pre(rec, bn, y):
    w = rec["bnw"][bn]
    v = flat(y) * w["scale"].double() + w["shift"].double()
    return v, U * v.abs()  # fmaf: one rounding


def stem_input(x_u8):
    """The normalised bf16 image both stems feed the convolution: bf16(fmaf(x, fp32(1/127.5), -1)), NCHW float64.
    x * m - 1 is exact in float64 (8 x 24 significant bits), so one fp32 rounding reproduces fmaf."""
    m = float(torch.tensor(1.0 / 127.5, dtype=torch.float32))
    return (x_u8.double() * m - 1.0).float().to(torch.bfloat16).double().permute(0, 3, 1, 2)


def check_stem_pool(rep, rec, key):
    """p0 = maxpool3x3/2(relu(BN(y0))): the value of each window's maximum, and pool_idx pointing at a maximum."""
    v, e = bn_pre(rec, "bn1", rec["y0"])
    a = v.clamp(min=0).view(rec["y0"].shape)
    ab = bf16_bound(a, e.view(a.shape))
    mx = nhwc(F.max_pool2d(nchw(a), 3, 2, 1))
    # rounding is monotone: the maximum of the rounded values is the rounded maximum
    rep.bounded(f"{key} p0", rec["p0"], mx, nhwc(F.max_pool2d(nchw(ab), 3, 2, 1)))
    idx = rec["pool_idx"].long()
    N, Ho, Wo, C_ = idx.shape
    ho = torch.arange(Ho, device=DEV).view(1, Ho, 1, 1)
    wo = torch.arange(Wo, device=DEV).view(1, 1, Wo, 1)
    h, w = 2 * ho - 1 + idx // 3, 2 * wo - 1 + idx % 3
    H, W = a.shape[1:3]
    inside = (idx <= 8) & (h >= 0) & (h < H) & (w >= 0) & (w < W)
    rep.equal(f"{key} pool_idx range", bool(inside.all()), f"{int((~inside).sum())} indices outside their window")
    n = torch.arange(N, device=DEV).view(N, 1, 1, 1)
    c = torch.arange(C_, device=DEV).view(1, 1, 1, C_)
    at = a[n, h.clamp(0, H - 1), w.clamp(0, W - 1), c]
    # the indexed element must be a maximum of its window up to the rounding of both
    tie = 2 * nhwc(F.max_pool2d(nchw(ab), 3, 2, 1))
    rep.bounded(f"{key} pool_idx", at, mx, tie, teeth_ref=mx)


def check_head(rep, rec, model):
    """GAP, FC logits (+bias), loss.  Returns nothing; the training backward head is checked separately."""
    feat = rec["out"]["layer4.2"].double()
    N, Hf, Wf, C_ = feat.shape
    ref = feat.mean((1, 2))
    e = (Hf * Wf - 1) * U * feat.abs().mean((1, 2)) + 2 * U * ref.abs()
    rep.bounded("avgpool pooled", rec["pooled"], ref, bf16_bound(ref, e))
    W = model.fc.weight
    K = W.shape[0]
    p = rec["pooled"].double()
    l_ref, l_abs = p @ W.t(), p.abs() @ W.abs().t()
    rep.bounded("fc logits16", rec["logits16"][:, :K], l_ref, bf16_bound(l_ref, UM * gemm_depth(C_) * l_abs))
    rep.equal("fc logits16 padding", bool((rec["logits16"][:, K:] == 0).all()), "padded logit columns are not zero")
    z_ref = rec["logits16"][:, :K].double() + model.fc.bias
    rep.bounded("fc logits", rec["logits"], z_ref, U * z_ref.abs())
    z = rec["logits"].double()
    lse = torch.logsumexp(z, 1)
    zl = z.gather(1, rec["labels"].view(-1, 1)).squeeze(1)
    # __expf / __logf (fast math): <= 2 + 1.2|x| ulp for |x| < 40, summed over K classes; 2^-16 covers it
    rep.bounded("loss rows", rec["loss_rows"], lse - zl, 2.0 ** -16 * (1 + lse.abs() + zl.abs()))
    return z


def check_forward_train(rep, rec, model):
    """Every forward layer of a training step: conv outputs, batch statistics, running statistics, BN apply, block
    outputs and masks, the stem pool, GAP and the head."""
    A = rec["act"]
    ref, ab = conv_fwd_stem(rec, model)
    rep.bounded("conv1 y", rec["y0"], ref, bf16_bound(ref, UM * gemm_depth(192) * ab))
    check_stats(rep, rec, "bn1", rec["y0"], model.bn1)
    check_affine(rep, rec, "bn1")
    check_stem_pool(rep, rec, "maxpool")
    x_in = rec["p0"]
    for name, blk in blocks(model):
        for c, bn, x, y in (("conv1", "bn1", x_in, "y1"), ("conv2", "bn2", A[name + ".a1"], "y2"),
                            ("conv3", "bn3", A[name + ".a2"], "y3")):
            conv = getattr(blk, c)
            ref, ab = conv_fwd(x, conv)
            rep.bounded(f"{name}.{c} y", A[f"{name}.{y}"], ref, bf16_bound(ref, UM * gemm_depth(conv.weight[0].numel()) * ab))
            check_stats(rep, rec, f"{name}.{bn}", A[f"{name}.{y}"], getattr(blk, bn))
            check_affine(rep, rec, f"{name}.{bn}")
        for bn, y, a in (("bn1", "y1", "a1"), ("bn2", "y2", "a2")):
            v, e = bn_pre(rec, f"{name}.{bn}", A[f"{name}.{y}"])
            ref = v.clamp(min=0)
            rep.bounded(f"{name}.{bn} relu", flat(A[f"{name}.{a}"]), ref, bf16_bound(ref, e))
        v3, e3 = bn_pre(rec, f"{name}.bn3", A[name + ".y3"])
        if blk.downsample is not None:
            conv = blk.downsample[0]
            ref, ab = conv_fwd(x_in, conv)
            rep.bounded(f"{name}.downsample.0 y", A[name + ".yd"], ref,
                        bf16_bound(ref, UM * gemm_depth(conv.weight[0].numel()) * ab))
            bd = f"{name}.downsample.1"
            check_stats(rep, rec, bd, A[name + ".yd"], blk.downsample[1])
            check_affine(rep, rec, bd)
            r, er = bn_pre(rec, bd, A[name + ".yd"])
        else:
            r, er = flat(x_in), 0.0
        pre = v3 + r
        e = e3 + er + U * pre.abs()
        ref = pre.clamp(min=0)
        out = flat(A[name + ".out"])
        rep.bounded(f"{name} out", out, ref, bf16_bound(ref, e))
        mask = unpack_mask(A[name + ".mask"], out.shape)
        rep.equal(f"{name} mask", bool((mask == (out > 0)).all()),
                  f"{int((mask != (out > 0)).sum())} mask bits differ from out > 0")
        x_in = A[name + ".out"]
    check_head(rep, rec, model)


def conv_fwd_stem(rec, model):
    c = model.conv1
    xs = rec["x_stem"]
    return (nhwc(F.conv2d(xs, c.weight, stride=c.stride, padding=c.padding)),
            nhwc(F.conv2d(xs.abs(), c.weight.abs(), stride=c.stride, padding=c.padding)))


def blocks(model):
    return [(f"layer{li}.{bi}", blk) for li in range(1, 5) for bi, blk in enumerate(getattr(model, f"layer{li}"))]


def check_backward(rep, rec, model):
    """Every backward layer: head, BatchNorm backward of all 53 BNs, dgrad (plain, block-gradient and compact forms)
    and wgrad of all 53 convolutions, max-pool backward."""
    A, cap, dx = rec["act"], rec["bwd"], rec["dx"]
    K = model.fc.weight.shape[0]
    z = rec["logits"].double()
    p = torch.softmax(z, 1)
    onehot = F.one_hot(rec["labels"], K).double()
    ref = (p - onehot) / N_BATCH
    rep.bounded("fc dlogits", rec["dlogits16"][:, :K], ref, bf16_bound(ref, 2.0 ** -16 * p / N_BATCH))
    rep.equal("fc dlogits padding", bool((rec["dlogits16"][:, K:] == 0).all()), "padded dlogit columns are not zero")
    dl = rec["dlogits16"].double()
    rep.bounded("fc.bias grad", rec["grads"]["fc.bias"], dl[:, :K].sum(0), 4 * U * dl[:, :K].abs().sum(0),
                param="fc.bias")
    pooled = rec["pooled"].double()
    rep.bounded("fc.weight grad", rec["grads"]["fc.weight"], dl.t() @ pooled,
                UM * rec["depth"]["wgrad"]["fc"] * (dl.abs().t() @ pooled.abs()), param="fc.weight")
    Wfc = torch.zeros(dl.shape[1], pooled.shape[1], dtype=torch.float64, device=DEV)
    Wfc[:K] = model.fc.weight
    ref = dl @ Wfc
    rep.bounded("fc dpooled", rec["dpooled"], ref, bf16_bound(ref, UM * gemm_depth(dl.shape[1]) * (dl.abs() @ Wfc.abs())))

    bl = blocks(model)
    for i in range(len(bl) - 1, -1, -1):
        name, blk = bl[i]
        x_in = A[bl[i - 1][0] + ".out"] if i > 0 else rec["p0"]
        mask = unpack_mask(A[name + ".mask"], A[name + ".out"].shape)
        c3 = cap[name + ".bn3"]
        # gradient arriving at the block output
        if i == len(bl) - 1:
            feat = A[name + ".out"]
            ref = (rec["dpooled"].double() / (feat.shape[1] * feat.shape[2]))[:, None, None, :].expand(feat.shape)
            rep.bounded("avgpool backward", c3["g1"], ref, bf16_bound(ref, 2 * U * ref.abs()))
        elif c3["g1"] is not None:
            nxt, nblk = bl[i + 1]
            rep.equal(f"{name}.bn3 g1 wiring", torch.equal(c3["g1"], dx[nxt + ".conv1"]),
                      f"main-path gradient is not {nxt}.conv1's dgrad")
            skip = dx[nxt + ".downsample.0"] if nblk.downsample is not None else cap[nxt + ".bn3"]["dz"]
            rep.equal(f"{name}.bn3 g2 wiring", torch.equal(c3["g2"], skip), f"skip gradient is not {nxt}'s")
        if c3["g1"] is not None:
            g = c3["g1"].double() + (c3["g2"].double() if c3["g2"] is not None else 0.0)
            dz_sum = g * mask
            rep.bounded(f"{name}.bn3 dz", c3["dz"], dz_sum, bf16_bound(dz_sum, U * dz_sum.abs()))
            # the reduction reads fp32 g1 + g2 (one rounding), the apply pass the stored bf16 dz
            check_bn_bwd(rep, rec, name + ".bn3", dz_sum, c3["dz"], A[name + ".y3"], dz_err=U * dz_sum.abs())
        else:
            check_bn_bwd(rep, rec, name + ".bn3", c3["dz"], c3["dz"], A[name + ".y3"])
        # conv3, bn2, conv2, bn1
        for c, bn_out, x, bn_in, y_in in (("conv3", "bn3", A[name + ".a2"], "bn2", "y2"),
                                          ("conv2", "bn2", A[name + ".a1"], "bn1", "y1")):
            conv = getattr(blk, c)
            dy = cap[f"{name}.{bn_out}"]["dy"]
            check_conv_bwd(rep, rec, f"{name}.{c}", conv, x, dy, dx[f"{name}.{c}"])
            cb = cap[f"{name}.{bn_in}"]
            rep.equal(f"{name}.{bn_in} g1 wiring", torch.equal(cb["g1"], dx[f"{name}.{c}"]),
                      f"incoming gradient is not {name}.{c}'s dgrad")
            v, _ = bn_pre(rec, f"{name}.{bn_in}", A[f"{name}.{y_in}"])
            dz = flat(cb["g1"]) * (v > 0)
            check_bn_bwd(rep, rec, f"{name}.{bn_in}", dz, dz, A[f"{name}.{y_in}"])
        if blk.downsample is not None:
            bd = name + ".downsample.1"
            cd = cap[bd]
            rep.equal(f"{bd} g1 wiring", torch.equal(cd["g1"], c3["dz"]), "incoming gradient is not the block's dz")
            check_bn_bwd(rep, rec, bd, cd["g1"], cd["g1"], A[name + ".yd"])
            check_conv_bwd(rep, rec, name + ".downsample.0", blk.downsample[0], x_in, cd["dy"], dx[name + ".downsample.0"])
        # conv1: its dgrad is either the plain gradient of the block input or, fused, the previous block's complete dz
        dy1 = cap[name + ".bn1"]["dy"]
        prev_fused = i > 0 and (bl[i - 1][0] + ".bn3") in rec["block_fused"]
        if prev_fused:
            skip = dx[name + ".downsample.0"] if blk.downsample is not None else c3["dz"]
            if skip.shape != x_in.shape:  # compact stride-2 skip gradient: the 1x1/2 projection's dgrad is zero elsewhere
                full = torch.zeros(x_in.shape, dtype=torch.float64, device=DEV)
                full[:, ::2, ::2] = skip.double()
                skip = full
            check_conv_bwd(rep, rec, name + ".conv1", blk.conv1, x_in, dy1, dx[name + ".conv1"],
                           skip=skip.double(), mask=unpack_mask(A[bl[i - 1][0] + ".mask"], x_in.shape))
        else:
            check_conv_bwd(rep, rec, name + ".conv1", blk.conv1, x_in, dy1, dx[name + ".conv1"])

    # stem: max-pool backward of (main + projection gradient of layer1.0), BN + ReLU backward, 7x7/2 wgrad
    g = (dx["layer1.0.conv1"].double() + dx["layer1.0.downsample.0"].double())
    idx = rec["pool_idx"].long()
    N, Ho, Wo, C_ = idx.shape
    H, W = rec["y0"].shape[1:3]
    ho = torch.arange(Ho, device=DEV).view(1, Ho, 1, 1).expand_as(idx)
    wo = torch.arange(Wo, device=DEV).view(1, 1, Wo, 1).expand_as(idx)
    n = torch.arange(N, device=DEV).view(N, 1, 1, 1).expand_as(idx)
    c = torch.arange(C_, device=DEV).view(1, 1, 1, C_).expand_as(idx)
    h = (2 * ho - 1 + idx // 3).clamp(0, H - 1)
    w = (2 * wo - 1 + idx % 3).clamp(0, W - 1)
    da = torch.zeros(rec["y0"].shape, dtype=torch.float64, device=DEV)
    da.index_put_((n, h, w, c), g, accumulate=True)
    da_abs = torch.zeros_like(da)
    da_abs.index_put_((n, h, w, c), dx["layer1.0.conv1"].double().abs() + dx["layer1.0.downsample.0"].double().abs(),
                      accumulate=True)
    # <= 4 windows of two bf16 terms each, summed in fp32 (<= 5 additions), then rounded to bf16.  Where the float64
    # sum is exact in fp32 (almost everywhere) every order gives bf16(da); elsewhere the kernel may be one bf16 step off.
    bound = bf16_bound(da, 5 * U * da_abs)
    da16 = da.float().to(torch.bfloat16).double()
    dz_err = torch.where(da.float().double() == da, 0.0, 2 * bound)
    v, _ = bn_pre(rec, "bn1", rec["y0"])
    keep = (v > 0).view(da.shape)
    if "bn1" in cap:   # the pooled gradient is materialised: it is what the BatchNorm backward reads
        rep.bounded("maxpool backward", cap["bn1"]["g1"], da, bound)
        da16, dz_err = cap["bn1"]["g1"].double(), 0.0
    dz = da16 * keep
    check_bn_bwd(rep, rec, "bn1", dz, dz, rec["y0"], dz_err * keep)
    xs = rec["x_stem"]
    c1 = model.conv1
    dy0 = nchw(rec["dy0"])
    ref = torch.nn.grad.conv2d_weight(xs, c1.weight.shape, dy0, stride=c1.stride, padding=c1.padding)
    ab = torch.nn.grad.conv2d_weight(xs.abs(), c1.weight.shape, dy0.abs(), stride=c1.stride, padding=c1.padding)
    rep.bounded("conv1.weight wgrad", kernel_grad(rec, "conv1.weight"), ref, UM * rec["depth"]["wgrad"]["conv1"] * ab,
                param="conv1.weight")


def check_conv_bwd(rep, rec, full, conv, x, dy, dx_got, skip=None, mask=None):
    """wgrad from the engine's input activation and captured dy; dgrad dx, plain or in the block-gradient form
    (dgrad + skip) * mask; a compact (stride-2 sub-grid) dx is compared on that sub-grid."""
    ref, ab = conv_dgrad(dy, conv, x.shape)
    e = UM * gemm_depth(conv.weight.shape[0] * conv.weight[0, 0].numel()) * ab
    if skip is not None:
        ref = (ref + skip) * mask.view(ref.shape)
        e = (e + U * ref.abs()) * mask.view(ref.shape)
        rep.bounded(f"{full} dx (block gradient)", dx_got, ref, bf16_bound(ref, e))
    elif dx_got.shape != ref.shape:
        ref, e = ref[:, ::2, ::2], e[:, ::2, ::2]
        rep.bounded(f"{full} dx (compact)", dx_got, ref, bf16_bound(ref, e))
    else:
        rep.bounded(f"{full} dx", dx_got, ref, bf16_bound(ref, e))
    wref, wab = conv_wgrad(x, dy, conv)
    rep.bounded(f"{full}.weight wgrad", kernel_grad(rec, full + ".weight"), wref,
                UM * rec["depth"]["wgrad"][full] * wab, param=full + ".weight")


def check_train_step(rec, model, exempt=None) -> Report:
    rep = Report(exempt)
    check_forward_train(rep, rec, model)
    check_backward(rep, rec, model)
    return rep


# ------------------------------------------------------------------------------------------------ inference
def check_inference(rec, model) -> Report:
    """The fused-epilogue inference build: BatchNorm from running statistics in every conv epilogue."""
    rep = Report()
    A = rec["act"]
    ref, ab = conv_fwd_stem(rec, model)
    rep.bounded("conv1 y", rec["y0"], ref, bf16_bound(ref, UM * gemm_depth(192) * ab))

    def eval_affine(bn, mod):
        w = rec["bnw"][bn]
        rm, rv = (t.double() for t in rec["run_before"][bn])
        g, b = rec["gamma"][bn].double(), rec["beta"][bn].double()
        sc = g * (rv + mod.eps).rsqrt()
        d_sc = 7 * U * sc.abs()   # var + eps, rsqrtf (2 ulp), gamma * invstd
        rep.bounded(f"{bn} scale", w["scale"], sc, d_sc)
        sh = b - rm * sc
        rep.bounded(f"{bn} shift", w["shift"], sh, rm.abs() * d_sc + 2 * U * (b.abs() + (rm * sc).abs()))
        return w["scale"].double(), w["shift"].double()

    eval_affine("bn1", model.bn1)
    check_stem_pool(rep, rec, "maxpool")
    x_in = rec["p0"]
    for name, blk in blocks(model):
        def epi(c, bn, x, res=None, relu=True):
            conv = getattr(blk, c) if isinstance(c, str) else c
            sc, sh = eval_affine(bn, getattr(blk, bn.split(".", 2)[-1]) if "downsample" not in bn else blk.downsample[1])
            acc, ab = conv_fwd(x, conv)
            v = flat(acc) * sc + sh
            e = sc.abs() * flat(ab) * UM * gemm_depth(conv.weight[0].numel()) + U * v.abs()
            if res is not None:
                v = v + flat(res)
                e = e + U * v.abs()
            ref = v.clamp(min=0) if relu else v
            return ref, e

        for c, bn, x, a in (("conv1", "bn1", x_in, "a1"), ("conv2", "bn2", A[name + ".a1"], "a2")):
            ref, e = epi(c, f"{name}.{bn}", x)
            rep.bounded(f"{name}.{c}+{bn} {a}", flat(A[f"{name}.{a}"]), ref, bf16_bound(ref, e))
        res = x_in
        if blk.downsample is not None:
            ref, e = epi(blk.downsample[0], f"{name}.downsample.1", x_in, relu=False)
            rep.bounded(f"{name}.downsample yd", flat(A[name + ".yd"]), ref, bf16_bound(ref, e))
            res = A[name + ".yd"]
        ref, e = epi("conv3", f"{name}.bn3", A[name + ".a2"], res=res)
        rep.bounded(f"{name}.conv3+bn3 out", flat(A[name + ".out"]), ref, bf16_bound(ref, e))
        x_in = A[name + ".out"]
    check_head(rep, rec, model)
    run_ok = all(torch.equal(rec["run_after"][bn][k], rec["run_before"][bn][k]) for bn in rec["bnw"] for k in (0, 1))
    rep.equal("running statistics", run_ok, "an inference forward changed the running statistics")
    return rep


# ------------------------------------------------------------------------------------------------ engine + capture
def _batch():
    g = torch.Generator(device="cpu").manual_seed(2)
    x = torch.randint(0, 256, (N_BATCH, SIZE, SIZE, 3), generator=g, dtype=torch.uint8)
    y = torch.randint(0, CLASSES, (N_BATCH,), generator=g)
    return x.to(DEV), y.to(DEV)


def _engine(training=True, **kw):
    """Batch 8 at 224 x 224, 10 classes; every gamma, beta and running statistic random (every residual branch carries
    gradient and the running update is visible); no dropout, no augmentation."""
    import b200ddl  # noqa: F401
    from b200ddl.models.resnet_engine import ResNet50Engine

    eng = ResNet50Engine(batch=N_BATCH, num_classes=CLASSES, image_size=SIZE, seed=0, dropout=0.0,
                         zero_init_residual=False, **kw)
    g = torch.Generator(device="cpu").manual_seed(1)
    for n in eng.bn_names:
        c = eng.bn_channels[n]
        eng.p(n + ".weight").copy_(torch.rand(c, generator=g) + 0.5)
        eng.p(n + ".bias").copy_(torch.randn(c, generator=g) * 0.3)
        eng.running_mean[n].copy_(torch.randn(c, generator=g) * 0.2)
        eng.running_var[n].copy_(torch.rand(c, generator=g) + 0.5)
    eng.build(training=training)
    eng.sync_weights()
    eng.set_input(*_batch())
    return eng


def _oracle(eng):
    """torchvision ResNet-50 in float64 with the engine's parameters (conv and FC filters rounded to bf16, as the
    engine's GEMMs read them) and its running statistics before the step."""
    import torchvision

    sd = eng.state_dict()
    for k, v in sd.items():
        if k.endswith(".weight") and v.dim() > 1:
            sd[k] = v.to(torch.bfloat16)
    model = torchvision.models.resnet50(num_classes=eng.num_classes)
    missing, unexpected = model.load_state_dict({k: v.double() for k, v in sd.items()}, strict=False)
    assert not unexpected and all(k.endswith("num_batches_tracked") for k in missing), (missing, unexpected)
    return model.double().to(DEV)


def _col_reduce_depth(M, C_):
    """elementwise.cu col_reduce_kernel: a thread's row partial, the shared-memory sum over row lanes, one atomic per block."""
    blocks = max(1, min(-(-M // 32), 132 * 8))
    rpb = 256 // min(C_ // 8, 256)
    return -(-(-(-M // blocks)) // rpb) + rpb + blocks


def _epilogue_depth(plans, C_):
    """conv_igemm statistics epilogue: 15 + 1 in a thread's 16-row partials, one register addition per tile of the
    column's n-block, 8 row-group atomics per flush (at most one flush per tile)."""
    tiles = sum(p.tiles for p in plans)
    n_blocks = max(1, -(-C_ // plans[0].block_n))
    return 17 + 9 * -(-tiles // n_blocks)


def _wgrad_depth(px, plan):
    """conv_wgrad: k16 MMAs over one pixel chunk (at most one box of 128 pixels more than an even share), <= 16 inside
    an MMA, one atomic flush per chunk."""
    return -(-(-(-px // plan.px_chunks) + 128) // 16) + 16 + plan.px_chunks


def _depths(eng):
    from b200ddl.ops.conv import sm_count

    N = eng.batch
    H0 = eng.y0.shape[1]
    fwd, bwd, wg = {}, {}, {}
    tiles0 = N * H0
    grid0 = min(tiles0, sm_count())
    # stem statistics: <= 15 in a thread's partial, 8 shared-memory row groups per tile of the CTA, one global atomic
    # per CTA
    fwd["bn1"] = 16 + 8 * -(-tiles0 // grid0) + grid0 if eng.native_stem else _col_reduce_depth(N * H0 * H0, 64)
    if eng.fuse_stem_bwd and not eng.fuse_bn_coeffs:
        tiles = N * (H0 // 16) ** 2      # stem_pool_bn_bwd: 16 x 16-pixel tiles, 8 pixels per thread per tile
        grid = min(132 * 3, tiles)
        bwd["bn1"] = 8 * -(-tiles // grid) + 2 + 8 + grid
    else:
        bwd["bn1"] = _col_reduce_depth(N * H0 * H0, 64)
    wg["conv1"] = 8 * -(-tiles0 // grid0) + 16 + grid0   # stem wgrad: 128-pixel tiles (8 k16 steps), one flush per CTA
    wg["fc"] = _wgrad_depth(N, eng._fc_wg.plan)
    for bi, b in enumerate(eng.blocks):
        n = b.name
        for c, bn in (("conv1", "bn1"), ("conv2", "bn2"), ("conv3", "bn3"), ("downsample.0", "downsample.1")):
            if c == "downsample.0" and not b.downsample:
                continue
            full, bname = f"{n}.{c}", f"{n}.{bn}"
            C_ = eng.bn_channels[bname]
            fwd[bname] = _epilogue_depth([eng._fwd[full].plan], C_)
            px = N * (b.h_out if c != "conv1" else b.h_in) ** 2
            wg[full] = _wgrad_depth(px, eng._wg[full].plan)
            M = N * (b.h_in if c == "conv1" else b.h_out) ** 2
            if bname in eng._fused_reduce:
                src = eng._dg[f"{n}.conv2" if bn == "bn1" else f"{n}.conv3"]
                bwd[bname] = _epilogue_depth([p for p, _, _ in src.parts], C_)
            elif bname in eng._block_fused:
                src = eng._dg[f"{eng.blocks[bi + 1].name}.conv1"]
                bwd[bname] = _epilogue_depth([p for p, _, _ in src.parts], C_)
            else:
                bwd[bname] = _col_reduce_depth(M, C_)
    return dict(fwd=fwd, bwd=bwd, wgrad=wg)


def _clone(t):
    return None if t is None else t.clone()


def _common_record(eng):
    rec = dict(
        act={k: v.clone() for k, v in eng.act.items()},
        y0=eng.y0.clone(), p0=eng.p0.clone(), pool_idx=eng.pool_idx.clone(), pooled=eng.pooled.clone(),
        logits16=eng.logits16.clone(), logits=eng.logits.clone(), loss_rows=eng.loss_rows.clone(),
        labels=eng.labels.clone(), x_stem=stem_input(eng.x_u8), native_stem=eng.native_stem,
        bnw={bn: {k: eng.bnw[bn][k].clone() for k in ("mean", "invstd", "scale", "shift")} for bn in eng.bn_names},
        gamma={bn: eng.p(bn + ".weight").clone() for bn in eng.bn_names},
        beta={bn: eng.p(bn + ".bias").clone() for bn in eng.bn_names},
        run_after={bn: (eng.running_mean[bn].clone(), eng.running_var[bn].clone()) for bn in eng.bn_names},
    )
    rec["out"] = {b.name: rec["act"][b.name + ".out"] for b in eng.blocks}
    return rec


def run_train_step(eng):
    """One eager training step (forward + backward, no optimizer) with the backward intermediates captured: every
    BatchNorm's incoming gradient (before its backward) and dy / dz (after), every conv's dgrad output."""
    run_before = {bn: (eng.running_mean[bn].clone(), eng.running_var[bn].clone()) for bn in eng.bn_names}
    bwd, dx = {}, {}
    bn_bwd, conv_bwd = eng._bn_bwd, eng._conv_bwd

    def cap_bn_bwd(bn, mode, g1, g2, out, y, dy, dz, count):
        r = dict(g1=_clone(g1), g2=_clone(g2))
        bn_bwd(bn, mode, g1, g2, out, y, dy, dz, count)
        r.update(dy=dy.clone(), dz=_clone(dz))
        bwd[bn] = r

    def cap_conv_bwd(full, cname):
        conv_bwd(full, cname)
        dx[full] = eng._dg[full].dx.clone()

    eng._bn_bwd, eng._conv_bwd = cap_bn_bwd, cap_conv_bwd
    try:
        eng.forward(training=True)
        eng.backward()
    finally:
        del eng._bn_bwd, eng._conv_bwd
    torch.cuda.synchronize()
    rec = _common_record(eng)
    rec.update(
        run_before=run_before, bwd=bwd, dx=dx, block_fused=set(eng._block_fused),
        dlogits16=eng.dlogits16.clone(), dpooled=eng.dpooled.clone(),
        dy0=eng._scr["dzA"][:eng.y0.numel()].view(eng.y0.shape).clone(),
        grads={s.name: eng.g(s.name).clone() for s in eng.param_specs},
        depth=_depths(eng),
    )
    return rec


def _fail_report(rep, title):
    rep.print(title)
    assert not rep.failures, f"{title}: {len(rep.failures)} failures\n" + "\n".join(rep.failures[:40])


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("path", list(PATHS))
def test_train_step_matches_float64_per_layer(path, monkeypatch):
    kw, env = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = _engine(**kw)
    model = _oracle(eng)
    rec = run_train_step(eng)
    rep = check_train_step(rec, model, TORCH_STEM_EXEMPT if path == "torch_stem" else None)
    _fail_report(rep, f"train step [{path}]")
    assert rep.params == {s.name for s in eng.param_specs}, sorted({s.name for s in eng.param_specs} ^ rep.params)
    assert len(rep.params) == 161
    n_bn = {k.rsplit(" ", 1)[0] for k, *_ in rep.rows if k.endswith(" running_var")}
    assert len(n_bn) == 53, len(n_bn)


def test_inference_build_matches_float64_per_layer():
    eng = _engine(training=False)
    assert eng._infer_fused, "the inference build did not take the fused-epilogue path"
    model = _oracle(eng)
    run_before = {bn: (eng.running_mean[bn].clone(), eng.running_var[bn].clone()) for bn in eng.bn_names}
    eng.forward(training=False)
    torch.cuda.synchronize()
    rec = _common_record(eng)
    rec["run_before"] = run_before
    _fail_report(check_inference(rec, model), "inference build")


def test_checker_reports_corruptions():
    """One clean step, then five corruptions of its captured results; the checker must name each corrupted layer."""
    eng = _engine()
    model = _oracle(eng)
    rec = run_train_step(eng)
    clean = check_train_step(rec, model)
    _fail_report(clean, "clean step")

    def with_(**parts):
        r = dict(rec)
        for k, v in parts.items():
            r[k] = v
        return r

    cases = []
    # 1. one mid-network dgamma scaled by 1 + 2^-6
    g = dict(rec["grads"])
    g["layer3.3.bn2.weight"] = g["layer3.3.bn2.weight"] * (1 + 2.0 ** -6)
    cases.append(("dgamma x (1 + 2^-6)", with_(grads=g), "layer3.3.bn2 dgamma"))
    # 2. the wgrads of two equal-shape convs swapped
    g = dict(rec["grads"])
    g["layer3.1.conv2.weight"], g["layer3.2.conv2.weight"] = g["layer3.2.conv2.weight"], g["layer3.1.conv2.weight"]
    cases.append(("swapped wgrads", with_(grads=g), "layer3.2.conv2.weight wgrad"))
    # 3. bn2's backward computed with the previous block's y2 (what a mis-wired y pointer produces)
    bn = "layer3.2.bn2"
    cb = rec["bwd"][bn]
    y_wrong = rec["act"]["layer3.1.y2"]
    v, _ = bn_pre(rec, bn, y_wrong)
    dz = flat(cb["g1"]) * (v > 0)
    w = rec["bnw"][bn]
    r = bn_bwd_ref(dz, dz, y_wrong, w["mean"], w["invstd"], rec["gamma"][bn], 1)
    g = dict(rec["grads"])
    g[bn + ".weight"], g[bn + ".bias"] = r["dgamma"].float(), r["dbeta"].float()
    bwd = dict(rec["bwd"])
    bwd[bn] = dict(cb, dy=r["dy"].view(cb["dy"].shape).to(torch.bfloat16))
    cases.append(("previous block's y2 in bn2 backward", with_(grads=g, bwd=bwd), "layer3.2.bn2 dy"))
    # 4. the running variance updated with the biased batch variance
    bn = "layer4.2.bn2"
    M, mean, var, _, _ = stats_ref(rec["act"]["layer4.2.y2"], 1)
    rm1, rv1 = rec["run_after"][bn]
    rv0 = rec["run_before"][bn][1].double()
    ra = dict(rec["run_after"])
    ra[bn] = (rm1, ((1 - 0.1) * rv0 + 0.1 * var).float())
    cases.append(("biased running variance", with_(run_after=ra), "layer4.2.bn2 running_var"))
    # 5. one channel of one dgrad dx shifted by one bf16 ulp at 1 % of its pixels
    full = "layer2.1.conv2"
    d = rec["dx"][full].clone()
    gen = torch.Generator(device=DEV).manual_seed(5)
    pick = (torch.rand(d.shape[:-1], device=DEV, generator=gen) < 0.01) & (d[..., 7] != 0)
    col = d[..., 7].contiguous()
    bits = col.view(torch.int16)
    bits[pick] += 1
    d[..., 7] = col
    dxs = dict(rec["dx"])
    dxs[full] = d
    cases.append(("one bf16 ulp in 1 % of one channel", with_(dx=dxs), "layer2.1.conv2 dx"))

    for what, r, key in cases:
        rep = check_train_step(r, model)
        hit = [f for f in rep.failures if f.startswith(key)]
        print(f"{what}: {len(rep.failures)} failures, e.g. {rep.failures[:1]}")
        assert hit, f"{what}: the checker did not report {key!r}; failures: {rep.failures[:5]}"
