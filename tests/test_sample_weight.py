"""Keras loss weighting on the GPU: the weighted instantiations of softmax_ce_head, softmax_ce_soft_head and
softmax_kd_head (csrc/head_stem.cu) against their unweighted kernels and the float64 head references, and the native
engines' class-weighted training steps, launch profiles, graph capture rule and weighted evaluation."""
from __future__ import annotations

import pytest
import torch

from exact_util import DEV, U, check_equal
from test_distill import _mix, kd_bounds
from test_elementwise_exact import BF, NAN, bf, check_bound, f32, head_data
from test_mix import soft_bounds

pytestmark = pytest.mark.gpu

HEADS = ["ce", "soft", "kd"]


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


class _Head:
    """One head's inputs (bf16 logits with NaN padding, bias, labels, mix rows, a teacher for kd) and a launcher that
    returns its four outputs [logits32, dlogits16, loss_rows, stats]."""

    def __init__(self, kind, K, B, seed):
        g = gen(seed)
        self.kind, self.K, self.B, self.ld = kind, K, B, (K + 63) // 64 * 64 + 64
        l16, self.bias, self.labels = head_data(B, K, g)
        t16, self.tbias, _ = head_data(B, K, g)
        self.lg16 = torch.full((B, self.ld), NAN, device=DEV, dtype=BF)
        self.lg16[:, :K] = bf(l16)
        self.tg16 = torch.full((B, K + 16), NAN, device=DEV, dtype=BF)
        self.tg16[:, :K] = bf(t16)
        self.logit, self.tlogit = (l16 + self.bias).float().double(), (t16 + self.tbias).float().double()
        self.mix = None if kind == "ce" else _mix("mixup", B)
        self.eps = 0.0 if kind == "ce" else 0.1
        self.gs = 1.0 / 256

    def target(self):
        from b200ddl.models.augment import target_argmax

        return target_argmax(self.labels, self.mix)

    def run(self, **weights):
        e, B, K = _ops(), self.B, self.K
        out = [torch.full((B, K), NAN, device=DEV), torch.full((B, self.ld), NAN, device=DEV, dtype=BF),
               torch.full((B,), NAN, device=DEV), torch.zeros(4 if self.kind == "kd" else 2, device=DEV)]
        if self.kind == "ce":
            e.softmax_ce_head(self.lg16, f32(self.bias), self.labels, *out, self.gs, **weights)
        elif self.kind == "soft":
            e.softmax_ce_soft_head(self.lg16, f32(self.bias), self.labels, self.mix, self.eps, *out, self.gs, **weights)
        else:
            e.softmax_kd_head(self.lg16, f32(self.bias), self.tg16, f32(self.tbias), self.labels, self.mix, self.eps,
                              0.3, 3.0, *out, self.gs, **weights)
        torch.cuda.synchronize()
        return out

    def reference(self):
        """float64 per-row loss and bound, dlogits and bound (+ the kd head's two terms and bounds)."""
        if self.kind == "kd":
            return kd_bounds(self.logit, self.tlogit, self.labels, self.mix, self.eps, 0.3, 3.0, self.gs)
        return soft_bounds(self.logit, self.labels, self.mix, self.eps, self.gs)


def _both_ways(h, w_rows):
    """The weighted head run with w_rows as the class table (read at each row's target class) and as row weights."""
    table = torch.ones(h.K, device=DEV)
    tgt = h.target()
    table[tgt] = w_rows   # rows of one target class share one weight by construction of w_rows
    assert torch.equal(table[tgt], w_rows)
    return {"class": h.run(class_weight=table), "row": h.run(row_weight=w_rows)}


def _class_consistent(h, w_of_class):
    return w_of_class[h.target()]


@pytest.mark.parametrize("B", [64, 37])
@pytest.mark.parametrize("K", [5, 1000])
@pytest.mark.parametrize("kind", HEADS)
def test_all_ones_is_the_unweighted_kernel_bit_for_bit(kind, K, B):
    h = _Head(kind, K, B, seed=K + B)
    plain = h.run()
    for how, out in _both_ways(h, torch.ones(B, device=DEV)).items():
        for nm, a, b in zip(("logits32", "dlogits16", "loss_rows", "stats"), out, plain):
            if nm == "stats":   # fp32 atomics: the sum order varies between launches; the count is exact
                assert float(a[1]) == float(b[1])
                check_bound(f"{kind} {how} K={K} B={B} loss sum", a[:1], b[:1].double(),
                            (B * U * plain[2].double().abs().sum()).view(1))
            else:
                check_equal(f"{kind} {how} K={K} B={B} {nm}", a, b)


@pytest.mark.parametrize("B", [64, 37])
@pytest.mark.parametrize("K", [5, 1000])
@pytest.mark.parametrize("kind", HEADS)
def test_power_of_two_weights_scale_exactly(kind, K, B):
    """w in {0, 1/4, 1/2, 1, 2, 4} per class: logits32 is untouched, every loss row and dlogit is exactly the unweighted
    one times w (a product by a power of two is exact, and so is its bf16 rounding) - except that fast math flushes a
    product below 2^-126 to zero - the count is unweighted and the loss sums are the float64 sums of those rows within
    the fp32 summation bound."""

    def times(v, w):
        p = v.float() * w
        return torch.where(p.abs() < 2.0 ** -126, torch.zeros_like(p), p)

    h = _Head(kind, K, B, seed=3 * K + B)
    plain = h.run()
    pow2 = torch.tensor([0.0, 0.25, 0.5, 1.0, 2.0, 4.0], device=DEV)
    w = _class_consistent(h, pow2[torch.arange(K, device=DEV) % 6])
    for how, out in _both_ways(h, w).items():
        name = f"{kind} {how} K={K} B={B}"
        check_equal(name + " logits32", out[0], plain[0])
        exp = times(plain[1], w[:, None])
        # bf16(d) w exactly 2^-126: the fp32 d w the kernel formed may lie just below it and flush to zero
        edge = (exp.abs() == 2.0 ** -126) & (out[1].float() == 0)
        check_equal(name + " dlogits16", torch.where(edge, exp, out[1].float()).to(BF), exp.to(BF))
        check_equal(name + " loss_rows", out[2], times(plain[2], w))
        assert float(out[3][1]) == float(plain[3][1]), name + " count"
        rows = plain[2].double() * w.double()
        check_bound(name + " loss sum", out[3][:1], rows.sum().view(1), (B * U * rows.abs().sum()).view(1))


@pytest.mark.parametrize("B", [64, 37])
@pytest.mark.parametrize("K", [5, 1000])
@pytest.mark.parametrize("kind", HEADS)
def test_arbitrary_weights_within_the_float64_bounds(kind, K, B):
    """Random weights in [0, 3), as a class table and as row weights: the head references' bounds scaled by w, plus one
    rounding of the product (and the bf16 rounding of the weighted dlogit)."""
    h = _Head(kind, K, B, seed=5 * K + B)
    ref = h.reference()
    loss, lb, d, db = (ref[0], ref[1], ref[-2], ref[-1])
    w_cls = torch.rand(K, device=DEV, generator=gen(K)) * 3
    w = _class_consistent(h, w_cls).double()
    for how, out in _both_ways(h, w.float()).items():
        name = f"{kind} {how} K={K} B={B}"
        lw, lwb = loss * w, lb * w + U * (loss.abs() + lb) * w
        check_bound(name + " loss_rows", out[2], lw, lwb)
        check_bound(name + " loss sum", out[3][:1], lw.sum().view(1), (lwb.sum() + B * U * lw.abs().sum()).view(1))
        dw, dwb = d * w[:, None], db * w[:, None]
        # + 2^-126: fast math flushes a weighted dlogit below the smallest normal to zero
        check_bound(name + " dlogits", out[1][:, :K], dw,
                    dwb + U * (dw.abs() + dwb) + 2.0 ** -8 * (dw.abs() + 2 * dwb) + 2.0 ** -126)
        check_equal(name + " padded dlogits", out[1][:, K:], torch.zeros(B, h.ld - K, device=DEV))
        if kind == "kd":
            for i, (t, tb) in enumerate(((ref[2], ref[3]), (ref[4], ref[5]))):
                tw, twb = t * w, tb * w + U * (t.abs() + tb) * w
                check_bound(f"{name} term {i} sum", out[3][2 + i:3 + i], tw.sum().view(1),
                            (twb.sum() + B * U * tw.abs().sum()).view(1))


def test_binding_checks():
    h = _Head("ce", 5, 8, seed=1)
    for bad in (dict(class_weight=torch.ones(5, device=DEV), row_weight=torch.ones(8, device=DEV)),
                dict(class_weight=torch.ones(4, device=DEV)), dict(row_weight=torch.ones(9, device=DEV)),
                dict(row_weight=torch.ones(8, device=DEV, dtype=torch.float64)), dict(class_weight=torch.ones(5))):
        with pytest.raises(RuntimeError):
            h.run(**bad)


# ================================================================================================ engines
N_ENG, S_ENG, K_ENG = 16, 224, 5
ENGINES = [("resnet50", 17), ("mobilenetv2", None)]
IDS = ["resnet50-ft17", "mobilenetv2-frozen"]


def _engine(arch, k):
    if arch == "resnet50":
        from b200ddl.models.resnet_engine import ResNet50Engine

        return ResNet50Engine(batch=N_ENG, num_classes=K_ENG, image_size=S_ENG, seed=0, fine_tune_at=k)
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    return MobileNetV2Engine(batch=N_ENG, num_classes=K_ENG, image_size=S_ENG, dropout=0.0, seed=0, fine_tune_at=k)


def _batch(seed=1):
    g = gen(seed)
    x = torch.randint(0, 256, (N_ENG, S_ENG, S_ENG, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.arange(N_ENG, device=DEV) % K_ENG
    return x, y[torch.randperm(N_ENG, device=DEV, generator=g)]


def _check_fc_grads(eng, y, w, name):
    """The FC weight / bias gradients of the step just run against float64 (1/N) sum_n w_n dl_n built from the engine's
    own logits and pooled features.  Bounds: bf16 rounding of each dlogit (2^-8 relative, doubled for the softmax) and
    the fp32 sums."""
    N, K = eng.batch, eng.num_classes
    logits = eng.logits.double()
    d = (torch.softmax(logits, 1) - torch.nn.functional.one_hot(y, K).double()) * w.double()[:, None] / N
    x = eng.pooled.double()
    C = x.shape[1]
    ref_w, bnd_w = d.t() @ x, 2.0 ** -7 * (d.abs().t() @ x.abs()) + 1e-6
    ref_b, bnd_b = d.sum(0), 2.0 ** -7 * d.abs().sum(0) + 1e-6
    check_bound(name + " fc.weight grad", eng.g("fc.weight").view(-1, C)[:K], ref_w, bnd_w)
    check_bound(name + " fc.bias grad", eng.g("fc.bias").view(-1)[:K], ref_b, bnd_b)
    zero = w == 0
    if bool(zero.any()):
        assert bool((eng.dlogits16[zero] == 0).all()), name + ": a weight-0 row has a non-zero dlogit"


@pytest.mark.parametrize("arch,k", ENGINES, ids=IDS)
def test_class_weighted_graphed_step(arch, k):
    """One graphed step with class_weight: FC gradients against the float64 reference; rows of the weight-0 class have
    exactly zero dlogits."""
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    eng = _engine(arch, k)
    table = torch.tensor([0.0, 2.0, 0.5, 1.0, 3.25])
    eng.set_weighting("class")
    eng.set_class_weight(table)
    step = EngineTrainStep(eng, optim.SGD(0.0))
    x, y = _batch()
    step.load(x, y)
    step.run()
    torch.cuda.synchronize()
    assert step.graph is not None
    _check_fc_grads(eng, y, table.to(DEV)[y], f"{arch} k={k}")


def _kernel_names(step):
    step.run()   # eager warm-up (use_graph=False)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step.run()
        torch.cuda.synchronize()
    return [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
            and "emcpy" not in ev.name and "emset" not in ev.name]


@pytest.mark.parametrize("arch,k", ENGINES, ids=IDS)
def test_launch_profile(arch, k):
    """An unweighted step launches the unweighted head and, after a weighted phase, exactly the same kernel sequence
    again; a weighted step (class or sample) swaps the head for its weighted instantiation and nothing else."""
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    eng = _engine(arch, k)
    step = EngineTrainStep(eng, optim.SGD(0.0), use_graph=False)
    x, y = _batch()
    step.load(x, y)
    plain = _kernel_names(step)
    heads = [i for i, n in enumerate(plain) if "softmax_ce_head_kernel" in n]
    assert len(heads) == 1 and "softmax_ce_head_kernel<false>" in plain[heads[0]]
    for mode in ("class", "sample"):
        eng.set_weighting(mode)
        step.load(x, y, torch.ones(N_ENG, device=DEV))
        got = _kernel_names(step)
        want = list(plain)
        want[heads[0]] = plain[heads[0]].replace("softmax_ce_head_kernel<false>", "softmax_ce_head_kernel<true>")
        assert got == want, mode
    eng.set_weighting(None)
    assert _kernel_names(step) == plain


@pytest.mark.parametrize("arch,k", ENGINES, ids=IDS)
def test_capture_rule(arch, k):
    """Trainer.fit: a new class_weight with the mode unchanged reuses the captured graph; weighted -> unweighted ->
    weighted captures again at each change, and every phase matches its own reference."""
    from b200ddl import optim
    from b200ddl.train import Trainer

    eng = _engine(arch, k)
    tr = Trainer(eng).compile(optim.SGD(0.0))
    x, y = _batch()
    ones = torch.ones(K_ENG)
    phases = [({0: 2.0, 3: 0.0}, True), ({1: 0.25, 4: 4.0}, False), (None, True), ({0: 2.0, 3: 0.0}, True)]
    graph = None
    for cw, recapture in phases:
        tr.fit([(x, y)], epochs=1, verbose=0, class_weight=cw)
        g = tr.backend.step.graph
        assert (g is not graph) == recapture, (cw, recapture)
        graph = g
        table = ones.clone()
        for c, v in (cw or {}).items():
            table[c] = v
        _check_fc_grads(eng, y, table.to(DEV)[y], f"{arch} class_weight={cw}")


@pytest.mark.parametrize("arch,k", ENGINES, ids=IDS)
def test_evaluate_weights_loss_not_accuracy(arch, k):
    from b200ddl import optim
    from b200ddl.train import Trainer

    eng = _engine(arch, k)
    tr = Trainer(eng).compile(optim.SGD(0.0))
    x, y = _batch()
    w = torch.linspace(0.0, 3.0, N_ENG, device=DEV)
    for batch, weights in (((x, y, w), w), ((x, y), torch.ones(N_ENG, device=DEV))):
        loss, acc = tr.evaluate([batch])
        logits = eng.logits.double()
        rows = torch.logsumexp(logits, 1) - logits.gather(1, y[:, None]).squeeze(1)
        assert loss == pytest.approx(float((rows * weights.double()).mean()), rel=1e-5, abs=1e-6)
        assert acc == float((logits.argmax(1) == y).double().mean())
