"""ResNet-50 fine-tuning on the native engine (`ResNet50Engine(fine_tune_at=k, batchnorm=...)`), on the GPU."""
from __future__ import annotations

import pytest
import torch
import torch.nn.functional as F

from exact_util import DEV

pytestmark = pytest.mark.gpu

B = 8
FREE = dict(zero_init_residual=False)   # every trainable tensor gets a gradient from the first step on


def _engine(k=None, mode="inference", batch=B, dropout=0.0, **kw):
    from b200ddl.models.resnet_engine import ResNet50Engine

    return ResNet50Engine(batch=batch, num_classes=5, seed=0, dropout=dropout, fine_tune_at=k,
                          batchnorm=mode if k is not None else "inference", **{**FREE, **kw})


def _batch(seed, batch=B, size=224):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randint(0, 256, (batch, size, size, 3), device=DEV, dtype=torch.uint8, generator=g)
    return x, torch.randint(0, 5, (batch,), device=DEV, generator=g)


def _randomise_running(eng, seed=3):
    """Non-trivial running statistics (a fresh engine has mean 0 / var 1)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    tot = eng.running.numel() // 2
    eng.running[:tot].copy_(torch.randn(tot, device=DEV, generator=g) * 0.1)
    eng.running[tot:].copy_(torch.rand(tot, device=DEV, generator=g) + 0.5)
    eng.sync_weights()


# ================================================================================================ kernel
@pytest.mark.parametrize("C", [64, 200, 2048])
def test_bn_bwd_coeffs_inference(C):
    """dgamma = invstd * (sum_dzy - mean * sum_dz), dbeta = sum_dz, A = gamma * invstd, B = C = 0; sums zeroed.  Each
    output is one or two fp32 roundings of the float64 value (|rel err| <= 2 * 2^-24 + 2^-24 for dgamma: a product of a
    rounded difference of two rounded products)."""
    from b200ddl import ops

    e = ops.ext("_b200_ops")
    g = torch.Generator(device=DEV).manual_seed(C)
    r = lambda: torch.randn(C, device=DEV, generator=g, dtype=torch.float64)
    sdz, sdzy, gamma, mean, invstd = r(), r(), r(), r(), r().abs() + 0.1
    f = lambda t: t.float().contiguous()
    s0, s1 = f(sdz), f(sdzy)
    outs = [torch.full((C,), float("nan"), device=DEV) for _ in range(5)]
    e.bn_bwd_coeffs(s0, s1, f(gamma), f(mean), f(invstd), 1234.0, *outs, inference=True)
    torch.cuda.synchronize()
    d = lambda t: t.float().double()
    sdz, sdzy, gamma, mean, invstd = map(d, (sdz, sdzy, gamma, mean, invstd))
    dg_ref = invstd * (sdzy - mean * sdz)
    eps = 2.0 ** -24
    bound_dg = 3 * eps * invstd * (sdzy.abs() + (mean * sdz).abs()) + 1e-30
    assert ((outs[0].double() - dg_ref).abs() <= bound_dg).all()
    assert torch.equal(outs[1].double(), sdz)
    assert ((outs[2].double() - gamma * invstd).abs() <= eps * (gamma * invstd).abs()).all()
    assert torch.equal(outs[3], torch.zeros_like(outs[3])) and torch.equal(outs[4], torch.zeros_like(outs[4]))
    assert torch.equal(s0, torch.zeros_like(s0)) and torch.equal(s1, torch.zeros_like(s1))
    # the training-mode call is unchanged by the new argument
    a = [torch.zeros(C, device=DEV) for _ in range(5)]
    b = [torch.zeros(C, device=DEV) for _ in range(5)]
    args = (f(gamma), f(mean), f(invstd), 77.0)
    e.bn_bwd_coeffs(f(sdz), f(sdzy), *args, *a)
    e.bn_bwd_coeffs(f(sdz), f(sdzy), *args, *b, inference=False)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_bn_bwd_coeffs_rejects_bad_operands():
    from b200ddl import ops

    e = ops.ext("_b200_ops")
    C = 64
    f = lambda n=C: torch.zeros(n, device=DEV)
    before = ops.kernel_launches()
    for bad in (lambda: e.bn_bwd_coeffs(f(), f(), f(), f(), f(), 1.0, f(), f(), f(C - 8), f(), f(), inference=True),
                lambda: e.bn_bwd_coeffs(f(), f(), f().bfloat16(), f(), f(), 1.0, f(), f(), f(), f(), f(), inference=True),
                lambda: e.bn_bwd_coeffs(f(), f(), f(), f(), f().cpu(), 1.0, f(), f(), f(), f(), f(), inference=True)):
        with pytest.raises(RuntimeError):
            bad()
    assert ops.kernel_launches() == before


def test_engine_rejects_training_mode_fusions():
    with pytest.raises(ValueError):
        _engine(8, "inference", fuse_bn_coeffs=True)
    with pytest.raises(ValueError):
        _engine(0, "inference", fuse_stem_bwd=True)
    _engine(8, "training", fuse_bn_coeffs=True)


# ================================================================================================ k = 0, training = today
def _kernel_names(eng, opt):
    from b200ddl.models.resnet_engine import EngineTrainStep

    step = EngineTrainStep(eng, opt, use_graph=False)
    x, y = _batch(1)
    step.load(x, y)
    step.run()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step.run()
        torch.cuda.synchronize()
    return [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
            and "emcpy" not in ev.name and "emset" not in ev.name]


def test_k0_training_is_the_full_engine():
    """fine_tune_at=0 with training-mode BatchNorm launches exactly the fully trainable engine's kernels, and after 3
    graph steps its parameters, running statistics and losses are as close to the full engine's as runs of the full
    engine are to each other.  The weight-gradient GEMMs and the statistics epilogues add fp32 partial sums with
    atomics, so runs differ in the last bits, by an amount that varies several-fold from pair to pair (two runs
    sometimes agree almost exactly): a single pair is no yardstick.  The candidate's mean distance to four full-engine
    runs is compared with the mean distance over their six pairs."""
    import itertools

    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    def run(k):
        eng = _engine(k, "training", zero_init_residual=True)
        step = EngineTrainStep(eng, optim.SGD(0.1, momentum=0.9), use_graph=True)
        losses = []
        for i in range(3):
            step.load(*_batch(10 + i))
            step.run()
            losses.append(step.result()[0])
        assert eng.arch == ("resnet50" if k is None else "resnet50_head")
        return [eng.params.double(), eng.running.double(), torch.tensor(losses, dtype=torch.float64)]

    refs = [run(None) for _ in range(4)]
    cand = run(0)
    pairs = list(itertools.combinations(range(len(refs)), 2))

    def rel(a, b):
        return float((a - b).norm() / b.norm())

    for i, what in enumerate(("params", "running statistics", "losses")):
        spread = sum(rel(refs[b][i], refs[a][i]) for a, b in pairs) / len(pairs)
        diff = sum(rel(cand[i], r[i]) for r in refs) / len(refs)
        assert diff <= max(4 * spread, 1e-6), f"{what}: k = 0 vs full {diff}, full runs {spread}"
    a = _kernel_names(_engine(None, "training", zero_init_residual=True), optim.SGD(0.1, momentum=0.9))
    b = _kernel_names(_engine(0, "training", zero_init_residual=True), optim.SGD(0.1, momentum=0.9))
    assert a == b and len(a) > 100


# ================================================================================================ launch sets
BLOCKS = [(f"layer{s + 1}.{i}", i == 0) for s, n in enumerate((3, 4, 6, 3)) for i in range(n)]   # (name, downsample)


@pytest.mark.parametrize("k", [17, 14, 8, 4, 1, 0])
@pytest.mark.parametrize("mode", ["inference", "training"])
def test_launch_sets(k, mode):
    eng = _engine(k, mode).build(training=True)
    exp_wg, exp_dg, fused = set(), set(), set()
    for bi, (n, ds) in enumerate(BLOCKS):
        convs = ["conv1", "conv2", "conv3"] + (["downsample.0"] if ds else [])
        if bi + 1 < k:
            fused |= {f"{n}.{c}" for c in convs}
            continue
        exp_wg |= {f"{n}.{c}" for c in convs}
        exp_dg |= {f"{n}.{c}" for c in convs if c in ("conv2", "conv3") or bi + 1 > k or k == 0}
    assert set(eng._wg) == exp_wg and set(eng._dg) == exp_dg
    assert (eng._fc_dg is None) == (k == 17)
    assert (k == 0) == hasattr(eng, "_stem_wg")
    for name in fused:   # frozen blocks: fused-epilogue plans, no pre-BatchNorm activation, no mask
        blk = name.rsplit(".", 1)[0] if not name.endswith("downsample.0") else name[:-len(".downsample.0")]
        assert blk + ".y1" not in eng.act and blk + ".mask" not in eng.act and name in eng._fwd
    n_wd = len(exp_dg) + (k < 17)
    assert len(eng._wd_slices) == n_wd
    assert eng.grads.numel() == eng.trainable_numel


def _step_kernels(eng):
    from b200ddl import optim

    return _kernel_names(eng, optim.SGD(0.01, momentum=0.9))


@pytest.mark.parametrize("k", [17, 14, 4, 1, 0])
@pytest.mark.parametrize("mode", ["inference", "training"])
def test_step_launches(k, mode):
    """What one eager training step launches (torch.profiler), counted from the block table: frozen blocks run only
    fused-epilogue convolutions (conv_igemm kStats = 4) - no bn_apply, bn_finalize, backward kernel or weight gradient
    - and their running-statistics affine is not recomputed per step (bn_finalize runs for the trainable BatchNorms and
    the stem only)."""
    import re

    names = _step_kernels(_engine(k, mode))
    frozen_convs = trainable_convs = trainable_bns = trainable_blocks = 0
    for bi, (n, ds) in enumerate(BLOCKS):
        if bi + 1 < k:
            frozen_convs += 3 + ds
        else:
            trainable_convs += 3 + ds
            trainable_bns += 3 + ds
            trainable_blocks += 1

    def count(pat):
        return sum(1 for nm in names if re.search(pat, nm))

    got = dict(fused=count(r"conv_igemm_kernel<\s*\d+\s*,\s*4\s*[,>]"), wgrad=count(r"conv_wgrad_kernel"),
               bn_apply=count(r"bn_apply_kernel"), bn_finalize=count(r"bn_finalize_kernel"),
               bn_bwd_coeffs=count(r"bn_bwd_coeffs_kernel"), gap_bwd=count(r"gap_bwd_kernel"))
    want = dict(fused=frozen_convs, wgrad=trainable_convs + 1, bn_apply=3 * trainable_blocks,
                bn_finalize=trainable_bns + 1, bn_bwd_coeffs=trainable_bns + (k == 0), gap_bwd=int(k < 17))
    assert got == want, (got, want, sorted(set(names))[:40])


# ================================================================================================ logits
@pytest.mark.parametrize("k", [17, 14, 4, 0])
def test_inference_mode_train_logits_equal_eval(k):
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineEvalStep, EngineTrainStep

    eng = _engine(k, "inference")
    _randomise_running(eng)
    step = EngineTrainStep(eng, optim.SGD(0.0), use_graph=False)
    x, y = _batch(5)
    step.load(x, y)
    step.run()
    torch.cuda.synchronize()
    train_logits = eng.logits.clone()
    ev = EngineEvalStep(eng, use_graph=False)
    eng.set_input(x, y)
    ev.run()
    torch.cuda.synchronize()
    assert torch.equal(train_logits, eng.logits)
    if k == 17:
        inf = _engine(17, "inference")
        inf.load_state_dict(eng.state_dict())
        EngineEvalStep(inf, use_graph=False)
        inf.set_input(x, y)
        inf.forward(training=False)
        torch.cuda.synchronize()
        assert torch.equal(train_logits, inf.logits)


# ================================================================================================ frozen weights
OPTS = {
    "sgd": lambda o: o.SGD(0.05, momentum=0.9, nesterov=True, weight_decay=1e-4),
    "adamw": lambda o: o.AdamW(1e-3, weight_decay=0.05),
    "lamb": lambda o: o.Lamb(1e-3, weight_decay=0.01),
    "rmsprop": lambda o: o.RMSprop(1e-3, centered=True),
    "ema": lambda o: o.SGD(0.05, momentum=0.9, use_ema=True, ema_overwrite_frequency=1),
    "accum": lambda o: o.SGD(0.05, momentum=0.9, gradient_accumulation_steps=2),
    "clip": lambda o: o.SGD(0.05, momentum=0.9, global_clipnorm=0.5),
}


@pytest.mark.parametrize("opt", sorted(OPTS))
@pytest.mark.parametrize("k,mode", [(14, "inference"), (8, "training")])
def test_frozen_weights_never_change(opt, k, mode):
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    eng = _engine(k, mode, dropout=0.2)
    T = eng.trainable_numel
    p0, w0, r0 = eng.params.clone(), eng.w16.clone(), eng.running.clone()
    rm0 = {n: v.clone() for n, v in eng.running_mean.items()}
    rv0 = {n: v.clone() for n, v in eng.running_var.items()}
    step = EngineTrainStep(eng, OPTS[opt](optim), use_graph=True)
    for i in range(4):
        step.load(*_batch(20 + i))
        step.run()
    torch.cuda.synchronize()
    assert torch.equal(eng.params[T:], p0[T:]) and torch.equal(eng.w16[T:], w0[T:])
    for s in eng.trainable_specs:
        assert not torch.equal(eng.p(s.name), p0[s.offset:s.offset + s.numel].view(s.shape)), s.name
    for n in eng.bn_names:
        if eng.spec[n + ".weight"].offset >= T:   # frozen BatchNorm: running statistics bit-unchanged
            assert torch.equal(eng.running_mean[n], rm0[n]) and torch.equal(eng.running_var[n], rv0[n]), n
    if mode == "inference":
        assert torch.equal(eng.running, r0)
    else:
        assert not torch.equal(eng.running, r0)


# ================================================================================================ against the module
@pytest.mark.parametrize("k,mode", [(16, "inference"), (14, "inference"), (14, "training"), (4, "inference"),
                                    (1, "training"), (0, "inference")])
def test_gradients_match_fp32_module(k, mode):
    """One step on the same weights and batch, dropout 0: the engine's gradient of every trainable tensor against the
    fp32 torch module's, gated as the other engine-vs-module checks are (DESIGN.md 4b): the engine's relative L2
    distance to fp32 may be at most 4x the module's own distance under bf16 autocast (floor 2e-2).  bf16 rounding is
    what both distances measure; a BatchNorm backward with the wrong statistics or a missing block gradient moves whole
    tensors far past the gate."""
    from b200ddl import optim
    from b200ddl.models.resnet import ResNet50Head
    from b200ddl.models.resnet_engine import EngineTrainStep
    from b200ddl.ops.conv import weight_from_kernel_layout

    eng = _engine(k, mode)
    _randomise_running(eng)
    step = EngineTrainStep(eng, optim.SGD(0.0), use_graph=False)
    x, y = _batch(7)
    sd = {n: v.to(DEV) for n, v in eng.state_dict().items()}   # before the step moves training-mode statistics
    step.load(x, y)
    step.run()
    torch.cuda.synchronize()
    m = ResNet50Head(5, 0.0, k, mode).to(DEV)
    xin = x.permute(0, 3, 1, 2).float() / 127.5 - 1.0
    grads = {}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    for kind in ("fp32", "autocast"):
        missing = m.load_state_dict(sd, strict=False).missing_keys
        assert all(n.endswith("num_batches_tracked") for n in missing)
        m.train()
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=kind == "autocast"):
            logits = m(xin).float()
        torch.nn.functional.cross_entropy(logits, y).backward()
        grads[kind] = {n: p.grad.detach().double() for n, p in m.named_parameters() if p.requires_grad}
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    assert sorted(grads["fp32"]) == sorted(s.name for s in eng.trainable_specs)

    def rel(a, b):
        return float((a - b).norm() / b.norm().clamp_min(1e-30))

    worst = []
    for s in eng.trainable_specs:
        got = eng.g(s.name)
        if s.kind == "conv":
            r = int(round(s.shape[0] ** 0.5))
            got = weight_from_kernel_layout(got, r, r)
        elif s.kind == "fc_w":
            got = got[:5]
        ref = grads["fp32"][s.name]
        gate = max(4 * rel(grads["autocast"][s.name], ref), 2e-2)
        worst.append((rel(got.double(), ref) / gate, s.name))
    worst.sort(reverse=True)
    print("worst gradient distances (ratio to gate, name):", worst[:3])
    assert worst[0][0] <= 1.0, worst[:5]


# ================================================================================================ composition
def test_fit_with_augmentation_mixup_and_label_smoothing_lowers_loss():
    from b200ddl import optim
    from b200ddl.models import Augmentation, build_model
    from b200ddl.train import Trainer
    from b200ddl.train.losses import CategoricalCrossentropy

    aug = Augmentation(flip="horizontal", rotation=0.05, mixup=0.2)
    m = build_model(64, 64, 3, 5, dropout=0.0, arch="resnet50_head", fine_tune_at=14, batch_size=16,
                    augmentation=aug)
    g = torch.Generator().manual_seed(0)
    ys = torch.randint(0, 5, (16,), generator=g)
    # learnable: the class sets the image's mean brightness
    xs = (ys.view(16, 1, 1, 1).float() * 50 + torch.rand(16, 64, 64, 3, generator=g) * 30).to(torch.uint8)
    data = [(xs, ys)] * 8
    tr = Trainer(m).compile(optim.SGD(0.01, momentum=0.9), loss=CategoricalCrossentropy(from_logits=True,
                                                                                       label_smoothing=0.1))
    h = tr.fit(data, steps_per_epoch=8, epochs=3, verbose=0)
    print("losses", h.history["loss"])
    assert all(v == v for v in h.history["loss"]) and h.history["loss"][-1] < h.history["loss"][0]


def test_distillation_from_resnet50_teacher():
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.train import Trainer
    from b200ddl.train.losses import Distillation

    teacher = build_model(64, 64, 3, 5, dropout=0.0, arch="resnet50", batch_size=16, seed=1)
    student = build_model(64, 64, 3, 5, dropout=0.0, arch="resnet50_head", fine_tune_at=16, batch_size=16)
    g = torch.Generator().manual_seed(1)
    data = [(torch.randint(0, 256, (16, 64, 64, 3), dtype=torch.uint8, generator=g), torch.randint(0, 5, (16,), generator=g))
            for _ in range(3)]
    tr = Trainer(student).compile(optim.SGD(0.01, momentum=0.9), loss=Distillation(teacher, alpha=0.5, temperature=2.0))
    h = tr.fit(data, steps_per_epoch=3, epochs=1, verbose=0)
    assert all(v == v for v in h.history["distillation_loss"])


def test_tracking_round_trip_on_gpu(tmp_path):
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.tracking.models import _describe, load_model, save_model
    from b200ddl.train import Trainer

    m = build_model(64, 64, 3, 5, dropout=0.0, arch="resnet50_head", fine_tune_at=14, batchnorm="training",
                    batch_size=8)
    tr = Trainer(m).compile(optim.SGD(0.05, momentum=0.9))
    g = torch.Generator().manual_seed(2)
    data = [(torch.randint(0, 256, (8, 64, 64, 3), dtype=torch.uint8, generator=g), torch.randint(0, 5, (8,), generator=g))
            for _ in range(2)]
    tr.fit(data, steps_per_epoch=2, epochs=1, verbose=0)
    d = _describe(m)
    assert (d["arch"], d["fine_tune_at"], d["batchnorm"]) == ("resnet50_head", 14, "training")
    save_model(tr, str(tmp_path / "m"))
    got = load_model(str(tmp_path / "m"))
    assert got.model.arch == "resnet50_head" and got.model.fine_tune_at == 14 and got.model.batchnorm == "training"
    sa, sb = m.state_dict(), got.model.state_dict()
    assert all(torch.equal(sa[n], sb[n]) for n in sa)
    # the loaded trainer predicts on the inference build (every block's BatchNorm folded into the epilogues): the same
    # logits as a fresh inference engine with the saved weights, and within bf16 rounding of the training build's
    x = data[0][0].numpy()
    fresh = build_model(64, 64, 3, 5, dropout=0.0, arch="resnet50_head", fine_tune_at=14, batchnorm="training",
                        batch_size=8)
    fresh.load_state_dict(sa)
    p_loaded, p_fresh, p_train = got.predict(x), Trainer(fresh).predict(x), tr.predict(x)
    assert (p_loaded == p_fresh).all()
    scale = float(abs(p_train).max())
    assert float(abs(p_loaded - p_train).max()) <= 0.05 * scale + 1e-3


def test_two_phase_checkpoint(tmp_path):
    """Keras's recipe: train the head at k = 17, then load those weights and fine-tune at k = 14; and a fully
    trainable resnet50 checkpoint loads into a fine-tuning engine."""
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.train import Trainer

    g = torch.Generator().manual_seed(4)
    data = [(torch.randint(0, 256, (8, 64, 64, 3), dtype=torch.uint8, generator=g), torch.randint(0, 5, (8,), generator=g))]
    a = Trainer(build_model(64, 64, 3, 5, arch="resnet50_head", batch_size=8)).compile(optim.Adam(1e-3))
    a.fit(data, steps_per_epoch=2, epochs=1, verbose=0)
    a.save_weights(str(tmp_path / "head.pt"))
    a.save(str(tmp_path / "head_full.pt"))
    b = Trainer(build_model(64, 64, 3, 5, arch="resnet50_head", fine_tune_at=14, batch_size=8)).compile(optim.SGD(1e-3))
    b.load_weights(str(tmp_path / "head.pt"))
    sa, sb = a.get_weights(), b.get_weights()
    assert all(torch.equal(sa[n], sb[n]) for n in sa)
    b.fit(data, steps_per_epoch=1, epochs=1, verbose=0)
    full = Trainer(build_model(64, 64, 3, 5, arch="resnet50", batch_size=8)).compile(optim.SGD(1e-3))
    c = Trainer(build_model(64, 64, 3, 5, arch="resnet50_head", fine_tune_at=8, batch_size=8)).compile(optim.SGD(1e-3))
    c.set_weights(full.get_weights())
    sa, sc = full.get_weights(), c.get_weights()
    assert all(torch.equal(sa[n], sc[n]) for n in sa)
    ck = torch.load(str(tmp_path / "head_full.pt"))
    assert ck["optimizer"]["state"]["m"].numel() == a.model.trainable_numel


# ================================================================================================ float64 oracle
# The per-layer float64 oracle of tests/test_resnet_engine_oracle.py (its helpers, bounds and 1/16 teeth rule), applied
# to a fine-tuning step: every frozen fused-epilogue layer up to the boundary input, the forward of every trainable
# block, the backward of every trainable BatchNorm (with the inference-mode coefficients where the mode says so), the
# gradient of every trainable tensor, and the running statistics (updated by the rule in training mode, untouched
# everywhere else).
import test_resnet_engine_oracle as O  # noqa: E402

ORACLE_CASES = [(16, "inference"), (14, "inference"), (14, "training"), (4, "inference"), (1, "training"),
                (0, "inference")]


def _ft_depths(eng):
    """Summation depths (as test_resnet_engine_oracle._depths) of the trainable layers of a fine-tuning engine."""
    from b200ddl.ops.conv import sm_count

    N, H0 = eng.batch, eng.y0.shape[1]
    fwd, bwd, wg = {}, {}, {"fc": O._wgrad_depth(N, eng._fc_wg.plan)}
    if eng._k == 0:
        tiles0 = N * H0
        grid0 = min(tiles0, sm_count())
        fwd["bn1"] = 16 + 8 * -(-tiles0 // grid0) + grid0
        bwd["bn1"] = O._col_reduce_depth(N * H0 * H0, 64)
        wg["conv1"] = 8 * -(-tiles0 // grid0) + 16 + grid0
    for bi, b in enumerate(eng.blocks):
        if bi < eng._first:
            continue
        n = b.name
        for c, bn in (("conv1", "bn1"), ("conv2", "bn2"), ("conv3", "bn3"), ("downsample.0", "downsample.1")):
            if c == "downsample.0" and not b.downsample:
                continue
            full, bname = f"{n}.{c}", f"{n}.{bn}"
            C_ = eng.bn_channels[bname]
            fwd[bname] = O._epilogue_depth([eng._fwd[full].plan], C_)
            wg[full] = O._wgrad_depth(N * (b.h_out if c != "conv1" else b.h_in) ** 2, eng._wg[full].plan)
            M = N * (b.h_in if c == "conv1" else b.h_out) ** 2
            if bname in eng._fused_reduce:
                src = eng._dg[f"{n}.conv2" if bn == "bn1" else f"{n}.conv3"]
                bwd[bname] = O._epilogue_depth([p for p, _, _ in src.parts], C_)
            elif bname in eng._block_fused:
                src = eng._dg[f"{eng.blocks[bi + 1].name}.conv1"]
                bwd[bname] = O._epilogue_depth([p for p, _, _ in src.parts], C_)
            else:
                bwd[bname] = O._col_reduce_depth(M, C_)
    return dict(fwd=fwd, bwd=bwd, wgrad=wg)


def _run_ft_step(eng):
    """One eager training step with the backward intermediates captured (test_resnet_engine_oracle.run_train_step for
    an engine whose first trainable block has no conv1 / downsample dgrad and whose gradient buffer is the trainable
    prefix)."""
    run_before = {bn: (eng.running_mean[bn].clone(), eng.running_var[bn].clone()) for bn in eng.bn_names}
    bwd, dx = {}, {}
    bn_bwd, conv_bwd = eng._bn_bwd, eng._conv_bwd

    def cap_bn_bwd(bn, mode, g1, g2, out, y, dy, dz, count):
        r = dict(g1=O._clone(g1), g2=O._clone(g2))
        bn_bwd(bn, mode, g1, g2, out, y, dy, dz, count)
        r.update(dy=dy.clone(), dz=O._clone(dz))
        bwd[bn] = r

    def cap_conv_bwd(full, cname):
        conv_bwd(full, cname)
        if full in eng._dg:
            dx[full] = eng._dg[full].dx.clone()

    eng._bn_bwd, eng._conv_bwd = cap_bn_bwd, cap_conv_bwd
    try:
        eng.forward(training=True)
        eng.backward()
    finally:
        del eng._bn_bwd, eng._conv_bwd
    torch.cuda.synchronize()
    rec = O._common_record(eng)
    rec.update(run_before=run_before, bwd=bwd, dx=dx, block_fused=set(eng._block_fused),
               dlogits16=eng.dlogits16.clone(), dpooled=eng.dpooled.clone(),
               dy0=eng._scr["dzA"][:eng.y0.numel()].view(eng.y0.shape).clone() if eng._k == 0 else None,
               grads={s.name: eng.g(s.name).clone() for s in eng.trainable_specs}, depth=_ft_depths(eng),
               k=eng._k, bn_train=eng._bn_train)
    return rec


def _check_eval_affine(rep, rec, bn, eps):
    """Running-statistics BatchNorm: mean / invstd as the backward reads them, and scale / shift as apply reads them."""
    w = rec["bnw"][bn]
    rm, rv = (t.double() for t in rec["run_before"][bn])
    rep.equal(f"{bn} mean (running)", torch.equal(w["mean"].double(), rm), "mean is not the running mean")
    ref_is, d_is = O.invstd_bound(rv, torch.zeros_like(rv), eps)
    rep.bounded(f"{bn} invstd (running)", w["invstd"], ref_is, d_is)
    g, b = rec["gamma"][bn].double(), rec["beta"][bn].double()
    sc = g * w["invstd"].double()
    rep.bounded(f"{bn} scale", w["scale"], sc, O.U * sc.abs())
    sh = b - rm * w["scale"].double()
    rep.bounded(f"{bn} shift", w["shift"], sh, 2 * O.U * (b.abs() + (rm * w["scale"].double()).abs()))


def _check_bn_bwd(rep, rec, bn, dz_sum, dz_apply, y, dz_err=0.0):
    """O.check_bn_bwd, or with running-statistics BatchNorm the inference coefficients: dgamma / dbeta as in training
    mode (with the running mean / invstd the forward used), dy = gamma * invstd * dz (B = C = 0)."""
    if rec["bn_train"]:
        return O.check_bn_bwd(rep, rec, bn, dz_sum, dz_apply, y, dz_err)
    w = rec["bnw"][bn]
    r = O.bn_bwd_ref(dz_sum, dz_apply, y, w["mean"], w["invstd"], rec["gamma"][bn], rec["depth"]["bwd"][bn], dz_err)
    rep.bounded(f"{bn} dbeta", rec["grads"][bn + ".bias"], r["dbeta"], r["d_dbeta"], param=bn + ".bias")
    rep.bounded(f"{bn} dgamma", rec["grads"][bn + ".weight"], r["dgamma"], r["d_dgamma"], param=bn + ".weight")
    da = O.flat(dz_apply)
    err = dz_err if not torch.is_tensor(dz_err) else O.flat(dz_err)
    A = rec["gamma"][bn].double() * w["invstd"].double()
    dy = A * da
    e = da.abs() * O.U * A.abs() + A.abs() * err + O.U * dy.abs()
    rep.bounded(f"{bn} dy", O.flat(rec["bwd"][bn]["dy"] if bn != "bn1" else rec["dy0"]), dy, O.bf16_bound(dy, e))


def _check_wgrad(rep, rec, full, conv, x, dy):
    wref, wab = O.conv_wgrad(x, dy, conv)
    rep.bounded(f"{full}.weight wgrad", O.kernel_grad(rec, full + ".weight"), wref,
                O.UM * rec["depth"]["wgrad"][full] * wab, param=full + ".weight")


def check_ft_step(rec, model):
    rep = O.Report()
    k, A = rec["k"], rec["act"]
    bl = O.blocks(model)
    first = max(k - 1, 0)
    # ---- stem
    ref, ab = O.conv_fwd_stem(rec, model)
    rep.bounded("conv1 y", rec["y0"], ref, O.bf16_bound(ref, O.UM * O.gemm_depth(192) * ab))
    if k == 0 and rec["bn_train"]:
        O.check_stats(rep, rec, "bn1", rec["y0"], model.bn1)
        O.check_affine(rep, rec, "bn1")
    else:
        _check_eval_affine(rep, rec, "bn1", model.bn1.eps)
    O.check_stem_pool(rep, rec, "maxpool")
    x_in = rec["p0"]
    # ---- frozen blocks: fused epilogues (folded running statistics), up to the boundary input
    for name, blk in bl[:first]:
        def epi(conv, bn, x, res=None, relu=True):
            _check_eval_affine(rep, rec, bn, 1e-5)
            w = rec["bnw"][bn]
            acc, ab = O.conv_fwd(x, conv)
            v = O.flat(acc) * w["scale"].double() + w["shift"].double()
            e = w["scale"].double().abs() * O.flat(ab) * O.UM * O.gemm_depth(conv.weight[0].numel()) + O.U * v.abs()
            if res is not None:
                v = v + O.flat(res)
                e = e + O.U * v.abs()
            ref = v.clamp(min=0) if relu else v
            return ref, e

        for c, bn, x, a in (("conv1", "bn1", x_in, "a1"), ("conv2", "bn2", A[name + ".a1"], "a2")):
            ref, e = epi(getattr(blk, c), f"{name}.{bn}", x)
            rep.bounded(f"{name}.{c}+{bn} {a}", O.flat(A[f"{name}.{a}"]), ref, O.bf16_bound(ref, e))
        res = x_in
        if blk.downsample is not None:
            ref, e = epi(blk.downsample[0], f"{name}.downsample.1", x_in, relu=False)
            rep.bounded(f"{name}.downsample yd", O.flat(A[name + ".yd"]), ref, O.bf16_bound(ref, e))
            res = A[name + ".yd"]
        ref, e = epi(blk.conv3, f"{name}.bn3", A[name + ".a2"], res=res)
        key = f"{name}.conv3+bn3 out" + (" (boundary input)" if name == bl[first - 1][0] and k < 17 else "")
        rep.bounded(key, O.flat(A[name + ".out"]), ref, O.bf16_bound(ref, e))
        x_in = A[name + ".out"]
    # ---- trainable blocks, forward
    for name, blk in bl[first:]:
        convs = [("conv1", "bn1", x_in, "y1"), ("conv2", "bn2", A[name + ".a1"], "y2"), ("conv3", "bn3", A[name + ".a2"], "y3")]
        if blk.downsample is not None:
            convs.append(("downsample.0", "downsample.1", x_in, "yd"))
        for c, bn, x, y in convs:
            conv = blk.downsample[0] if c == "downsample.0" else getattr(blk, c)
            bnmod = blk.downsample[1] if c == "downsample.0" else getattr(blk, bn)
            ref, ab = O.conv_fwd(x, conv)
            rep.bounded(f"{name}.{c} y", A[f"{name}.{y}"], ref,
                        O.bf16_bound(ref, O.UM * O.gemm_depth(conv.weight[0].numel()) * ab))
            if rec["bn_train"]:
                O.check_stats(rep, rec, f"{name}.{bn}", A[f"{name}.{y}"], bnmod)
                O.check_affine(rep, rec, f"{name}.{bn}")
            else:
                _check_eval_affine(rep, rec, f"{name}.{bn}", bnmod.eps)
        for bn, y, a in (("bn1", "y1", "a1"), ("bn2", "y2", "a2")):
            v, e = O.bn_pre(rec, f"{name}.{bn}", A[f"{name}.{y}"])
            ref = v.clamp(min=0)
            rep.bounded(f"{name}.{bn} relu", O.flat(A[f"{name}.{a}"]), ref, O.bf16_bound(ref, e))
        v3, e3 = O.bn_pre(rec, f"{name}.bn3", A[name + ".y3"])
        if blk.downsample is not None:
            r, er = O.bn_pre(rec, f"{name}.downsample.1", A[name + ".yd"])
        else:
            r, er = O.flat(x_in), 0.0
        pre = v3 + r
        ref = pre.clamp(min=0)
        out = O.flat(A[name + ".out"])
        rep.bounded(f"{name} out", out, ref, O.bf16_bound(ref, e3 + er + O.U * pre.abs()))
        mask = O.unpack_mask(A[name + ".mask"], out.shape)
        rep.equal(f"{name} mask", bool((mask == (out > 0)).all()), "mask bits differ from out > 0")
        x_in = A[name + ".out"]
    O.check_head(rep, rec, model)
    # ---- running statistics: only trainable BatchNorms in training mode move (checked above); the rest are untouched
    moved = set()
    if rec["bn_train"]:
        moved = {f"{n}.{bn}" for n, blk in bl[first:] for bn in ("bn1", "bn2", "bn3", "downsample.1")}
        moved |= {"bn1"} if k == 0 else set()
    for bn in rec["bnw"]:
        if bn not in moved:
            same = all(torch.equal(rec["run_after"][bn][i], rec["run_before"][bn][i]) for i in (0, 1))
            rep.equal(f"{bn} running statistics unchanged", same, "a frozen / inference-mode BatchNorm's statistics moved")
    # ---- backward
    cap, dx = rec["bwd"], rec["dx"]
    Kc = model.fc.weight.shape[0]
    z = rec["logits"].double()
    p = torch.softmax(z, 1)
    ref = (p - F.one_hot(rec["labels"], Kc).double()) / O.N_BATCH
    # + 2^-126: a running-statistics network at random init has widely spread logits, and a probability below the
    # smallest normal fp32 value (here down to 1e-213) underflows to zero in the kernel's fp32 softmax
    rep.bounded("fc dlogits", rec["dlogits16"][:, :Kc], ref, O.bf16_bound(ref, 2.0 ** -16 * p / O.N_BATCH + 2.0 ** -126))
    dl, pooled = rec["dlogits16"].double(), rec["pooled"].double()
    rep.bounded("fc.bias grad", rec["grads"]["fc.bias"], dl[:, :Kc].sum(0), 4 * O.U * dl[:, :Kc].abs().sum(0),
                param="fc.bias")
    rep.bounded("fc.weight grad", rec["grads"]["fc.weight"], dl.t() @ pooled,
                O.UM * rec["depth"]["wgrad"]["fc"] * (dl.abs().t() @ pooled.abs()), param="fc.weight")
    Wfc = torch.zeros(dl.shape[1], pooled.shape[1], dtype=torch.float64, device=DEV)
    Wfc[:Kc] = model.fc.weight
    ref = dl @ Wfc
    rep.bounded("fc dpooled", rec["dpooled"], ref, O.bf16_bound(ref, O.UM * O.gemm_depth(dl.shape[1]) * (dl.abs() @ Wfc.abs())))
    for i in range(len(bl) - 1, first - 1, -1):
        name, blk = bl[i]
        x_in = A[bl[i - 1][0] + ".out"] if i > 0 else rec["p0"]
        mask = O.unpack_mask(A[name + ".mask"], A[name + ".out"].shape)
        c3 = cap[name + ".bn3"]
        if i == len(bl) - 1:
            feat = A[name + ".out"]
            ref = (rec["dpooled"].double() / (feat.shape[1] * feat.shape[2]))[:, None, None, :].expand(feat.shape)
            rep.bounded("avgpool backward", c3["g1"], ref, O.bf16_bound(ref, 2 * O.U * ref.abs()))
        elif c3["g1"] is not None:
            nxt, nblk = bl[i + 1]
            rep.equal(f"{name}.bn3 g1 wiring", torch.equal(c3["g1"], dx[nxt + ".conv1"]), "main-path gradient")
            skip = dx[nxt + ".downsample.0"] if nblk.downsample is not None else cap[nxt + ".bn3"]["dz"]
            rep.equal(f"{name}.bn3 g2 wiring", torch.equal(c3["g2"], skip), "skip gradient")
        if c3["g1"] is not None:
            g = c3["g1"].double() + (c3["g2"].double() if c3["g2"] is not None else 0.0)
            dz_sum = g * mask
            rep.bounded(f"{name}.bn3 dz", c3["dz"], dz_sum, O.bf16_bound(dz_sum, O.U * dz_sum.abs()))
            _check_bn_bwd(rep, rec, name + ".bn3", dz_sum, c3["dz"], A[name + ".y3"], dz_err=O.U * dz_sum.abs())
        else:
            _check_bn_bwd(rep, rec, name + ".bn3", c3["dz"], c3["dz"], A[name + ".y3"])
        for c, bn_out, x, bn_in, y_in in (("conv3", "bn3", A[name + ".a2"], "bn2", "y2"),
                                          ("conv2", "bn2", A[name + ".a1"], "bn1", "y1")):
            conv = getattr(blk, c)
            O.check_conv_bwd(rep, rec, f"{name}.{c}", conv, x, cap[f"{name}.{bn_out}"]["dy"], dx[f"{name}.{c}"])
            cb = cap[f"{name}.{bn_in}"]
            rep.equal(f"{name}.{bn_in} g1 wiring", torch.equal(cb["g1"], dx[f"{name}.{c}"]), "incoming gradient")
            v, _ = O.bn_pre(rec, f"{name}.{bn_in}", A[f"{name}.{y_in}"])
            dz = O.flat(cb["g1"]) * (v > 0)
            _check_bn_bwd(rep, rec, f"{name}.{bn_in}", dz, dz, A[f"{name}.{y_in}"])
        boundary = i == first and k > 0
        if blk.downsample is not None:
            bd = name + ".downsample.1"
            cd = cap[bd]
            rep.equal(f"{bd} g1 wiring", torch.equal(cd["g1"], c3["dz"]), "incoming gradient is not the block's dz")
            _check_bn_bwd(rep, rec, bd, cd["g1"], cd["g1"], A[name + ".yd"])
            if boundary:
                _check_wgrad(rep, rec, name + ".downsample.0", blk.downsample[0], x_in, cd["dy"])
            else:
                O.check_conv_bwd(rep, rec, name + ".downsample.0", blk.downsample[0], x_in, cd["dy"],
                                 dx[name + ".downsample.0"])
        dy1 = cap[name + ".bn1"]["dy"]
        if boundary:   # the frozen prefix takes no gradient: weight gradient only
            rep.equal(f"{name} boundary", name + ".conv1" not in dx and name + ".downsample.0" not in dx,
                      "a data gradient was computed into the frozen prefix")
            _check_wgrad(rep, rec, name + ".conv1", blk.conv1, x_in, dy1)
        elif i > 0 and (bl[i - 1][0] + ".bn3") in rec["block_fused"]:
            skip = dx[name + ".downsample.0"] if blk.downsample is not None else c3["dz"]
            if skip.shape != x_in.shape:
                full = torch.zeros(x_in.shape, dtype=torch.float64, device=DEV)
                full[:, ::2, ::2] = skip.double()
                skip = full
            O.check_conv_bwd(rep, rec, name + ".conv1", blk.conv1, x_in, dy1, dx[name + ".conv1"],
                             skip=skip.double(), mask=O.unpack_mask(A[bl[i - 1][0] + ".mask"], x_in.shape))
        else:
            O.check_conv_bwd(rep, rec, name + ".conv1", blk.conv1, x_in, dy1, dx[name + ".conv1"])
    if k == 0:   # the stem, as in O.check_backward (the pooled gradient is materialised: fuse_stem_bwd is off)
        g = dx["layer1.0.conv1"].double() + dx["layer1.0.downsample.0"].double()
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
        rep.bounded("maxpool backward", cap["bn1"]["g1"], da, O.bf16_bound(da, 5 * O.U * da_abs))
        v, _ = O.bn_pre(rec, "bn1", rec["y0"])
        dz = cap["bn1"]["g1"].double() * (v > 0).view(da.shape)
        _check_bn_bwd(rep, rec, "bn1", dz, dz, rec["y0"])
        xs, c1, dy0 = rec["x_stem"], model.conv1, O.nchw(rec["dy0"])
        ref = torch.nn.grad.conv2d_weight(xs, c1.weight.shape, dy0, stride=c1.stride, padding=c1.padding)
        ab = torch.nn.grad.conv2d_weight(xs.abs(), c1.weight.shape, dy0.abs(), stride=c1.stride, padding=c1.padding)
        rep.bounded("conv1.weight wgrad", O.kernel_grad(rec, "conv1.weight"), ref,
                    O.UM * rec["depth"]["wgrad"]["conv1"] * ab, param="conv1.weight")
    return rep


def _ft_oracle_engine(k, mode):
    eng = O._engine(fine_tune_at=k, batchnorm=mode)
    return eng, O._oracle(eng)


@pytest.mark.parametrize("k,mode", ORACLE_CASES)
def test_finetune_step_matches_float64_per_layer(k, mode):
    eng, model = _ft_oracle_engine(k, mode)
    rec = _run_ft_step(eng)
    rep = check_ft_step(rec, model)
    O._fail_report(rep, f"fine-tuning step [k={k}, {mode}]")
    assert rep.params == {s.name for s in eng.trainable_specs}, sorted({s.name for s in eng.trainable_specs} ^ rep.params)
    if mode == "training":
        n_bn = {key.rsplit(" ", 1)[0] for key, *_ in rep.rows if key.endswith(" running_var")}
        assert n_bn == {n for n in eng.bn_names if eng.spec[n + ".weight"].offset < eng.trainable_numel}


def test_finetune_checker_flags_batch_statistics_backward():
    """A step in which one trainable BatchNorm's backward used its batch statistics instead of the running ones (what
    the training-mode coefficients would compute) must be reported, at that BatchNorm."""
    eng, model = _ft_oracle_engine(14, "inference")
    rec = _run_ft_step(eng)
    O._fail_report(check_ft_step(rec, model), "clean fine-tuning step")
    bn = "layer4.1.bn2"
    cb = rec["bwd"][bn]
    y = rec["act"]["layer4.1.y2"]
    v, _ = O.bn_pre(rec, bn, y)
    dz = O.flat(cb["g1"]) * (v > 0)
    M, mean, var, _, _ = O.stats_ref(y, 1)
    r = O.bn_bwd_ref(dz, dz, y, mean, (var + 1e-5).rsqrt(), rec["gamma"][bn], 1)
    g = dict(rec["grads"])
    g[bn + ".weight"], g[bn + ".bias"] = r["dgamma"].float(), r["dbeta"].float()
    bwd = dict(rec["bwd"])
    bwd[bn] = dict(cb, dy=r["dy"].view(cb["dy"].shape).to(torch.bfloat16))
    bad = dict(rec, grads=g, bwd=bwd)
    rep = check_ft_step(bad, model)
    hit = [f for f in rep.failures if f.startswith(bn + " dy") or f.startswith(bn + " dgamma")]
    print(f"batch statistics in {bn}'s backward: {len(rep.failures)} failures, e.g. {rep.failures[:2]}")
    assert hit, rep.failures[:5]
