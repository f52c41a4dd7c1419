"""Random augmentation in the training step (csrc/augment.cu, models/augment.py), on the GPU.

Kernel cases follow test_elementwise_exact.py: outputs between guard bands, compared bit for bit with the torch integer
reference in models/augment.py, mismatch reports that name image, row, column and channel.  Engine cases check that
every training step feeds the stem the reference-augmented batch of its optimizer step (graphed and eager alike), that
training on it matches an augmentation-free engine fed that batch, and that evaluation never augments.
"""
from __future__ import annotations

import itertools

import pytest
import torch

from exact_util import DEV, Guarded, check_equal

pytestmark = pytest.mark.gpu

POISON_I32 = -0x5A5A5A5B


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _aug(*a, **k):
    from b200ddl.models.augment import Augmentation

    return Augmentation(*a, **k)


class GuardedI32:
    """int32 output inside a buffer whose guard words before and after it hold a poison value no kernel writes."""

    def __init__(self, shape, guard=1024):
        n = 1
        for s in shape:
            n *= s
        self.g = guard
        self.buf = torch.full((n + 2 * guard,), POISON_I32, dtype=torch.int32, device=DEV)
        self.t = self.buf[guard:guard + n].view(shape)

    def check_guards(self, name):
        for side, part in (("before", self.buf[:self.g]), ("after", self.buf[-self.g:])):
            if bool((part != POISON_I32).any()):
                pytest.fail(f"{name}: guard words {side} the output were written")


def _pix(n, y, x, c):
    return f"[image {n}, row {y}, column {x}, channel {c}]"


# ================================================================================================ augment_params
FLIPS = [None, "horizontal", "vertical", "horizontal_and_vertical"]
CONFIGS = [dict(flip=f, rotation=r, zoom=z, translation=t)
           for f, r, z, t in itertools.product(FLIPS, (0.0, 0.2, 0.5), (0.0, 0.3, 0.9), (0.0, 0.2, 1.0))]
KEYS = [(0, 0, 1), (7, 3, 2), (123456789, 1, 100_000)]   # (seed, rank, step)
PARAM_N = [1, 255, 256, 1000]


@pytest.mark.parametrize("N", PARAM_N)
def test_augment_params_exact(N):
    """Every option combination (flip mode x rotation x zoom x translation), several (seed, rank, step), at 224 x 224
    and at 37 x 53: the int32 [N, 8] table equals the reference bit for bit."""
    from b200ddl.models.augment import augment_key, params_reference

    e = _ops()
    step = torch.zeros(1, device=DEV, dtype=torch.int32)
    for cfg, (seed, rank, t), (H, W) in itertools.product(CONFIGS, KEYS, ((224, 224), (37, 53))):
        aug = _aug(**cfg)
        key = augment_key(seed, rank)
        zq, txq, tyq = aug.quantised(H, W)
        rot = aug.rotation_table().to(DEV)
        out = GuardedI32((N, 8))
        step.fill_(t)
        e.augment_params(out.t, step, rot, H, W, key, aug.flip_mode, zq, txq, tyq)
        torch.cuda.synchronize()
        name = f"augment_params N={N} {cfg} seed={seed} rank={rank} step={t} {H}x{W}"
        out.check_guards(name)
        ref = params_reference(aug, N, H, W, key, t, device=DEV)
        check_equal(name, out.t, ref, lambda n, f: f"[image {n}, field {f}]")


# ================================================================================================ augment_warp
WARP_CASES = [  # (N, H, W, config): 37 x 53 leaves a ragged last tile (N*H*W % 2048 != 0)
    (4, 224, 224, dict(flip="horizontal", rotation=0.2, zoom=0.2, translation=0.1)),
    (3, 37, 53, dict(flip="horizontal_and_vertical", rotation=0.1, zoom=0.3, translation=0.2)),
    (5, 37, 53, dict(flip="vertical", rotation=0.5, zoom=0.9, translation=1.0)),      # extreme: most taps outside
    (2, 224, 224, dict(flip=None, rotation=0.5, zoom=0.9, translation=1.0)),
    (64, 224, 224, dict(flip="horizontal", rotation=0.05, zoom=0.1, translation=0.1)),  # grid-stride loop runs twice
]


@pytest.mark.parametrize("fill", [("reflect", 0), ("constant", 0), ("constant", 201)])
@pytest.mark.parametrize("case", range(len(WARP_CASES)))
def test_augment_warp_exact(case, fill):
    from b200ddl.models.augment import augment_key, params_reference, warp_reference

    N, H, W, cfg = WARP_CASES[case]
    aug = _aug(**cfg, fill_mode=fill[0], fill_value=fill[1])
    x = torch.randint(0, 256, (N, H, W, 3), device=DEV, dtype=torch.uint8, generator=gen(case))
    params = params_reference(aug, N, H, W, augment_key(case, 0), 5, device=DEV).contiguous()
    out = Guarded((N, H, W, 3), torch.uint8)
    _ops().augment_warp(x, out.t, params, aug.fill_mode, aug.fill_value)
    torch.cuda.synchronize()
    name = f"augment_warp {N}x{H}x{W} {cfg} fill={fill}"
    out.check_guards(name)
    check_equal(name, out.t, warp_reference(x, params, aug.fill_mode, aug.fill_value), _pix)


def test_warp_cases_reach_every_loop():
    """The big case runs the warp's grid-stride loop over tiles more than once; a small one ends on a partial tile whose
    bytes are not a whole number of 16-byte stores, with tiles that span two images; and the extreme cases have most
    taps outside the image."""
    from b200ddl.models.augment import augment_key, params_reference

    blocks_cap, tile = 132 * 8, 256 * 8   # csrc/ops_api.h kAugWarpMaxBlocks (grid upper bound); pixels per tile
    assert any(n * h * w > blocks_cap * tile for n, h, w, _ in WARP_CASES)
    assert any((n * h * w) % tile and (n * h * w * 3) % 16 and h * w < tile for n, h, w, _ in WARP_CASES)
    N, H, W, cfg = WARP_CASES[2]
    p = params_reference(_aug(**cfg), 1000, H, W, augment_key(2, 0), 5).long()
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    sx = (p[:, 0, None, None] * xs + p[:, 1, None, None] * ys + p[:, 2, None, None]) >> 16
    sy = (p[:, 3, None, None] * xs + p[:, 4, None, None] * ys + p[:, 5, None, None]) >> 16
    outside = ((sx < 0) | (sx >= W - 1) | (sy < 0) | (sy >= H - 1)).float().mean()
    assert outside > 0.5, f"only {outside:.2f} of the taps fall outside"


def test_identity_configuration_returns_input():
    from b200ddl.models.augment import DeviceAugmenter

    x = torch.randint(0, 256, (7, 37, 53, 3), device=DEV, dtype=torch.uint8, generator=gen(9))
    a = DeviceAugmenter(_aug(), x, seed=3)
    for t in (1, 2, 99):
        a.set_step(t)
        a.run()
        torch.cuda.synchronize()
        check_equal(f"identity augmentation at step {t}", a.out, x, _pix)


def test_malformed_inputs_raise():
    e = _ops()
    aug = _aug(flip="horizontal", rotation=0.1)
    N, H, W = 4, 32, 48
    x = torch.zeros(N, H, W, 3, device=DEV, dtype=torch.uint8)
    out = torch.zeros_like(x)
    params = torch.zeros(N, 8, device=DEV, dtype=torch.int32)
    step = torch.zeros(1, device=DEV, dtype=torch.int32)
    rot = aug.rotation_table().to(DEV)
    ok_p = dict(params=params, step=step, rot_table=rot, H=H, W=W, key=1, flip_mode=1, zq=0, txq=0, tyq=0)
    ok_w = dict(x=x, out=out, params=params, fill_mode="reflect", fill_value=0)
    bad_p = [dict(params=params.float()), dict(params=params.cpu()), dict(params=torch.zeros(N, 7, device=DEV, dtype=torch.int32)),
             dict(params=torch.zeros(8, N, device=DEV, dtype=torch.int32).t()), dict(step=step.long()), dict(step=step.cpu()),
             dict(step=torch.zeros(2, device=DEV, dtype=torch.int32)), dict(rot_table=rot[:100]),
             dict(rot_table=rot.float()), dict(H=0), dict(W=4096), dict(key=-1), dict(key=1 << 32), dict(flip_mode=4),
             dict(zq=65536), dict(zq=-1), dict(txq=W * 65536 + 1), dict(tyq=-1)]
    bad_w = [dict(x=x.float()), dict(x=x.cpu()), dict(x=x.permute(0, 2, 1, 3)), dict(out=out[:, :, :-1]),
             dict(out=torch.zeros(N, H, W, 3, device=DEV, dtype=torch.int32)), dict(out=x),
             dict(out=torch.zeros(out.numel() + 8, device=DEV, dtype=torch.uint8)[8:].view(out.shape)),
             dict(params=torch.zeros(N + 1, 8, device=DEV, dtype=torch.int32)), dict(params=params.long()),
             dict(fill_mode="nearest"), dict(fill_value=256), dict(fill_value=-1),
             dict(x=torch.zeros(N, H, W, 4, device=DEV, dtype=torch.uint8))]
    e.augment_params(**ok_p)
    e.augment_warp(**ok_w)
    torch.cuda.synchronize()
    for fn, ok, bads in ((e.augment_params, ok_p, bad_p), (e.augment_warp, ok_w, bad_w)):
        for bad in bads:
            with pytest.raises(RuntimeError):
                fn(**{**ok, **bad})
    torch.cuda.synchronize()


# ================================================================================================ engines
AUG = dict(flip="horizontal", rotation=0.1, zoom=0.2, translation=0.1)
ENGINES = [("resnet50", None), ("mobilenetv2", None), ("mobilenetv2", 0), ("mobilenetv2", 14)]


def _engine(arch, k, augmentation, seed=0):
    if arch == "resnet50":
        from b200ddl.models.resnet_engine import ResNet50Engine

        return ResNet50Engine(batch=32, num_classes=5, image_size=224, seed=seed, augmentation=augmentation)
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    return MobileNetV2Engine(batch=16, num_classes=5, image_size=64, dropout=0.0, seed=seed, fine_tune_at=k,
                             augmentation=augmentation)


def _batch(eng, seed=1):
    g = gen(seed)
    x = torch.randint(0, 256, (eng.batch, eng.image_size, eng.image_size, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (eng.batch,), device=DEV, generator=g)
    return x, y


@pytest.mark.parametrize("arch,k", ENGINES)
def test_training_steps_feed_the_stem_the_reference_batch(arch, k):
    """After graphed steps t = 1, 2, 3 the buffer the stem reads equals the reference augmentation at step t (so
    the graph reads the step from device memory and warm-up leaks nothing into step 1); the eager path gives the same
    three buffers, and consecutive steps differ."""
    from b200ddl import optim
    from b200ddl.models.augment import augment_key, augment_reference
    from b200ddl.models.resnet_engine import EngineTrainStep

    aug = _aug(**AUG)
    runs = {}
    for use_graph in (True, False):
        eng = _engine(arch, k, aug, seed=5)
        x, y = _batch(eng)
        step = EngineTrainStep(eng, optim.SGD(0.01, momentum=0.9), use_graph=use_graph)
        bufs = []
        for t in (1, 2, 3):
            step.load(x, y)
            step.run()
            torch.cuda.synchronize()
            bufs.append(eng._augmenter.out.clone())
            ref = augment_reference(aug, x, augment_key(5, 0), t)
            check_equal(f"{arch} k={k} graph={use_graph} step {t}", bufs[-1], ref, _pix)
        runs[use_graph] = bufs
    for t in range(3):
        check_equal(f"{arch} k={k}: eager vs graphed step {t + 1}", runs[False][t], runs[True][t], _pix)
    assert not torch.equal(runs[True][0], runs[True][1]) and not torch.equal(runs[True][1], runs[True][2])


def _one_step(eng, x, y, t):
    eng.build(training=True)
    eng.set_input(x, y)
    eng.set_augment_step(t)
    eng.forward(training=True)
    eng.backward()
    torch.cuda.synchronize()
    return (torch.tensor(eng.loss_and_acc()[0]), eng.logits.clone(), eng.grads[:eng.flat_numel].clone(),
            eng.loss_rows.clone())


@pytest.mark.parametrize("arch,k", ENGINES)
def test_first_step_matches_engine_fed_the_augmented_batch(arch, k):
    """Step-1 loss, logits and every gradient (the stem / first trainable layer included) of an engine built with the
    augmentation equal those of an augmentation-free engine fed the reference-augmented batch: within 4x the largest
    difference between 4 reruns of the augmentation-free engine, and for the frozen MobileNetV2 (head only) the logits
    and per-image losses bit for bit (the batch loss is a sum of fp32 atomics, so its last bit follows the order of the adds)."""
    from b200ddl.models.augment import augment_key, augment_reference

    aug = _aug(**AUG)
    a = _engine(arch, k, aug, seed=2)
    x, y = _batch(a)
    xa = augment_reference(aug, x, augment_key(2, 0), 1)
    got = _one_step(a, x, y, 1)
    ref = _one_step(_engine(arch, k, None, seed=2), xa, y, 1)
    if arch == "mobilenetv2" and k is None:
        check_equal("frozen MobileNetV2: logits", got[1], ref[1])
        check_equal("frozen MobileNetV2: per-image losses", got[3], ref[3])
    reruns = [_one_step(_engine(arch, k, None, seed=2), xa, y, 1) for _ in range(4)]
    for i, name in ((0, "loss"), (1, "logits"), (2, "grads")):
        spread = max(float((r[i].double() - ref[i].double()).abs().max()) for r in reruns)
        diff = float((got[i].double() - ref[i].double()).abs().max())
        scale = float(ref[i].double().abs().max())
        assert diff <= max(4 * spread, 1e-6 * scale), f"{arch} k={k} {name}: differs by {diff}, reruns by {spread}"
    # the gradient really depends on the augmentation: the un-augmented batch gives another one
    plain = _one_step(_engine(arch, k, None, seed=2), x, y, 1)
    assert float((plain[2] - ref[2]).abs().max()) > 4 * max(float((r[2] - ref[2]).abs().max()) for r in reruns)


@pytest.mark.parametrize("arch,k", ENGINES)
def test_evaluate_and_predict_never_augment(arch, k):
    """evaluate / predict of an engine built with the augmentation, after a training step (so the augmenter and the
    training graph have run), give bit for bit the logits of an augmentation-free engine with the same state."""
    from b200ddl import optim
    from b200ddl.train import Trainer

    eng = _engine(arch, k, _aug(**AUG), seed=4)
    x, y = _batch(eng, seed=8)
    tr = Trainer(eng)
    tr.compile(optim.SGD(0.0))       # lr 0: the weights stay put; ResNet-50's running statistics do move
    tr.fit([(x, y)], epochs=1, verbose=0)
    plain = _engine(arch, k, None, seed=4)
    plain.load_state_dict(eng.state_dict())
    tr_plain = Trainer(plain)
    tr_plain.compile(optim.SGD(0.0))
    res = []
    for t, e in ((tr, eng), (tr_plain, plain)):
        ev = t.evaluate([(x, y)], verbose=0)
        res.append((ev, e.logits.clone(), torch.as_tensor(t.predict(x.cpu().numpy()))))
    check_equal(f"{arch} k={k}: evaluate logits", res[0][1], res[1][1])
    check_equal(f"{arch} k={k}: predict", res[0][2], res[1][2])
    assert res[0][0] == pytest.approx(res[1][0], rel=1e-6), (res[0][0], res[1][0])


# kernel launches of one eager training step (forward + backward + SGD + refresh) without augmentation, measured on an
# H100 with the commit before augmentation existed: augmentation=None must not change the step.  A change that adds or
# removes launches of the step itself must update these numbers with it.  The augmentation adds exactly
# augment_params + augment_warp.
PARENT_STEP_LAUNCHES = {("resnet50", None): 395, ("mobilenetv2", None): 58, ("mobilenetv2", 0): 233,
                        ("mobilenetv2", 14): 109}


@pytest.mark.parametrize("arch,k", ENGINES)
def test_training_step_launch_count(arch, k):
    from b200ddl import ops, optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    counts = []
    for a in (None, _aug(**AUG)):
        eng = _engine(arch, k, a)
        x, y = _batch(eng)
        step = EngineTrainStep(eng, optim.SGD(0.01), use_graph=False)
        step.load(x, y)
        step.run()   # captures (warm-up) first
        torch.cuda.synchronize()
        n0 = ops.kernel_launches()
        step.load(x, y)
        step.run()
        torch.cuda.synchronize()
        counts.append(ops.kernel_launches() - n0)
    print(f"launches per step {arch} k={k}: {counts}")
    assert counts == [PARENT_STEP_LAUNCHES[(arch, k)], PARENT_STEP_LAUNCHES[(arch, k)] + 2]
