"""Color augmentation on the GPU: augment_color (csrc/augment.cu) against `color_reference` (models/augment.py), and
both native engines with color on.

As in test_augment.py: outputs between guard bands, compared bit for bit, mismatch reports that name image, row,
column and channel.  Every cluster size is forced once per case and must give the same bytes, in place and out of
place.
"""
from __future__ import annotations

import pytest
import torch

from exact_util import DEV, Guarded, check_equal
from test_augment import AUG, ENGINES, PARENT_STEP_LAUNCHES, _batch, _engine, _pix, gen

pytestmark = pytest.mark.gpu

CLUSTERS = (1, 2, 4, 8)


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def _aug(**k):
    from b200ddl.models.augment import Augmentation

    return Augmentation(**k)


ALL = dict(brightness=0.3, contrast=0.8, saturation=0.9, hue=0.4, grayscale=0.4)
CONFIGS = [dict(brightness=1.0), dict(contrast=1.0), dict(saturation=1.0), dict(hue=0.5), dict(grayscale=0.5), ALL]
# (N, H, W): 224 x 224 images start on 16-pixel boundaries; the others leave single pixels before and after the
# 16-pixel groups of most images (37 x 53, 17 x 31), or have no whole group at all (3 x 5)
SHAPES = [(1, 224, 224), (3, 37, 53), (32, 64, 48), (256, 224, 224), (5, 3, 5), (3, 17, 31), (1, 2048, 7)]


def _run(e, aug, src, dst, step, key, cluster):
    from b200ddl.models.augment import color_key

    _, H, W, _ = src.shape
    return e.augment_color(src, dst, step, H, W, color_key(key), *aug.color_quantised(), cluster)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
def test_augment_color_exact(cfg, shape):
    """Each stage alone and all together, out of place and in place, at every forced cluster size and at the size the
    launch picks: the bytes equal color_reference's, and the guard bands stay intact."""
    from b200ddl.models.augment import augment_key, color_reference

    N, H, W = shape
    if N * H * W > 1 << 22 and cfg != len(CONFIGS) - 1:
        pytest.skip("the 256 x 224 x 224 batch runs with all stages only")
    aug = _aug(**CONFIGS[cfg])
    e = _ops()
    x = torch.randint(0, 256, (N, H, W, 3), device=DEV, dtype=torch.uint8, generator=gen(cfg * 31 + N))
    x[0, : H // 3] = 200    # a flat band: gray pixels, ties between channels, a contrast mean away from 127.5
    key, t = augment_key(cfg, 1), 7 + cfg
    step = torch.full((1,), t, device=DEV, dtype=torch.int32)
    ref = color_reference(aug, x, key, t)
    name = f"augment_color {N}x{H}x{W} {CONFIGS[cfg]}"
    if cfg == 0:
        assert not torch.equal(ref, x)
    for cluster in CLUSTERS + (0,):
        out = Guarded((N, H, W, 3), torch.uint8)
        G = _run(e, aug, x, out.t, step, key, cluster)
        assert G == cluster or (cluster == 0 and G in CLUSTERS)
        inplace = Guarded((N, H, W, 3), torch.uint8, fill=0)
        inplace.t.copy_(x)
        _run(e, aug, inplace.t, inplace.t, step, key, cluster)
        torch.cuda.synchronize()
        for g, how in ((out, "out of place"), (inplace, "in place")):
            g.check_guards(f"{name} G={G} {how}")
            check_equal(f"{name} G={G} {how}", g.t, ref, _pix)


def test_cluster_choice_fills_the_gpu():
    """The launch picks the smallest G in 1, 2, 4, 8 with N G >= 2 x (resident CTAs), or 8.  Whatever the kernel's
    occupancy (R resident CTAs, 1 <= R / SMs <= 8 for 256-thread CTAs), that gives G = 8 for N < SMs / 4 (8 N < 2 SMs
    <= 2 R) and G = 1 for N >= 16 SMs (>= 2 R), and G never grows with N."""
    from b200ddl.models.augment import augment_key

    e = _ops()
    aug = _aug(**ALL)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    step = torch.ones(1, device=DEV, dtype=torch.int32)
    small, large = max(1, (sms - 1) // 4), 16 * sms
    chosen = {}
    for N in sorted({1, small, 256, 1024, large}):
        x = torch.zeros(N, 8, 8, 3, device=DEV, dtype=torch.uint8)
        chosen[N] = _run(e, aug, x, x, step, augment_key(0, 0), 0)
    torch.cuda.synchronize()
    print("cluster per image by batch:", chosen)
    assert chosen[1] == 8 and chosen[small] == 8 and chosen[large] == 1
    assert set(chosen.values()) <= set(CLUSTERS)
    Ns = sorted(chosen)
    assert all(chosen[a] >= chosen[b] for a, b in zip(Ns, Ns[1:]))


def test_malformed_inputs_raise():
    e = _ops()
    N, H, W = 4, 32, 48
    x = torch.zeros(N, H, W, 3, device=DEV, dtype=torch.uint8)
    out = torch.zeros_like(x)
    step = torch.zeros(1, device=DEV, dtype=torch.int32)
    ok = dict(src=x, dst=out, step=step, H=H, W=W, ckey=1, bq=100, cq=100, sq=100, hq=100, pq=100, cluster=0)
    big = torch.zeros(2 * x.numel() + 16, device=DEV, dtype=torch.uint8)
    bad = [dict(src=x.float()), dict(src=x.cpu()), dict(src=x.permute(0, 2, 1, 3)), dict(dst=out[:, :, :-1]),
           dict(dst=torch.zeros(N, H, W, 3, device=DEV, dtype=torch.int32)), dict(H=H + 1), dict(W=W - 1),
           dict(src=torch.zeros(N, H, W, 4, device=DEV, dtype=torch.uint8)),
           dict(dst=torch.zeros(out.numel() + 8, device=DEV, dtype=torch.uint8)[8:].view(out.shape)),
           dict(src=big[:x.numel()].view(x.shape), dst=big[48:48 + x.numel()].view(x.shape)),
           dict(step=step.long()), dict(step=step.cpu()), dict(step=torch.zeros(2, device=DEV, dtype=torch.int32)),
           dict(ckey=-1), dict(ckey=1 << 32), dict(bq=-1), dict(bq=255 * 256 + 1), dict(cq=65537), dict(sq=-1),
           dict(hq=3 * 65536 + 1), dict(pq=65537), dict(cluster=3), dict(cluster=16), dict(cluster=-1)]
    e.augment_color(**ok)
    e.augment_color(**{**ok, "dst": x})   # in place is allowed
    torch.cuda.synchronize()
    for b in bad:
        with pytest.raises(RuntimeError):
            e.augment_color(**{**ok, **b})
    torch.cuda.synchronize()
    big_side = torch.zeros(1, 2049, 1, 3, device=DEV, dtype=torch.uint8)
    with pytest.raises(RuntimeError):
        e.augment_color(**{**ok, "src": big_side, "dst": big_side, "H": 2049, "W": 1})


# ================================================================================================ engines
ENGINE_AUGS = [dict(**AUG, **ALL), dict(ALL), dict(**AUG, cutmix=1.0, **ALL)]
IDS = ["geometric+color", "color", "cutmix+color"]


@pytest.mark.parametrize("cfg", range(len(ENGINE_AUGS)), ids=IDS)
@pytest.mark.parametrize("arch,k", ENGINES)
def test_training_steps_feed_the_stem_the_reference_batch(arch, k, cfg):
    """Graphed steps t = 1, 2, 3 leave the reference batch of step t (color included) in the buffer the stem reads,
    the eager path gives the same three buffers, and consecutive steps differ."""
    from b200ddl import optim
    from b200ddl.models.augment import augment_key, augment_reference
    from b200ddl.models.resnet_engine import EngineTrainStep

    aug = _aug(**ENGINE_AUGS[cfg])
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
            check_equal(f"{arch} k={k} {IDS[cfg]} graph={use_graph} step {t}", bufs[-1], ref, _pix)
        runs[use_graph] = bufs
    for t in range(3):
        check_equal(f"{arch} k={k} {IDS[cfg]}: eager vs graphed step {t + 1}", runs[False][t], runs[True][t], _pix)
    assert not torch.equal(runs[True][0], runs[True][1]) and not torch.equal(runs[True][1], runs[True][2])


@pytest.mark.parametrize("arch,k", ENGINES)
def test_evaluate_and_predict_never_color(arch, k):
    """evaluate / predict of an engine trained one step with color on give bit for bit the logits of a color-free
    engine with the same state."""
    from b200ddl import optim
    from b200ddl.train import Trainer

    eng = _engine(arch, k, _aug(**AUG, **ALL), seed=4)
    x, y = _batch(eng, seed=8)
    tr = Trainer(eng)
    tr.compile(optim.SGD(0.0))
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


@pytest.mark.parametrize("arch,k", ENGINES)
def test_training_step_launch_count(arch, k):
    """Color adds one launch to the geometric augmentation's two; color alone is one launch."""
    from b200ddl import ops, optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    counts = []
    for a in (None, _aug(**AUG), _aug(**AUG, **ALL), _aug(**ALL)):
        eng = _engine(arch, k, a)
        x, y = _batch(eng)
        step = EngineTrainStep(eng, optim.SGD(0.01), use_graph=False)
        step.load(x, y)
        step.run()
        torch.cuda.synchronize()
        n0 = ops.kernel_launches()
        step.load(x, y)
        step.run()
        torch.cuda.synchronize()
        counts.append(ops.kernel_launches() - n0)
    print(f"launches per step {arch} k={k}: {counts}")
    p = PARENT_STEP_LAUNCHES[(arch, k)]
    assert counts == [p, p + 2, p + 3, p + 1]
