"""MixUp, CutMix and label smoothing on the GPU: augment_mix_params / augment_mix_warp (csrc/augment.cu) and
softmax_ce_soft_head (csrc/head_stem.cu) against the torch references in models/augment.py, and both native engines
with the options on.

The integer kernels are compared bit for bit.  The soft head is held to the float64 reference within bounds derived
like test_elementwise_exact.softmax_bounds, and to softmax_ce_head bit for bit where mu = 0 and eps = 0.
"""
from __future__ import annotations

import itertools

import pytest
import torch
import torch.nn.functional as F

from exact_util import DEV, U, Guarded, check_equal
from test_augment import AUG, ENGINES, PARENT_STEP_LAUNCHES, WARP_CASES, GuardedI32, _batch, _engine, _pix
from test_elementwise_exact import BF, NAN, RCP_ULP, bf, check_bound, f32, head_data, softmax_bounds

pytestmark = pytest.mark.gpu


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _aug(**k):
    from b200ddl.models.augment import Augmentation

    return Augmentation(**k)


MIXES = [dict(mixup=0.2), dict(mixup=2.0), dict(cutmix=1.0), dict(cutmix=0.3)]


# ================================================================================================ augment_mix_params
GEOMETRIC = [dict(), dict(flip="horizontal_and_vertical", rotation=0.2, zoom=0.3, translation=0.2),
             dict(flip="vertical", rotation=0.5, zoom=0.9, translation=1.0)]
KEYS = [(0, 0, 1), (7, 3, 2), (123456789, 1, 100_000)]   # (seed, rank, step)


@pytest.mark.parametrize("N", [1, 2, 255, 256, 1000])
def test_mix_params_exact(N):
    """The geometric rows equal augment_params' bit for bit, and the mix rows equal the reference, for MixUp and CutMix
    at several alpha, (seed, rank, step) keys and image sizes; the guard words around both outputs stay intact."""
    from b200ddl.models.augment import augment_key, mix_params_reference, params_reference

    e = _ops()
    step = torch.zeros(1, device=DEV, dtype=torch.int32)
    for geo, mix, (seed, rank, t), (H, W) in itertools.product(GEOMETRIC, MIXES, KEYS, ((224, 224), (37, 53))):
        aug = _aug(**geo, **mix)
        key = augment_key(seed, rank)
        zq, txq, tyq = aug.quantised(H, W)
        rot, lam = aug.rotation_table().to(DEV), aug.lambda_table().to(DEV)
        out, rows, plain = GuardedI32((N, 8)), GuardedI32((N, 8)), GuardedI32((N, 8))
        step.fill_(t)
        e.augment_mix_params(out.t, rows.t, step, rot, lam, H, W, key, aug.flip_mode, zq, txq, tyq, aug.mix_mode)
        e.augment_params(plain.t, step, rot, H, W, key, aug.flip_mode, zq, txq, tyq)
        torch.cuda.synchronize()
        name = f"augment_mix_params N={N} {geo} {mix} seed={seed} rank={rank} step={t} {H}x{W}"
        for g, nm in ((out, "params"), (rows, "mix"), (plain, "augment_params")):
            g.check_guards(f"{name} {nm}")
        check_equal(name + " geometric rows vs augment_params", out.t, plain.t, lambda n, f: f"[image {n}, field {f}]")
        check_equal(name + " geometric rows", out.t, params_reference(aug, N, H, W, key, t, device=DEV),
                    lambda n, f: f"[image {n}, field {f}]")
        check_equal(name + " mix rows", rows.t, mix_params_reference(aug, N, H, W, key, t, device=DEV),
                    lambda n, f: f"[image {n}, field {f}]")


# ================================================================================================ augment_mix_warp
MIX_WARP_CASES = WARP_CASES + [(6, 37, 53, dict())]   # the last: identity transform, mixing only


@pytest.mark.parametrize("mix", [dict(mixup=0.4), dict(cutmix=1.0)], ids=["mixup", "cutmix"])
@pytest.mark.parametrize("fill", [("reflect", 0), ("constant", 0), ("constant", 201)])
@pytest.mark.parametrize("case", range(len(MIX_WARP_CASES)))
def test_mix_warp_exact(case, fill, mix):
    from b200ddl.models.augment import augment_key, mix_params_reference, mix_warp_reference, params_reference

    N, H, W, cfg = MIX_WARP_CASES[case]
    aug = _aug(**cfg, **mix, fill_mode=fill[0], fill_value=fill[1])
    x = torch.randint(0, 256, (N, H, W, 3), device=DEV, dtype=torch.uint8, generator=gen(case))
    key = augment_key(case, 0)
    params = params_reference(aug, N, H, W, key, 5, device=DEV).contiguous()
    rows = mix_params_reference(aug, N, H, W, key, 5, device=DEV).contiguous()
    if aug.mix_mode == 2:
        assert bool((rows[:, 6] > 0).any()), "no CutMix box in the case"
    out = Guarded((N, H, W, 3), torch.uint8)
    _ops().augment_mix_warp(x, out.t, params, rows, aug.mix_mode, aug.fill_mode, aug.fill_value)
    torch.cuda.synchronize()
    name = f"augment_mix_warp {N}x{H}x{W} {cfg} {mix} fill={fill}"
    out.check_guards(name)
    check_equal(name, out.t, mix_warp_reference(x, params, rows, aug.mix_mode, aug.fill_mode, aug.fill_value), _pix)


def test_mix_malformed_inputs_raise():
    e = _ops()
    aug = _aug(flip="horizontal", cutmix=1.0)
    N, H, W = 4, 32, 48
    x = torch.zeros(N, H, W, 3, device=DEV, dtype=torch.uint8)
    out = torch.zeros_like(x)
    params = torch.zeros(N, 8, device=DEV, dtype=torch.int32)
    mix = torch.zeros(N, 8, device=DEV, dtype=torch.int32)
    mix[:, 7] = 1
    step = torch.zeros(1, device=DEV, dtype=torch.int32)
    rot, lam = aug.rotation_table().to(DEV), aug.lambda_table().to(DEV)
    ok_p = dict(params=params, mix=mix, step=step, rot_table=rot, lam_table=lam, H=H, W=W, key=1, flip_mode=1, zq=0,
                txq=0, tyq=0, mode=2)
    ok_w = dict(x=x, out=out, params=params, mix=mix, mode=2, fill_mode="reflect", fill_value=0)
    bad_p = [dict(mix=params), dict(mix=mix.float()), dict(mix=mix.cpu()), dict(mix=torch.zeros(N + 1, 8, device=DEV,
             dtype=torch.int32)), dict(lam_table=lam[:100]), dict(lam_table=lam.cpu()), dict(lam_table=lam.long()),
             dict(mode=0), dict(mode=3), dict(H=0), dict(key=-1), dict(flip_mode=4), dict(zq=65536)]
    bad_w = [dict(mix=mix[:, :7].contiguous()), dict(mix=mix.cpu()), dict(mix=mix.long()), dict(mode=0), dict(out=x),
             dict(x=x.cpu()), dict(out=out[:, :, :-1]), dict(fill_mode="wrap"), dict(fill_value=256),
             dict(params=torch.zeros(N - 1, 8, device=DEV, dtype=torch.int32))]
    e.augment_mix_params(**ok_p)
    e.augment_mix_warp(**ok_w)
    torch.cuda.synchronize()
    for fn, ok, bads in ((e.augment_mix_params, ok_p, bad_p), (e.augment_mix_warp, ok_w, bad_w)):
        for bad in bads:
            with pytest.raises(RuntimeError):
                fn(**{**ok, **bad})
    lg16 = torch.zeros(N, 8, device=DEV, dtype=BF)
    bias, labels = torch.zeros(5, device=DEV), torch.zeros(N, device=DEV, dtype=torch.int64)
    stats = torch.zeros(2, device=DEV)
    ok_h = dict(logits16=lg16, bias=bias, labels=labels, mix=mix, label_smoothing=0.1, stats=stats)
    bad_h = [dict(label_smoothing=1.5), dict(label_smoothing=-0.1), dict(mix=mix[:2].contiguous()), dict(mix=mix.long()),
             dict(mix=mix.cpu()), dict(labels=labels[:2]), dict(bias=torch.zeros(9, device=DEV)),
             dict(dlogits16=lg16), dict(loss_rows=torch.zeros(N + 1, device=DEV)), dict(stats=stats[:1]),
             dict(logits32=torch.zeros(N, 4, device=DEV))]
    e.softmax_ce_soft_head(**ok_h)
    torch.cuda.synchronize()
    for bad in bad_h:
        with pytest.raises(RuntimeError):
            e.softmax_ce_soft_head(**{**ok_h, **bad})
    torch.cuda.synchronize()


# ================================================================================================ soft head
def soft_bounds(logit, labels, mix, eps, grad_scale):
    """Float64 soft-target loss and dlogits of fp32 logits, with bounds for the fast-math kernel.

    The terms of softmax_bounds carry over: lse - l errs by at most (rel_se + e_log) 1.001 + u (|lse| + |lse - l|) for
    either label.  sum_k (max - l_k) runs ceil(K / 32) + 5 additions after one rounding per term; K log(se) errs by K
    (rel_se + e_log) plus its rounding.  mu and eps / K are correctly rounded, lambda = 1 - mu and 1 - eps round once,
    and the products and sums of the combination add at most 8 u of the magnitude of each of its three parts.
    dlogits: p as in softmax_bounds, the target t rounds at most 4 times (4 u t), p - t once, then bf16."""
    from b200ddl.models.augment import mix_weight, soft_targets

    B, K = logit.shape
    y = labels.long()
    mu = mix_weight(mix, B, logit.device, torch.float64)
    yp = y if mix is None else y[mix[:, 0].long()]
    _, lb_y, _, _ = softmax_bounds(logit, y, grad_scale)
    _, lb_p, _, _ = softmax_bounds(logit, yp, grad_scale)
    mx = logit.max(1, keepdim=True).values
    x = logit - mx
    ex = torch.exp(x)
    se = ex.sum(1, keepdim=True)
    e_exp = (2 + torch.floor(1.173 * x.abs())) * 2.0 ** -23 + U * x.abs()
    depth = -(-K // 32) + 5
    rel_se = (((ex * e_exp).sum(1, keepdim=True) + depth * U * se) / se).squeeze(1)
    lg = torch.log(se).squeeze(1)
    e_log = 2.0 ** -21.41 + 3 * 2.0 ** -23 * lg.abs()
    lse = mx.squeeze(1) + lg
    ly, lp = logit.gather(1, y.view(-1, 1)).squeeze(1), logit.gather(1, yp.view(-1, 1)).squeeze(1)
    sd = (-x).sum(1)
    keep, epsk = 1 - eps, eps / K
    a, b, c = keep * (1 - mu) * (lse - ly), keep * mu * (lse - lp), epsk * (sd + K * lg)
    loss = a + b + c
    lb = (keep * ((1 - mu) * lb_y + mu * lb_p) + epsk * ((depth + 1) * U * sd + K * (rel_se + e_log) * 1.001
                                                         + U * K * lg.abs())
          + 8 * U * (a.abs() + b.abs() + c.abs()))
    t = soft_targets(labels, K, mix, eps, torch.float64)
    p = ex / se
    d = (p - t) * grad_scale
    db = (p * (e_exp + rel_se.view(-1, 1) + RCP_ULP + U) * 1.001 + 4 * U * t + U * d.abs() / grad_scale) * grad_scale \
        + 2.0 ** -126
    return loss, lb, d, db


def _mix_rows(B, g):
    """Mix rows with random partners and label weights num / den: some 0, some 1, some exactly 1/2, the rest random."""
    m = torch.zeros(B, 8, device=DEV, dtype=torch.int32)
    m[:, 0] = torch.randint(0, B, (B,), device=DEV, generator=g, dtype=torch.int32)
    den = torch.randint(1, 1 << 22, (B,), device=DEV, generator=g, dtype=torch.int32)
    num = (torch.rand(B, device=DEV, generator=g) * (den.double() + 1)).floor().clamp(max=den).to(torch.int32)
    k = torch.arange(B, device=DEV) % 5
    num = torch.where(k == 0, 0, torch.where(k == 1, den, num))
    den = torch.where(k == 2, 256, den)
    num = torch.where(k == 2, 128, num)
    m[:, 6], m[:, 7] = num, den
    return m


@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("B", [1, 257])
@pytest.mark.parametrize("K,ld", [(5, 8), (33, 64), (1000, 1024)])
def test_soft_head(K, ld, B, eps):
    """softmax_ce_soft_head with and without mix rows: logits32 exact, the accuracy count exact (argmax of the logits
    against the integer argmax of the unsmoothed target, at every eps), padded dlogits exactly 0; loss rows, the loss sum and dlogits within
    soft_bounds.  Without mixing at eps = 0, and with mix rows whose mu is 0, every output is softmax_ce_head's."""
    from b200ddl.models.augment import target_argmax

    e = _ops()
    g = gen(K * B + int(eps * 10))
    l16, bias, labels = head_data(B, K, g)
    gs = 1.0 / 256
    lg16 = torch.full((B, ld), NAN, device=DEV, dtype=BF)
    lg16[:, :K] = bf(l16)
    logit = (l16 + bias).float().double()
    for mix in (None, _mix_rows(B, g)):
        logits32, dl16 = Guarded((B, K), torch.float32), Guarded((B, ld), BF)
        loss_rows, stats = Guarded((B,), torch.float32, guard=64), Guarded((2,), torch.float32, 0.0, guard=64)
        e.softmax_ce_soft_head(lg16, f32(bias), labels, mix, eps, logits32.t, dl16.t, loss_rows.t, stats.t, gs)
        torch.cuda.synchronize()
        name = f"softmax_ce_soft_head K={K} ld={ld} B={B} eps={eps} mix={mix is not None}"
        for gd, nm in ((logits32, "logits32"), (dl16, "dlogits16"), (loss_rows, "loss_rows"), (stats, "stats")):
            gd.check_guards(f"{name} {nm}")
        check_equal(name + " logits32", logits32.t, logit, lambda b, k: f"[warp {b} lane {k % 32}]")
        want = int((torch.from_numpy(logit.cpu().numpy().argmax(1)).to(DEV) == target_argmax(labels, mix)).sum())
        assert int(stats.t[1].item()) == want, f"{name}: accuracy count"
        check_equal(name + " padded dlogits", dl16.t[:, K:], torch.zeros(B, ld - K, device=DEV))
        loss, lb, d, db = soft_bounds(logit, labels, mix, eps, gs)
        check_bound(name + " loss", loss_rows.t, loss, lb)
        check_bound(name + " loss sum", stats.t[:1], loss.sum().view(1), (lb.sum() + B * U * loss.abs().sum()).view(1))
        check_bound(name + " dlogits", dl16.t[:, :K], d, db + 2.0 ** -8 * (d.abs() + db))
        if eps != 0.0:
            continue
        zero_mu = None if mix is None else mix.clone()
        if zero_mu is not None:
            zero_mu[:, 6] = 0
        soft = [torch.zeros(B, K, device=DEV), torch.zeros(B, ld, device=DEV, dtype=BF), torch.zeros(B, device=DEV),
                torch.zeros(2, device=DEV)]
        plain = [torch.zeros_like(t) for t in soft]
        e.softmax_ce_soft_head(lg16, f32(bias), labels, zero_mu, 0.0, *soft, gs)
        e.softmax_ce_head(lg16, f32(bias), labels, *plain, gs)
        torch.cuda.synchronize()
        for nm, a, b in zip(("logits32", "dlogits16", "loss rows"), soft, plain):
            check_equal(f"{name} mu = 0: {nm} vs softmax_ce_head", a, b)
        assert float(soft[3][1]) == float(plain[3][1]), f"{name} mu = 0: accuracy vs softmax_ce_head"
        check_bound(f"{name} mu = 0: loss sum vs softmax_ce_head", soft[3][:1], plain[3][:1].double(),
                    B * U * plain[2].double().abs().sum().view(1))


# ================================================================================================ engines
ENGINE_MIXES = [dict(mixup=0.2), dict(cutmix=1.0)]


@pytest.mark.parametrize("mix", ENGINE_MIXES, ids=["mixup", "cutmix"])
@pytest.mark.parametrize("arch,k", ENGINES)
def test_training_steps_mix_the_reference_batch(arch, k, mix):
    """Graphed and eager steps t = 1, 2, 3 feed the stem the reference mixed batch of step t and hold the reference
    mix rows; the loss rows and dlogits equal the soft-head reference applied to the engine's own logits32 (eps = 0.1)
    within soft_bounds; graphed and eager runs agree bit for bit on the batch."""
    from b200ddl import optim
    from b200ddl.models.augment import augment_key, augment_reference, mix_params_reference
    from b200ddl.models.resnet_engine import EngineTrainStep

    aug = _aug(**AUG, **mix)
    eps = 0.1
    runs = {}
    for use_graph in (True, False):
        eng = _engine(arch, k, aug, seed=5)
        eng.label_smoothing = eps
        x, y = _batch(eng)
        step = EngineTrainStep(eng, optim.SGD(0.01, momentum=0.9), use_graph=use_graph)
        N = eng.batch
        bufs = []
        for t in (1, 2, 3):
            step.load(x, y)
            step.run()
            torch.cuda.synchronize()
            name = f"{arch} k={k} {mix} graph={use_graph} step {t}"
            bufs.append(eng._augmenter.out.clone())
            check_equal(name + " stem batch", bufs[-1], augment_reference(aug, x, augment_key(5, 0), t), _pix)
            rows = mix_params_reference(aug, N, eng.image_size, eng.image_size, augment_key(5, 0), t, device=DEV)
            check_equal(name + " mix rows", eng._augmenter.mix, rows)
            K = eng.num_classes
            loss, lb, d, db = soft_bounds(eng.logits.double(), y, rows, eps, 1.0 / N)
            check_bound(name + " loss rows", eng.loss_rows, loss, lb)
            check_bound(name + " dlogits", eng.dlogits16[:, :K], d, db + 2.0 ** -8 * (d.abs() + db))
        runs[use_graph] = bufs
    for t in range(3):
        check_equal(f"{arch} k={k} {mix}: eager vs graphed step {t + 1}", runs[False][t], runs[True][t], _pix)


def test_mobilenet_gradients_match_torch_module_with_cutmix_and_smoothing():
    """fine_tune_at=14 with CutMix and eps = 0.1: every trainable gradient against the fp32 `FrozenBaseClassifier` on
    the reference mixed batch and soft targets, within the bound of
    test_mobilenet_finetune.test_gradients_match_torch_module (4x the bf16-autocast distance, floor 2e-2)."""
    from b200ddl.models.augment import augment_key, augment_reference, mix_params_reference, soft_targets
    from b200ddl.models.mobilenet import FrozenBaseClassifier, MobileNetV2Base
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine
    from test_mobilenet_finetune import _grad_as_torch, _rel

    k, N, S, eps = 14, 16, 64, 0.1
    aug = _aug(flip="horizontal", rotation=0.1, cutmix=1.0)
    eng = MobileNetV2Engine(batch=N, num_classes=5, image_size=S, dropout=0.0, seed=3, fine_tune_at=k, augmentation=aug)
    eng.label_smoothing = eps
    eng.build(training=True)
    g = gen(14)
    x = torch.randint(0, 256, (N, S, S, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (N,), device=DEV, generator=g)
    eng.set_input(x, y)
    eng.set_augment_step(1)
    eng.forward(training=True)
    eng.backward()
    torch.cuda.synchronize()
    key = augment_key(3, 0)
    xm = augment_reference(aug, x, key, 1)
    rows = mix_params_reference(aug, N, S, S, key, 1, device=DEV)
    assert bool((rows[:, 6] > 0).any())
    target = soft_targets(y, 5, rows, eps)
    base = MobileNetV2Base()
    mod = FrozenBaseClassifier(base, base.out_channels, 5, 0.0, True, k).to(DEV)
    mod.load_state_dict({n: v.to(DEV) for n, v in eng.state_dict().items()})
    mod.train()
    xin = xm.permute(0, 3, 1, 2).float() / 127.5 - 1.0
    grads = {}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    for mode in ("fp32", "autocast"):
        mod.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "autocast"):
            loss = F.cross_entropy(mod(xin).float(), target)
        loss.backward()
        grads[mode] = {n: p.grad.detach().float().cpu() for n, p in mod.named_parameters() if p.requires_grad}
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    names = [s.name for s in eng.param_specs]
    assert sorted(names) == sorted(grads["fp32"])
    worst = sorted(((_rel(_grad_as_torch(eng, n), grads["fp32"][n]) / max(4 * _rel(grads["autocast"][n],
                                                                                    grads["fp32"][n]), 2e-2), n)
                    for n in names), reverse=True)
    print("worst gradient distances (ratio to gate, name):", worst[:5])
    assert worst[0][0] <= 1.0, f"gradient off: {worst[:5]}"


@pytest.mark.parametrize("arch,k", ENGINES)
def test_evaluate_smooths_and_never_mixes(arch, k):
    """An engine trained with CutMix and compiled with label smoothing 0.1: evaluate gives the logits of a plain
    engine with the same state, bit for bit, its accuracy, and the smoothed loss of those logits; predict is bit for bit
    the plain engine's."""
    from b200ddl import optim
    from b200ddl.models.augment import soft_head_reference
    from b200ddl.train import Trainer
    from b200ddl.train.losses import CategoricalCrossentropy

    eng = _engine(arch, k, _aug(**AUG, cutmix=1.0), seed=4)
    x, y = _batch(eng, seed=8)
    tr = Trainer(eng)
    tr.compile(optim.SGD(0.0), loss=CategoricalCrossentropy(from_logits=True, label_smoothing=0.1))
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
    assert res[0][0][1] == res[1][0][1], "accuracy"
    loss, lb, _, _ = soft_bounds(res[0][1].double(), y, None, 0.1, 1.0)
    ref, _, _ = soft_head_reference(res[0][1], y, None, 0.1)
    assert float((loss - ref).abs().max()) < 1e-9
    N = eng.batch
    assert abs(res[0][0][0] - float(loss.mean())) <= float(lb.sum() + N * U * loss.abs().sum()) / N + 1e-7


# ================================================================================================ launch counts
@pytest.mark.parametrize("arch,k", ENGINES)
def test_training_step_launch_count(arch, k):
    """No options: the parent's count.  Mixing adds nothing to the augmented step (params and warp are replaced, the
    head swapped), and label smoothing alone swaps the head only."""
    from b200ddl import ops, optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    counts = []
    for a, eps in ((None, 0.0), (None, 0.1), (_aug(**AUG), 0.0), (_aug(**AUG, mixup=0.2), 0.0),
                   (_aug(**AUG, cutmix=1.0), 0.1)):
        eng = _engine(arch, k, a)
        eng.label_smoothing = eps
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
    assert counts == [p, p, p + 2, p + 2, p + 2]
