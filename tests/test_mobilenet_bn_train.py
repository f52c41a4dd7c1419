"""MobileNetV2 fine-tuning with training-mode BatchNorm (`fine_tune_at=k, batchnorm="training"`) on the GPU.

Kernel cases follow test_elementwise_exact.py: integer or power-of-two data so that the float64 reference is exact,
outputs between NaN guard bands, every sum below 2^24 (asserted) so that fp32 sums are exact in any order and equality
is demanded.

Engine cases compare with the fp32 torch module `FrozenBaseClassifier(fine_tune_at=k, batchnorm="training")` in train
mode on the same weights, gated as DESIGN.md 4b: the engine's relative L2 distance to fp32 is at most 4x the module's own
distance under bf16 autocast (floor 2e-2).
"""
from __future__ import annotations

import pytest
import torch
import torch.nn.functional as F

from exact_util import DEV, Guarded, check_equal, to_bf16_exact

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, device=DEV, generator=g).double()


def pow2(shape, lo, hi, g):
    return 2.0 ** ints(shape, lo, hi, g)


def bf(t):
    return t.to(BF).contiguous()


def f32(t):
    return t.float().contiguous()


def _exact_sums(name, terms, got_sum, got_sq=None):
    """Per-channel sums over every dim but the last, exact (asserted below 2^24)."""
    t = terms.reshape(-1, terms.shape[-1])
    ref_abs = (t.abs().sum(0), (t * t).sum(0))
    assert float(ref_abs[0].max()) < 2 ** 24 and float(ref_abs[1].max()) < 2 ** 24, f"{name}: test sums too large"
    check_equal(name + " sum", got_sum.double(), t.sum(0))
    if got_sq is not None:
        check_equal(name + " sqsum", got_sq.double(), (t * t).sum(0))


# ================================================================================================ bn_apply ReLU6
APPLY_CASES = [(70_000, 64), (333, 192)]   # C = 64: more rows than one pass of the capped grid (2112 CTAs x 32 rows)
APPLY_UNROLL = (1, 2, 4)                 # rows per iteration: the U = 1 / 2 / 4 instances


@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("case", APPLY_CASES, ids=lambda c: "x".join(map(str, c)))
def test_bn_apply_relu6(case, res):
    """out = min(max(y*scale + shift [+ res], 0), 6), values on and around 0 and 6."""
    e = _ops()
    M, C = case
    g = gen(M + C + res)
    y = ints((M, C), -24, 24, g)
    sc = pow2((C,), -2, 0, g)
    sh = ints((C,), -8, 8, g) * 0.25
    r = ints((M, C), -6, 6, g) * 0.5 if res else None
    z = y * sc + sh + (r if res else 0)
    ref = to_bf16_exact(z.clamp(0, 6))
    assert bool((z == 6).any()) and bool((z == 0).any()) and bool((z > 6).any()) and bool((z < 0).any())
    old = e.get_bn_rows_unroll()
    try:
        for u in APPLY_UNROLL:
            e.set_bn_rows_unroll(u)
            out = Guarded((M, C), BF)
            e.bn_apply(bf(y), f32(sc), f32(sh), bf(r) if res else None, None, None, out.t, True, None, True)
            torch.cuda.synchronize()
            name = f"bn_apply relu6 {case} res={res} unroll={u}"
            check_equal(name, out.t, ref, lambda m, c: f"[row {m}, channel {c}]")
            out.check_guards(name)
    finally:
        e.set_bn_rows_unroll(old)


# ================================================================================================ ReLU6 mask + sum(dz*c)
MASK_VARIANTS = [(relu6, g2) for relu6 in (True, False) for g2 in (False, True)]
MASK_M = {64: 40_000, 192: 333}   # C=64: more rows than one pass of the capped grid (1056 blocks x 32 rows)


@pytest.mark.parametrize("C", sorted(MASK_M))
@pytest.mark.parametrize("relu6,use_g2", MASK_VARIANTS)
def test_relu6_mask_reduce_dzc(C, relu6, use_g2):
    """dz = (g1 [+ g2]) * [0 < y < 6] (or unmasked), sum(dz) and sum(dz * c); in place (dz = g1) too."""
    e = _ops()
    M = MASK_M[C]
    g = gen(7 * C + 2 * relu6 + use_g2)
    g1 = ints((M, C), -3, 3, g)
    g2 = ints((M, C), -3, 3, g) if use_g2 else None
    special = torch.tensor([0.0, 6.0, 5.96875, 2.0 ** -100, 3.0, -1.0], device=DEV, dtype=torch.float64)
    y = special[torch.randint(0, special.numel(), (M, C), device=DEV, generator=g)]
    c = ints((M, C), -3, 3, g)
    gs = g1 + g2 if use_g2 else g1
    dz = gs * ((y > 0) & (y < 6)) if relu6 else gs
    for inplace in (False, True):
        g1b = bf(g1)
        out = Guarded((M, C), BF) if not inplace else None
        dzt = g1b if inplace else out.t
        s = Guarded((C,), torch.float32, fill=0.0)
        sc = Guarded((C,), torch.float32, fill=0.0)
        e.relu6_mask_reduce(g1b, bf(g2) if use_g2 else None, bf(y), dzt, s.t, relu6, bf(c), sc.t)
        torch.cuda.synchronize()
        name = f"relu6_mask_reduce+dzc C={C} relu6={relu6} g2={use_g2} inplace={inplace}"
        check_equal(name, dzt, to_bf16_exact(dz), lambda m, ch: f"[row {m}, channel {ch}]")
        _exact_sums(name, dz, s.t)
        _exact_sums(name + " dz*c", dz * c, sc.t)
        s.check_guards(name + " sum")
        sc.check_guards(name + " sum_dzc")
        if out is not None:
            out.check_guards(name)


# ================================================================================================ statistics convolutions
DW_CASES = [(2, 13, 11, 64), (1, 15, 17, 192)]   # odd H / W; Wo % 4 != 0 at stride 1 and 2
DW_BIG = (16, 192, 192, 8)   # more strips than one pass of the capped grid (1056 CTAs x 32 lanes), data in images 0, 15


def _dw_conv_ref(x, w, stride):
    C = x.shape[-1]
    y = F.conv2d(x.permute(0, 3, 1, 2), w.t().reshape(C, 1, 3, 3), stride=stride, padding=1, groups=C)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("tile_w", [4, 1])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("case", DW_CASES + [DW_BIG], ids=lambda c: "x".join(map(str, c)))
def test_dwconv3x3_stats(case, stride, tile_w):
    """c = depthwise 3x3 (pad 1) as bf16 without affine or clamp, sum(c) and sum(c^2) of the stored values."""
    e = _ops()
    N, H, W, C = case
    g = gen(11 * C + stride + tile_w)
    if case == DW_BIG:
        x = torch.zeros(N, H, W, C, device=DEV, dtype=torch.float64)
        for n in (0, N - 1):
            x[n] = ints((H, W, C), -1, 1, g)
        w = ints((9, C), -1, 1, g)
    else:
        x = ints((N, H, W, C), -2, 2, g)
        w = ints((9, C), -2, 2, g) * 0.5
    ref = _dw_conv_ref(x, w, stride)
    out = Guarded(tuple(ref.shape), BF)
    s = Guarded((C,), torch.float32, fill=0.0)
    q = Guarded((C,), torch.float32, fill=0.0)
    e.dwconv3x3_stats(bf(x), f32(w), out.t, s.t, q.t, stride, tile_w)
    torch.cuda.synchronize()
    name = f"dwconv3x3_stats {case} stride={stride} tile_w={tile_w}"
    check_equal(name, out.t, to_bf16_exact(ref), lambda n, h, ww, c: f"[image {n}, output ({h}, {ww}), channel {c}]")
    _exact_sums(name, ref, s.t, q.t)
    for t in (out, s, q):
        t.check_guards(name)


STEM_CASES = [(2, 34, 30), (10, 256, 256)]   # the second: more pixels than one pass of the grid, data in the last image


@pytest.mark.parametrize("case", STEM_CASES, ids=lambda c: "x".join(map(str, c)))
def test_mbv2_stem_stats(case):
    """c = 3x3/2 stem over bf16(x * mul + add) as bf16, 32 real channels (the padded ones are never written)."""
    e = _ops()
    N, H, W = case
    g = gen(H + W)
    x = torch.full((N, H, W, 3), 128, device=DEV, dtype=torch.uint8)
    lo, hi = (126, 130) if N == 2 else (127, 129)
    sel = slice(None) if N == 2 else slice(N - 1, N)
    x[sel] = torch.randint(lo, hi + 1, x[sel].shape, device=DEV, dtype=torch.uint8, generator=g)
    w = ints((27, 32), -2, 2, g) if N == 2 else ints((27, 32), -1, 1, g)
    wt = w.view(3, 3, 3, 32).permute(3, 2, 0, 1)
    ref = F.conv2d((x.double() - 128.0).permute(0, 3, 1, 2), wt, stride=2, padding=1).permute(0, 2, 3, 1)
    out = Guarded((N, H // 2, W // 2, 64), BF)
    s = Guarded((32,), torch.float32, fill=0.0)
    q = Guarded((32,), torch.float32, fill=0.0)
    e.mbv2_stem_stats(x, f32(w), out.t, s.t, q.t, 1.0, -128.0)
    torch.cuda.synchronize()
    name = f"mbv2_stem_stats {case}"
    check_equal(name, out.t[..., :32], to_bf16_exact(ref), lambda n, h, ww, c: f"[image {n}, ({h}, {ww}), channel {c}]")
    assert bool(out.untouched()[..., 32:].all()), f"{name}: padded channels written"
    _exact_sums(name, ref, s.t, q.t)
    for t in (out, s, q):
        t.check_guards(name)


def test_case_tables_cover_every_launch_site():
    """Both activations of bn_apply's ReLU6 instances (no residual / identity residual) at every rows-per-iteration
    variant with a grid-stride loop that runs more than once; all eight relu6_mask_reduce_kernel instances (four new, with
    sum(dz*c)) past one pass of the grid; the four dwconv3x3_stats_kernel instances (stride x tile) and the stem
    statistics kernel past one pass of their grids."""
    assert set(APPLY_UNROLL) == {1, 2, 4}
    M, C = APPLY_CASES[0]
    assert M > 132 * 16 * (256 // (C // 8))
    assert set(MASK_VARIANTS) == {(a, b) for a in (True, False) for b in (False, True)}
    assert MASK_M[64] > 1056 * 32
    N, H, W, C = DW_BIG
    for stride in (1, 2):
        Ho = (H - 1) // stride + 1
        for tw in (1, 4):
            units = N * Ho * ((Ho + tw - 1) // tw)
            assert units > (1056 // ((C // 8 + 7) // 8)) * 32
            # the first pass ends before the last image: the data there is read by a second pass
            assert (N - 1) * Ho * ((Ho + tw - 1) // tw) >= 1056 * 32
    n, h, w = STEM_CASES[-1]
    assert (n - 1) * (h // 2) * (w // 2) * 4 >= 132 * 16 * 256
    assert all(case[2] % 4 and ((case[2] - 1) // 2 + 1) % 4 for case in DW_CASES)


def test_malformed_inputs_raise():
    e = _ops()
    f = lambda *s: torch.zeros(*s, device=DEV)                        # noqa: E731
    b = lambda *s: torch.zeros(*s, device=DEV, dtype=BF)              # noqa: E731
    u8 = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.uint8)    # noqa: E731
    C, M = 64, 32
    y = b(M, C)
    x4, o4 = b(1, 8, 8, C), b(1, 8, 8, C)
    calls = {
        "bn_apply: relu6 without relu": lambda: e.bn_apply(y, f(C), f(C), None, None, None, b(M, C), False, None, True),
        "bn_apply: relu6 with mask": lambda: e.bn_apply(y, f(C), f(C), None, None, None, b(M, C), True,
                                                         u8(M * C // 8), True),
        "bn_apply: relu6 with res BN": lambda: e.bn_apply(y, f(C), f(C), b(M, C), f(C), f(C), b(M, C), True, None, True),
        "relu6_mask_reduce: c without sum_dzc": lambda: e.relu6_mask_reduce(y, None, y, b(M, C), f(C), True, y, None),
        "relu6_mask_reduce: sum_dzc without c": lambda: e.relu6_mask_reduce(y, None, y, b(M, C), f(C), True, None, f(C)),
        "relu6_mask_reduce: c size": lambda: e.relu6_mask_reduce(y, None, y, b(M, C), f(C), True, b(M - 1, C), f(C)),
        "relu6_mask_reduce: short sum_dzc": lambda: e.relu6_mask_reduce(y, None, y, b(M, C), f(C), True, b(M, C),
                                                                       f(C - 8)),
        "relu6_mask_reduce: dz is c": lambda: (lambda cc: e.relu6_mask_reduce(y, None, y, cc, f(C), True, cc, f(C)))(
            b(M, C)),
        "relu6_mask_reduce: fp32 c": lambda: e.relu6_mask_reduce(y, None, y, b(M, C), f(C), True, f(M, C), f(C)),
        "dwconv3x3_stats: stride 3": lambda: e.dwconv3x3_stats(x4, f(9 * C), o4, f(C), f(C), 3, 4),
        "dwconv3x3_stats: tile 2": lambda: e.dwconv3x3_stats(x4, f(9 * C), o4, f(C), f(C), 1, 2),
        "dwconv3x3_stats: out grid": lambda: e.dwconv3x3_stats(x4, f(9 * C), o4, f(C), f(C), 2, 4),
        "dwconv3x3_stats: short sum": lambda: e.dwconv3x3_stats(x4, f(9 * C), o4, f(C - 8), f(C), 1, 4),
        "dwconv3x3_stats: short w": lambda: e.dwconv3x3_stats(x4, f(9 * C - 4), o4, f(C), f(C), 1, 4),
        "dwconv3x3_stats: misaligned w": lambda: e.dwconv3x3_stats(x4, f(9 * C + 4)[1:9 * C + 1], o4, f(C), f(C), 1, 4),
        "dwconv3x3_stats: fp32 x": lambda: e.dwconv3x3_stats(f(1, 8, 8, C), f(9 * C), o4, f(C), f(C), 1, 4),
        "mbv2_stem_stats: odd H": lambda: e.mbv2_stem_stats(u8(1, 9, 8, 3), f(27 * 32), b(1, 4, 4, C), f(32), f(32),
                                                            1.0, 0.0),
        "mbv2_stem_stats: ldc < 32": lambda: e.mbv2_stem_stats(u8(1, 8, 8, 3), f(27 * 32), b(1, 4, 4, 16), f(32), f(32),
                                                               1.0, 0.0),
        "mbv2_stem_stats: out grid": lambda: e.mbv2_stem_stats(u8(1, 8, 8, 3), f(27 * 32), b(1, 4, 3, C), f(32), f(32),
                                                               1.0, 0.0),
        "mbv2_stem_stats: sum size": lambda: e.mbv2_stem_stats(u8(1, 8, 8, 3), f(27 * 32), b(1, 4, 4, C), f(64), f(32),
                                                               1.0, 0.0),
        "mbv2_stem_stats: short w": lambda: e.mbv2_stem_stats(u8(1, 8, 8, 3), f(27 * 31), b(1, 4, 4, C), f(32), f(32),
                                                              1.0, 0.0),
    }
    accepted = []
    for name, call in calls.items():
        try:
            call()
        except RuntimeError:
            continue
        accepted.append(name)
    torch.cuda.synchronize()
    assert not accepted, f"accepted malformed calls: {accepted}"


# ================================================================================================ engine
def _engine(k, batch=8, size=64, seed=0, dropout=0.0, batchnorm="training"):
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    return MobileNetV2Engine(batch=batch, num_classes=5, image_size=size, dropout=dropout, seed=seed, fine_tune_at=k,
                             batchnorm=batchnorm)


def _batch(batch, size, seed=1):
    g = gen(seed)
    x = torch.randint(0, 256, (batch, size, size, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (batch,), device=DEV, generator=g)
    return x, y


def _grad_as_torch(eng, name):
    gv = eng.g(name).detach()
    if name.startswith("fc.weight"):
        return gv[:eng.num_classes].cpu()
    if not name.endswith(".weight") or gv.dim() == 1:
        return gv.cpu()
    lay = next(l for l in eng._layers if l[1] + ".weight" == name)
    kind, cin, cout = lay[0], lay[3], lay[4]
    if kind == "stem":
        return gv.view(3, 3, 3, 32).permute(3, 2, 0, 1).cpu()
    if kind == "dw":
        return gv[:, :cin].t().reshape(cin, 1, 3, 3).cpu()
    return gv[:cout, :cin].reshape(cout, cin, 1, 1).cpu()


def _module(k, sd):
    from b200ddl.models.mobilenet import FrozenBaseClassifier, MobileNetV2Base

    base = MobileNetV2Base()
    mod = FrozenBaseClassifier(base, base.out_channels, 5, 0.0, True, k, batchnorm="training").to(DEV)
    mod.load_state_dict({n: v.to(DEV) for n, v in sd.items()})
    return mod


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _no_tf32():
    class _Ctx:
        def __enter__(self):
            self.old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

        def __exit__(self, *a):
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old
    return _Ctx()


def _run_steps(eng, opt, x, y, steps, use_graph=False):
    from b200ddl.models.resnet_engine import EngineTrainStep

    step = EngineTrainStep(eng, opt, use_graph=use_graph)
    out = []
    for _ in range(steps):
        step.load(x, y)
        step.run()
        out.append(step.result())
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("k", [0, 1, 4, 14, 18])
def test_step_matches_torch_module(k):
    """One training step against the fp32 module in train mode on the same weights: the loss, every trainable gradient,
    and the updated running mean / variance of every trainable BatchNorm (batch 16 at 96x96: 144 values per channel
    at the top of the net)."""
    N, S = 16, 96
    eng = _engine(k, batch=N, size=S)
    eng.build(training=True)
    sd0 = eng.state_dict()
    x, y = _batch(N, S, seed=k)
    eng.set_input(x, y)
    eng.forward(training=True)
    eng.backward()
    torch.cuda.synchronize()
    loss_eng = eng.loss_and_acc()[0]
    sd_eng = eng.state_dict()
    xin = x.permute(0, 3, 1, 2).float() / 127.5 - 1.0
    res = {}
    with _no_tf32():
        for mode in ("fp32", "autocast"):
            mod = _module(k, sd0)
            mod.train()
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "autocast"):
                loss = F.cross_entropy(mod(xin).float(), y)
            loss.backward()
            res[mode] = (float(loss), {n: p.grad.detach().float().cpu() for n, p in mod.named_parameters()
                                       if p.requires_grad}, {n: v.detach().float().cpu()
                                                             for n, v in mod.state_dict().items() if "running" in n})
    names = [s.name for s in eng.param_specs]
    assert sorted(names) == sorted(res["fp32"][1]), "engine and module train different tensors"
    worst = []

    def gate(what, d_eng, d_ac):
        worst.append((d_eng / max(4 * d_ac, 2e-2), what, d_eng, d_ac))

    l32, lac = res["fp32"][0], res["autocast"][0]
    gate("loss", abs(loss_eng - l32) / abs(l32), abs(lac - l32) / abs(l32))
    for n in names:
        gate(n, _rel(_grad_as_torch(eng, n), res["fp32"][1][n]), _rel(res["autocast"][1][n], res["fp32"][1][n]))
    stats = [n for n in res["fp32"][2] if int(n.split(".")[2]) >= k]
    assert len(stats) == 2 * sum(1 for lay in eng._layers if lay[8] >= k)
    for n in stats:
        gate(n, _rel(sd_eng[n], res["fp32"][2][n]), _rel(res["autocast"][2][n], res["fp32"][2][n]))
        assert int(sd_eng[n.replace("running_mean", "num_batches_tracked").replace("running_var",
                                                                                    "num_batches_tracked")]) == 0
    worst.sort(reverse=True)
    print(f"k={k} worst distances (ratio to gate, name, engine, autocast):", worst[:5])
    assert worst[0][0] <= 1.0, f"engine off: {worst[:5]}"


def test_k19_is_the_fine_tune_at_19_engine():
    """batchnorm='training' at k = 19 trains the head only: the same launches, first-step logits bit-identical to
    fine_tune_at=19 (the loss is an fp32 atomic sum over rows, so it is compared like the rest), and after 3 SGD steps
    everything differs no more than two fine_tune_at=19 runs do."""
    from b200ddl import ops, optim

    x, y = _batch(8, 96)
    res, launches = [], []
    for bn in ("inference", "training", "inference"):
        eng = _engine(19, size=96, dropout=0.5, batchnorm=bn)
        assert eng.running.numel() == 8
        losses = _run_steps(eng, optim.SGD(0.05, momentum=0.9), x, y, 1)
        first = (losses[0], eng.logits.clone())
        n0 = ops.kernel_launches()
        losses += _run_steps(eng, optim.SGD(0.05, momentum=0.9), x, y, 2)
        launches.append(ops.kernel_launches() - n0)
        res.append((first, torch.tensor(losses), eng.logits.clone(), eng.grads[:eng.flat_numel].clone(),
                    eng.params.clone()))
    ref, bt, ref2 = res
    assert launches[1] == launches[0]
    assert bt[0][0][0] == pytest.approx(ref[0][0][0], rel=1e-6) and bt[0][0][1] == ref[0][0][1]
    check_equal("k=19 training vs inference: first-step logits", bt[0][1], ref[0][1])
    for i, name in ((1, "losses"), (2, "logits"), (3, "grads"), (4, "params")):
        spread = float((ref2[i].double() - ref[i].double()).abs().max())
        diff = float((bt[i].double() - ref[i].double()).abs().max())
        scale = float(ref[i].double().abs().max())
        assert diff <= max(4 * spread, 1e-6 * scale), f"{name}: differs by {diff}, inference runs by {spread}"


@pytest.mark.parametrize("opt_name", ["sgd_wd", "adam_wd", "adadelta_wd"])
def test_frozen_part_and_padding_stay_fixed(opt_name):
    """After optimizer steps: features[:k] weights and running statistics bit-unchanged; the trainable layers' running
    statistics moved and count the steps; all padding (weights, affines, coefficients, activations) exactly zero."""
    from b200ddl import optim

    k = 14
    make = {"sgd_wd": lambda: optim.SGD(0.05, momentum=0.9, weight_decay=1e-2),
            "adam_wd": lambda: optim.Adam(1e-3, weight_decay=1e-2),
            "adadelta_wd": lambda: optim.Adadelta(1.0, weight_decay=1e-2)}[opt_name]
    eng = _engine(k, batch=8, size=64)
    sd0 = eng.state_dict()
    x, y = _batch(8, 64)
    _run_steps(eng, make(), x, y, 3)
    sd1 = eng.state_dict()
    moved = 0
    for n, v in sd0.items():
        feat = int(n.split(".")[2]) if n.startswith("base.features.") else None
        if feat is not None and feat < k:
            check_equal(f"{opt_name}: {n} changed", sd1[n], v)
        elif n.endswith("num_batches_tracked"):
            assert int(sd1[n]) == int(v) + 3, n
        elif feat is not None:
            moved += int(not torch.equal(sd1[n], v))
            assert "running" not in n or not torch.equal(sd1[n], v), f"{n} did not move"
    assert moved > 0
    zero = lambda name, t: check_equal(f"{opt_name}: padding of {name}", t, torch.zeros_like(t))  # noqa: E731
    for lay in eng._plan:
        c = lay["cout"]
        zero(lay["conv"] + " y", lay["y"][..., c:])
        if not lay["train"]:
            continue
        zero(lay["conv"] + " c", lay["c"][..., c:])
        zero(lay["conv"] + " g", lay["g"][..., c:])
        for key in ("shift", "bshift", "bscale", "cA", "cB", "cC", "sum", "sumc", "ssum", "ssq"):
            zero(f"{lay['conv']} {key}", lay[key][c:])
        w = eng.p(lay["conv"] + ".weight")
        if lay["kind"] == "pw":
            pad = w.clone()
            pad[:c, :lay["cin"]] = 0
            zero(lay["conv"] + " weight", pad)
        elif lay["kind"] == "dw":
            zero(lay["conv"] + " weight", w[:, c:])


def test_graph_matches_eager_and_warmup_leaves_no_trace():
    """capture() + n replays: num_batches_tracked == n (the warm-up steps were undone); the running statistics are as
    close to n eager steps as eager runs are to each other (fp32 atomics).  The distance between two runs varies
    several-fold from pair to pair, and two runs sometimes agree almost exactly, so a single pair is no yardstick: the
    graph run's mean distance to five eager runs is compared with the mean distance over the ten eager pairs."""
    import itertools

    from b200ddl import optim

    k, n = 4, 3
    x, y = _batch(8, 64, seed=5)
    eager = [f"eager{i}" for i in range(5)]
    runs = {}
    for name in eager + ["graph"]:
        eng = _engine(k)
        _run_steps(eng, optim.SGD(0.05, momentum=0.9), x, y, n, use_graph=name == "graph")
        runs[name] = eng.state_dict()
    for nm, v in runs["graph"].items():
        if nm.endswith("num_batches_tracked") and int(nm.split(".")[2]) >= k:
            assert int(v) == n, nm
    stats = [nm for nm in runs["graph"] if "running" in nm and int(nm.split(".")[2]) >= k]
    pairs = list(itertools.combinations(eager, 2))
    for nm in stats:
        spread = sum(_rel(runs[b][nm], runs[a][nm]) for a, b in pairs) / len(pairs)
        diff = sum(_rel(runs["graph"][nm], runs[a][nm]) for a in eager) / len(eager)
        assert diff <= max(4 * spread, 1e-3), f"{nm}: graph vs eager {diff}, eager runs {spread}"


@pytest.mark.parametrize("use_graph", [True, False])
def test_fit_lowers_loss_and_eval_uses_running_statistics(use_graph):
    """Trainer.fit on the engine lowers the loss; afterwards evaluate / predict agree with module.eval() loaded from the
    engine's state_dict (the on-device fold of the running statistics), within the 4b gate."""
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine
    from b200ddl.train import Trainer

    N, S, k = 16, 64, 14
    model = build_model(S, S, 3, 5, dropout=0.0, arch="mobilenetv2", batch_size=N, fine_tune_at=k, batchnorm="training")
    assert isinstance(model, MobileNetV2Engine) and model.batchnorm == "training"
    x, y = _batch(N, S, seed=3)
    tr = Trainer(model, use_graph=use_graph)
    tr.compile(optim.SGD(0.05, momentum=0.9))
    losses = tr.fit([(x, y)] * 10, epochs=3, verbose=0).history["loss"]
    assert losses[-1] < losses[0], losses
    ev = tr.evaluate([(x, y)], verbose=0)
    pred = torch.as_tensor(tr.predict(x.cpu().numpy()), device=DEV).float()
    mod = _module(k, model.state_dict())
    mod.eval()
    xin = x.permute(0, 3, 1, 2).float() / 127.5 - 1.0
    with _no_tf32(), torch.no_grad():
        l32 = mod(xin).float()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            lac = mod(xin).float()
    d_eng, d_ac = _rel(pred, l32), _rel(lac, l32)
    print(f"eval logits distance: engine {d_eng:.3e}, autocast {d_ac:.3e}")
    assert d_eng <= max(4 * d_ac, 2e-2)
    loss32 = float(F.cross_entropy(l32, y))
    assert abs(ev[0] - loss32) <= max(4 * abs(float(F.cross_entropy(lac, y)) - loss32), 2e-2 * loss32)


def test_resume_and_tracking_round_trip(tmp_path):
    """A run saved after 2 steps and resumed in a fresh trainer repeats the uninterrupted loss curve and ends with the
    same running statistics and step counts; a tracking round trip keeps batchnorm, weights and statistics."""
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.tracking.models import load_model, save_model
    from b200ddl.train import Trainer

    N, S, k = 8, 64, 12
    data = [_batch(N, S, seed=20 + i) for i in range(4)]

    def trainer():
        m = build_model(S, S, 3, 5, dropout=0.0, arch="mobilenetv2", batch_size=N, fine_tune_at=k, batchnorm="training")
        t = Trainer(m, use_graph=False)
        t.compile(optim.SGD(0.05, momentum=0.9))
        return t

    full = trainer()
    curve = [full.fit([b], epochs=1, verbose=0).history["loss"][0] for b in data]
    a = trainer()
    part = [a.fit([b], epochs=1, verbose=0).history["loss"][0] for b in data[:2]]
    a.save(str(tmp_path / "ck.pt"))
    b = trainer()
    _ = b.backend.step   # the engine backend attaches the optimizer (and its state) when the step is built
    b.load(str(tmp_path / "ck.pt"))
    part += [b.fit([d], epochs=1, verbose=0).history["loss"][0] for d in data[2:]]
    assert part == pytest.approx(curve, rel=2e-3), (part, curve)
    sa, sb = full.model.state_dict(), b.model.state_dict()
    for n in sa:
        if n.endswith("num_batches_tracked"):
            assert int(sb[n]) == int(sa[n]) == (4 if int(n.split(".")[2]) >= k else 0), n
        elif "running" in n:
            assert _rel(sb[n], sa[n]) <= 1e-3, n
    save_model(b.model, str(tmp_path / "m"))
    back = load_model(str(tmp_path / "m")).model
    assert back.batchnorm == "training" and back.fine_tune_at == k
    sc = back.state_dict()
    assert sorted(sc) == sorted(sb)
    for n in sb:
        check_equal(f"round trip {n}", sc[n], sb[n])


# launches of the parent's fine_tune_at=k training step (tests/test_augment.py PARENT_STEP_LAUNCHES) and the number of
# trainable conv + BatchNorm layers at k
INFERENCE_BN_STEP = {0: 233, 14: 109}
TRAINABLE_LAYERS = {0: 52, 14: 13}


@pytest.mark.parametrize("k", [0, 14])
def test_training_step_launch_count(k):
    """Per trainable layer, training-mode BatchNorm launches 5 more kernels than inference-mode fine-tuning: forward
    bn_finalize + bn_apply, backward bn_bwd_coeffs + bn_bwd_apply, and the inference fold after the optimizer; once per
    step, weight_prep_batched replaces mbv2_ft_finalize + mbv2_ft_refresh (-1).  k=0: 233 + 5*52 - 1 = 492;
    k=14: 109 + 5*13 - 1 = 173."""
    from b200ddl import ops, optim

    expected = {0: 492, 14: 173}[k]
    assert expected == INFERENCE_BN_STEP[k] + 5 * TRAINABLE_LAYERS[k] - 1
    eng = _engine(k, batch=8, size=64)
    assert sum(1 for lay in eng._layers if lay[8] >= k) == TRAINABLE_LAYERS[k]
    x, y = _batch(8, 64)
    from b200ddl.models.resnet_engine import EngineTrainStep

    step = EngineTrainStep(eng, optim.SGD(0.01), use_graph=False)
    step.load(x, y)
    step.run()
    torch.cuda.synchronize()
    n0 = ops.kernel_launches()
    step.load(x, y)
    step.run()
    torch.cuda.synchronize()
    assert ops.kernel_launches() - n0 == expected
