"""MobileNetV2 fine-tuning on the native engine (`fine_tune_at`, BatchNorm in inference mode), on the GPU.

Kernel cases (csrc/mobilenet_bwd.cu) follow test_elementwise_exact.py: integer or power-of-two data so that the float64
reference is exact, outputs between NaN guard bands, mismatch reports that name the element.  Every sum below stays under
2^24 in magnitude, so the fp32 partial sums are exact in any order and equality is demanded; the kernels' summation depth
(module comment of mobilenet_bwd.cu) only matters above that.

Engine cases compare with the fp32 torch module `FrozenBaseClassifier(fine_tune_at=k)` on the same weights, gated as the
ResNet-50 gradient check is (DESIGN.md 4b): the engine's relative L2 distance to fp32 against the module's own distance
under bf16 autocast.
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


# ================================================================================================ ReLU6 mask + sum
MASK_VARIANTS = [(relu6, g2) for relu6 in (True, False) for g2 in (False, True)]
MASK_M = {64: 40_000, 192: 333}   # C=64: more rows than one pass of the capped grid (1056 blocks x 32 rows)


@pytest.mark.parametrize("C", sorted(MASK_M))
@pytest.mark.parametrize("relu6,use_g2", MASK_VARIANTS)
def test_relu6_mask_reduce(C, relu6, use_g2):
    """dz = (g1 [+ g2]) * [0 < y < 6] (or unmasked), bf16; sum[c] += sum dz.  y hits exactly 0, exactly 6, 5.96875 (the
    bf16 value below 6) and tiny positives; the call also runs in place (dz is g1)."""
    e = _ops()
    M = MASK_M[C]
    g = gen(C + 2 * relu6 + use_g2)
    g1 = ints((M, C), -3, 3, g)
    g2 = ints((M, C), -3, 3, g) if use_g2 else None
    special = torch.tensor([0.0, 6.0, 5.96875, 2.0 ** -100, 2.0 ** -126, 3.0, -1.0], device=DEV, dtype=torch.float64)
    y = special[torch.randint(0, special.numel(), (M, C), device=DEV, generator=g)]
    gs = g1 + g2 if use_g2 else g1
    dz = gs * ((y > 0) & (y < 6)) if relu6 else gs
    yb = bf(y)
    assert bool(((yb.double() > 0) & (yb.double() < 2.0 ** -90)).any()), "tiny positive y lost in bf16"
    for inplace in (False, True):
        g1b = bf(g1)
        out = Guarded((M, C), BF) if not inplace else None
        dzt = g1b if inplace else out.t
        s = Guarded((C,), torch.float32, fill=0.0)
        e.relu6_mask_reduce(g1b, bf(g2) if use_g2 else None, yb, dzt, s.t, relu6)
        torch.cuda.synchronize()
        name = f"relu6_mask_reduce C={C} relu6={relu6} g2={use_g2} inplace={inplace}"
        check_equal(name, dzt, to_bf16_exact(dz), lambda m, c: f"[row {m}, channel {c}]")
        check_equal(name + " sum", s.t.double(), dz.sum(0))
        s.check_guards(name + " sum")
        if out is not None:
            out.check_guards(name)


# ================================================================================================ depthwise
DW_CASES = [(2, 13, 11, 64), (1, 15, 17, 192), (2, 7, 10, 960)]   # odd H / W; Wo % 4 != 0 at stride 1 and 2
DW_WGRAD_BIG = (32, 64, 64, 64)    # more 4-pixel strips than one pass of the capped grid (528 CTAs x 32 lanes)


def _dw_ref(x, w, dz, stride):
    """float64 gradients of F.conv2d(groups=C): (dx for filter w, dW [9, C])."""
    C = x.shape[-1]
    xx = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    ww = w.t().reshape(C, 1, 3, 3).clone().requires_grad_(True)
    y = F.conv2d(xx, ww, stride=stride, padding=1, groups=C)
    y.backward(dz.permute(0, 3, 1, 2))
    return xx.grad.permute(0, 2, 3, 1), ww.grad.reshape(C, 9).t()


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: "x".join(map(str, c)))
def test_dw_dgrad(case, stride):
    """dx = conv_transpose(dz, scale * w) of the depthwise 3x3, bit-exact against float64."""
    e = _ops()
    N, H, W, C = case
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    g = gen(3 * C + stride)
    dz = ints((N, Ho, Wo, C), -2, 2, g)
    w = ints((9, C), -2, 2, g) * 0.5
    sc = pow2((C,), -1, 1, g)
    dx_ref, _ = _dw_ref(torch.zeros(N, H, W, C, device=DEV, dtype=torch.float64), w * sc, dz, stride)
    out = Guarded((N, H, W, C), BF)
    e.dw_dgrad(bf(dz), f32(w), f32(sc), out.t, stride)
    torch.cuda.synchronize()
    name = f"dw_dgrad {case} stride={stride}"
    check_equal(name, out.t, to_bf16_exact(dx_ref), lambda n, h, ww, c: f"[thread for input ({h}, {ww // 4 * 4}) + {ww % 4}]")
    out.check_guards(name)


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("case", DW_CASES + [DW_WGRAD_BIG], ids=lambda c: "x".join(map(str, c)))
def test_dw_wgrad(case, stride):
    """G[9, C] = depthwise weight gradient, accumulated into G (prefilled with an integer to check it adds)."""
    e = _ops()
    N, H, W, C = case
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    g = gen(5 * C + stride)
    x = ints((N, H, W, C), -2, 2, g)
    dz = ints((N, Ho, Wo, C), -2, 2, g)
    _, gw = _dw_ref(x, torch.zeros(9, C, device=DEV, dtype=torch.float64), dz, stride)
    G = Guarded((9, C), torch.float32, fill=1.0)
    e.dw_wgrad(bf(dz), bf(x), G.t, stride)
    torch.cuda.synchronize()
    name = f"dw_wgrad {case} stride={stride}"
    check_equal(name, G.t.double(), gw + 1.0, lambda t, c: f"[tap {t}, channel {c}]")
    G.check_guards(name)


STEM_CASES = [(2, 34, 30), (8, 128, 128)]   # the second: more pixels than one pass of the capped grid (1056 x 16)


@pytest.mark.parametrize("case", STEM_CASES, ids=lambda c: "x".join(map(str, c)))
def test_mbv2_stem_wgrad(case):
    """G[27, 32] of the 3x3/2 stem over bf16(x * mul + add), k = (r*3 + s)*3 + c; padded dz channels are ignored."""
    e = _ops()
    N, H, W = case
    g = gen(H)
    x = torch.randint(126, 131, (N, H, W, 3), device=DEV, dtype=torch.uint8, generator=g)
    dz = ints((N, H // 2, W // 2, 64), -2, 2, g)
    dz[..., 32:] = 7.0   # never read
    xx = (x.double() - 128.0).permute(0, 3, 1, 2)
    wt = torch.zeros(32, 3, 3, 3, device=DEV, dtype=torch.float64, requires_grad=True)
    F.conv2d(xx, wt, stride=2, padding=1).backward(dz[..., :32].permute(0, 3, 1, 2))
    ref = wt.grad.permute(2, 3, 1, 0).reshape(27, 32)
    G = Guarded((27, 32), torch.float32, fill=0.0)
    e.mbv2_stem_wgrad(x, bf(dz), G.t, 1.0, -128.0)
    torch.cuda.synchronize()
    check_equal(f"mbv2_stem_wgrad {case}", G.t.double(), ref, lambda k, c: f"[k {k}, channel {c}]")
    G.check_guards(f"mbv2_stem_wgrad {case}")


# ================================================================================================ finalize / refresh
def test_mbv2_ft_finalize():
    """dW = s*G, dgamma = invstd*(<W_c, G_c> - mean*dbeta), dbeta = sum(dz): a pointwise row (bf16 W [cp, cin_p]), a
    depthwise row (fp32 [9, Cp]) and a stem row (fp32 [27, 32]), power-of-two s / invstd, exact."""
    e = _ops()
    g = gen(11)
    layers = [("pw", 40, 64, 96), ("dw", 72, 128, 128), ("stem", 32, 64, 27)]   # kind, c, cp, cin_p / count
    shapes = {"pw": lambda c, cp, ci: (cp, ci), "dw": lambda c, cp, ci: (9, cp), "stem": lambda c, cp, ci: (27, 32)}
    total, offs = 0, []
    for kind, c, cp, ci in layers:
        n = shapes[kind](c, cp, ci)
        offs.append((total, total + n[0] * n[1], total + n[0] * n[1] + 128))
        total += n[0] * n[1] + 256
    params = torch.zeros(total, device=DEV)
    grads = torch.full((total,), float("nan"), device=DEV)
    rows, keep, expect = [], [], []
    for (kind, c, cp, ci), (wo, go, bo) in zip(layers, offs):
        shp = shapes[kind](c, cp, ci)
        n = shp[0] * shp[1]
        W = ints(shp, -3, 3, g) * 0.5
        G = ints(shp, -40, 40, g)
        s, inv = pow2((cp,), -2, 2, g), pow2((cp,), -3, 1, g)
        mean, db = ints((cp,), -4, 4, g) * 0.25, ints((cp,), -100, 100, g)
        params[wo:wo + n] = W.flatten().float()
        grads[wo:wo + n] = G.flatten().float()
        if kind == "pw":
            dot = (W[:c] * G[:c]).sum(1)
            dW = G.clone()
            dW[:c] *= s[:c, None]
            count, cs, js = ci, ci, 1
        else:
            dot = (W[:, :c] * G[:, :c]).sum(0)
            dW = G.clone()
            dW[:, :c] *= s[None, :c]
            count, cs, js = shp[0], 1, shp[1]
        dev = [t.float().contiguous() for t in (s, inv, mean, db)]
        keep += dev
        rows.append([c, count, cs, js, int(kind == "pw"), wo, wo, go, bo] + [t.data_ptr() for t in dev])
        expect.append((kind, wo, n, dW, go, inv[:c] * (dot - mean[:c] * db[:c]), bo, db[:c]))
    w16 = params.to(BF)
    e.mbv2_ft_finalize(params, w16, grads, torch.tensor(rows, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    for kind, wo, n, dW, go, dg, bo, dbt in expect:
        check_equal(f"finalize {kind} dW", grads[wo:wo + n].double(), dW.flatten())
        check_equal(f"finalize {kind} dgamma", grads[go:go + dg.numel()].double(), dg)
        check_equal(f"finalize {kind} dbeta", grads[bo:bo + dbt.numel()].double(), dbt)


def test_mbv2_ft_refresh():
    """scale / shift bit-identical to the host fold (engine `_affine`) on random gamma, beta and statistics; padded
    channels 1 / 0; pointwise dgrad filter wd[ci, co] = bf16(scale[co] * W[co, ci])."""
    e = _ops()
    torch.manual_seed(0)
    c, cp, cin_p = 40, 64, 96
    gamma, beta = torch.randn(c), torch.randn(c)
    rmean, rvar = torch.randn(c), torch.rand(c) * 3 + 0.01
    inv = torch.rsqrt(rvar + 1e-5)
    sc = gamma * inv
    sh = beta - rmean * sc
    W = torch.zeros(cp, cin_p)
    W[:c, :70] = torch.randn(c, 70)
    params = torch.zeros(cp * cin_p + 128, device=DEV)
    params[:cp * cin_p] = W.flatten().to(DEV)
    params[cp * cin_p:cp * cin_p + c] = gamma.to(DEV)
    params[cp * cin_p + 64:cp * cin_p + 64 + c] = beta.to(DEV)
    inv_d = torch.zeros(cp, device=DEV)
    inv_d[:c] = inv.to(DEV)
    mean_d = torch.zeros(cp, device=DEV)
    mean_d[:c] = rmean.to(DEV)
    scale, shift = Guarded((cp,), torch.float32), Guarded((cp,), torch.float32)
    wd = Guarded((cin_p, cp), BF)
    row = [c, cp, cin_p, cp * cin_p, cp * cin_p + 64, 0, inv_d.data_ptr(), mean_d.data_ptr(), scale.t.data_ptr(),
           shift.t.data_ptr(), wd.t.data_ptr()]
    e.mbv2_ft_refresh(params, torch.tensor([row], dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    exp_sc, exp_sh = torch.ones(cp), torch.zeros(cp)
    exp_sc[:c], exp_sh[:c] = sc, sh
    check_equal("refresh scale", scale.t.cpu(), exp_sc)
    check_equal("refresh shift", shift.t.cpu(), exp_sh)
    check_equal("refresh dgrad filter", wd.t.cpu(), (W * exp_sc[:, None]).t().to(BF))
    for name, t in (("scale", scale), ("shift", shift), ("wd", wd)):
        t.check_guards("refresh " + name)


# ================================================================================================ bindings
def test_malformed_inputs_raise():
    """Every new binding rejects dtype, shape, C % 8, stride and alignment errors before launching."""
    e = _ops()
    f = lambda *s: torch.zeros(*s, device=DEV)                        # noqa: E731
    b = lambda *s: torch.zeros(*s, device=DEV, dtype=BF)              # noqa: E731
    u8 = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.uint8)    # noqa: E731
    C, M = 64, 32
    y = b(M, C)
    mis_b = b(M * C + 8)[1:M * C + 1].view(M, C)
    x4, dz4 = b(1, 8, 8, C), b(1, 8, 8, C)
    tbl = lambda n: torch.zeros(1, n, device=DEV, dtype=torch.int64)  # noqa: E731
    calls = {
        "relu6_mask_reduce: short sum": lambda: e.relu6_mask_reduce(y, None, y, y, f(C - 8), True),
        "relu6_mask_reduce: g2 size": lambda: e.relu6_mask_reduce(y, b(M - 1, C), y, y, f(C), True),
        "relu6_mask_reduce: misaligned dz": lambda: e.relu6_mask_reduce(y, None, y, mis_b, f(C), True),
        "relu6_mask_reduce: C % 8": lambda: e.relu6_mask_reduce(b(M, 12), None, b(M, 12), b(M, 12), f(12), True),
        "relu6_mask_reduce: fp32 g1": lambda: e.relu6_mask_reduce(f(M, C), None, y, y, f(C), True),
        "dw_dgrad: stride 3": lambda: e.dw_dgrad(dz4, f(9 * C), f(C), x4, 3),
        "dw_dgrad: dz shape": lambda: e.dw_dgrad(b(1, 8, 8, C), f(9 * C), f(C), x4, 2),
        "dw_dgrad: short w": lambda: e.dw_dgrad(dz4, f(9 * C - 4), f(C), x4, 1),
        "dw_dgrad: misaligned w": lambda: e.dw_dgrad(dz4, f(9 * C + 4)[1:9 * C + 1], f(C), x4, 1),
        "dw_dgrad: channel mismatch": lambda: e.dw_dgrad(b(1, 8, 8, 128), f(9 * C), f(C), x4, 1),
        "dw_wgrad: short G": lambda: e.dw_wgrad(dz4, x4, f(9 * C - 1), 1),
        "dw_wgrad: bf16 G": lambda: e.dw_wgrad(dz4, x4, b(9 * C), 1),
        "dw_wgrad: 3-d x": lambda: e.dw_wgrad(dz4, b(8, 8, C), f(9 * C), 1),
        "mbv2_stem_wgrad: odd H": lambda: e.mbv2_stem_wgrad(u8(1, 9, 8, 3), b(1, 4, 4, C), f(27 * 32), 1.0, 0.0),
        "mbv2_stem_wgrad: dz grid": lambda: e.mbv2_stem_wgrad(u8(1, 8, 8, 3), b(1, 4, 3, C), f(27 * 32), 1.0, 0.0),
        "mbv2_stem_wgrad: ldc < 32": lambda: e.mbv2_stem_wgrad(u8(1, 8, 8, 3), b(1, 4, 4, 16), f(27 * 32), 1.0, 0.0),
        "mbv2_stem_wgrad: short G": lambda: e.mbv2_stem_wgrad(u8(1, 8, 8, 3), b(1, 4, 4, C), f(27 * 31), 1.0, 0.0),
        "mbv2_ft_finalize: table width": lambda: e.mbv2_ft_finalize(f(256), b(256), f(256), tbl(12)),
        "mbv2_ft_finalize: short grads": lambda: e.mbv2_ft_finalize(f(256), b(256), f(255), tbl(13)),
        "mbv2_ft_finalize: fp32 w16": lambda: e.mbv2_ft_finalize(f(256), f(256), f(256), tbl(13)),
        "mbv2_ft_finalize: host table": lambda: e.mbv2_ft_finalize(f(256), b(256), f(256), tbl(13).cpu()),
        "mbv2_ft_refresh: table width": lambda: e.mbv2_ft_refresh(f(256), tbl(10)),
        "mbv2_ft_refresh: int32 table": lambda: e.mbv2_ft_refresh(f(256), tbl(11).int()),
        "mbv2_ft_refresh: empty table": lambda: e.mbv2_ft_refresh(f(256), tbl(11)[:0]),
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


def test_case_tables_cover_every_launch_site():
    """The cases reach all four relu6_mask_reduce_kernel instances (relu6 x g2) with a grid-stride loop that runs more
    than once, both strides of dw_dgrad_kernel and dw_wgrad_kernel (the latter also past one pass of its grid), the
    stem weight gradient past one pass, and one table row of every layer kind in finalize."""
    assert set(MASK_VARIANTS) == {(a, b) for a in (True, False) for b in (False, True)}
    assert max(MASK_M[c] for c in MASK_M if c == 64) > 1056 * 32
    N, H, W, C = DW_WGRAD_BIG
    assert N * H * ((W + 3) // 4) > (528 // ((C // 8 + 7) // 8)) * 32
    n, h, w = STEM_CASES[-1]
    assert n * (h // 2) * (w // 2) > 1056 * 16
    assert all(case[2] % 4 and ((case[2] - 1) // 2 + 1) % 4 for case in DW_CASES)


# ================================================================================================ engine
def _engine(k, batch=8, size=64, seed=0, dropout=0.0):
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    return MobileNetV2Engine(batch=batch, num_classes=5, image_size=size, dropout=dropout, seed=seed, fine_tune_at=k)


def _batch(batch, size, seed=1):
    g = gen(seed)
    x = torch.randint(0, 256, (batch, size, size, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (batch,), device=DEV, generator=g)
    return x, y


def _grad_as_torch(eng, name):
    """Engine gradient of `name` in the torch parameter's shape (padding dropped)."""
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


def _run_steps(eng, opt, x, y, steps):
    from b200ddl.models.resnet_engine import EngineTrainStep

    step = EngineTrainStep(eng, opt, use_graph=False)
    out = []
    for _ in range(steps):
        step.load(x, y)
        step.run()
        out.append(step.result())
    torch.cuda.synchronize()
    return out


def test_fine_tune_at_19_matches_frozen_engine():
    """fine_tune_at=19 trains the head only and launches exactly what the frozen engine launches: the first step's loss
    and logits are bit-identical, and after 3 SGD steps the losses, logits, gradients and parameters differ from the
    frozen engine's no more than two frozen-engine runs differ from each other (the head's weight-gradient GEMM adds
    with fp32 atomics, so the frozen engine itself is not bit-reproducible from step 2 on)."""
    from b200ddl import optim

    x, y = _batch(8, 96)
    res = []
    for k in (None, 19, None):
        eng = _engine(k, size=96, dropout=0.5)
        losses = _run_steps(eng, optim.SGD(0.05, momentum=0.9), x, y, 1)
        first = (losses[0], eng.logits.clone())
        losses += _run_steps(eng, optim.SGD(0.05, momentum=0.9), x, y, 2)
        res.append((first, torch.tensor(losses), eng.logits.clone(), eng.grads[:eng.flat_numel].clone(),
                    eng.params.clone()))
    frozen, ft, frozen2 = res
    assert ft[0][0] == frozen[0][0]
    check_equal("fine_tune_at=19 vs frozen: first-step logits", ft[0][1], frozen[0][1])
    for i, name in ((1, "losses"), (2, "logits"), (3, "grads"), (4, "params")):
        spread = float((frozen2[i].double() - frozen[i].double()).abs().max())
        diff = float((ft[i].double() - frozen[i].double()).abs().max())
        scale = float(frozen[i].double().abs().max())
        assert diff <= max(4 * spread, 1e-6 * scale), f"{name}: fine_tune_at=19 differs by {diff}, frozen runs by {spread}"


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.mark.parametrize("k", [0, 1, 4, 14, 18])
def test_gradients_match_torch_module(k):
    """Every trainable gradient against the fp32 `FrozenBaseClassifier(fine_tune_at=k)` on the same weights: the
    engine's relative L2 distance to fp32 may be at most 4x the module's own distance under bf16 autocast (floor
    2e-2 for tensors autocast happens to reproduce almost exactly)."""
    from b200ddl.models.mobilenet import FrozenBaseClassifier, MobileNetV2Base

    N, S = (16, 64) if k != 4 else (8, 96)
    eng = _engine(k, batch=N, size=S)
    eng.build(training=True)
    x, y = _batch(N, S, seed=k)
    eng.set_input(x, y)
    eng.forward(training=True)
    eng.backward()
    torch.cuda.synchronize()
    base = MobileNetV2Base()
    mod = FrozenBaseClassifier(base, base.out_channels, 5, 0.0, True, k).to(DEV)
    mod.load_state_dict({n: v.to(DEV) for n, v in eng.state_dict().items()})
    mod.train()
    xin = x.permute(0, 3, 1, 2).float() / 127.5 - 1.0
    grads = {}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False   # a true fp32 reference
    for mode in ("fp32", "autocast"):
        mod.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "autocast"):
            loss = F.cross_entropy(mod(xin).float(), y)
        loss.backward()
        grads[mode] = {n: p.grad.detach().float().cpu() for n, p in mod.named_parameters() if p.requires_grad}
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    names = [s.name for s in eng.param_specs]
    assert sorted(names) == sorted(grads["fp32"]), "engine and module train different tensors"
    worst = []
    for n in names:
        d_eng = _rel(_grad_as_torch(eng, n), grads["fp32"][n])
        d_ac = _rel(grads["autocast"][n], grads["fp32"][n])
        worst.append((d_eng / max(4 * d_ac, 2e-2), n, d_eng, d_ac))
    worst.sort(reverse=True)
    print("worst gradient distances (ratio to gate, name, engine, autocast):", worst[:5])
    assert worst[0][0] <= 1.0, f"gradient off: {worst[:5]}"


@pytest.mark.parametrize("opt_name", ["sgd_wd", "adam", "adam_wd", "adadelta_wd"])
def test_frozen_part_and_padding_stay_fixed(opt_name):
    """After optimizer steps, features[:k] weights and every running statistic are bit-unchanged, the trainable layers
    did change, and the zero padding of the pointwise weights is still exactly zero."""
    from b200ddl import optim

    k = 14
    make = {"sgd_wd": lambda: optim.SGD(0.05, momentum=0.9, weight_decay=1e-2), "adam": lambda: optim.Adam(1e-3),
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
        if "running" in n or "num_batches" in n or (feat is not None and feat < k):
            check_equal(f"{opt_name}: {n} changed", sd1[n], v)
        elif feat is not None:
            moved += int(not torch.equal(sd1[n], v))
    assert moved > 0, "no trainable base tensor moved"
    for lay in eng._layers:
        if lay[0] == "pw" and lay[8] >= k:
            w = eng.p(lay[1] + ".weight")
            pad = w.clone()
            pad[:lay[4], :lay[3]] = 0
            assert int(pad.count_nonzero()) == 0, f"{opt_name}: padding of {lay[1]} is no longer zero"


@pytest.mark.parametrize("use_graph", [True, False])
def test_fit_lowers_loss_and_eval_uses_trained_weights(use_graph):
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine
    from b200ddl.train import Trainer

    N, S = 16, 64
    model = build_model(S, S, 3, 5, dropout=0.0, arch="mobilenetv2", batch_size=N, fine_tune_at=14)
    assert isinstance(model, MobileNetV2Engine) and model.fine_tune_at == 14
    x, y = _batch(N, S, seed=3)
    tr = Trainer(model, use_graph=use_graph)
    tr.compile(optim.SGD(0.1, momentum=0.9))
    hist = tr.fit([(x, y)] * 30, epochs=1, verbose=0)
    losses = hist.history["loss"] if hasattr(hist, "history") else hist
    ev = tr.evaluate([(x, y)], verbose=0)
    fresh = _engine(14, batch=N, size=S)
    fresh.load_state_dict(model.state_dict())
    fresh.build(training=False)
    fresh.set_input(x, y)
    fresh.forward(training=False)
    torch.cuda.synchronize()
    first = _engine(14, batch=N, size=S)
    first.build(training=False)
    first.set_input(x, y)
    first.forward(training=False)
    torch.cuda.synchronize()
    loss_trained, loss_init = fresh.loss_and_acc()[0], first.loss_and_acc()[0]
    assert loss_trained < loss_init - 0.05, (loss_init, loss_trained, losses)
    assert abs(ev[0] - loss_trained) < 1e-6, (ev, loss_trained)
    pred = tr.predict(x.cpu().numpy())
    check_equal("predict after fit vs inference build", torch.as_tensor(pred, device=DEV).float(), fresh.logits)


def test_tracking_round_trip(tmp_path):
    from b200ddl import optim
    from b200ddl.tracking.models import load_model, save_model
    from b200ddl.train import Trainer

    eng = _engine(16, batch=8, size=64)
    x, y = _batch(8, 64)
    _run_steps(eng, optim.SGD(0.05), x, y, 2)
    save_model(eng, str(tmp_path / "m"))
    tr = load_model(str(tmp_path / "m"))
    assert tr.model.fine_tune_at == 16
    a, b = eng.state_dict(), tr.model.state_dict()
    assert sorted(a) == sorted(b)
    for n in a:
        check_equal(f"round trip {n}", b[n], a[n])
