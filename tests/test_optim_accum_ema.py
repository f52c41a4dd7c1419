"""Gradient accumulation and weight EMA on the GPU: the `grad_accumulate` / `ema_update` kernels (csrc/optim.cu) bit for
bit against the torch path, their argument checks, CUDA-graph replay of the optimizer, both engines' two step
variants, the end of `fit`, launch counts and two ranks."""
from __future__ import annotations

import math

import pytest
import torch

from exact_util import DEV, Guarded, check_equal

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
RED_CAP = 132 * 8
OPT_N = 4 * (2 * RED_CAP * 256 + 5)   # the capped grid loops twice with a ragged tail


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def guarded(t):
    g = Guarded(tuple(t.shape), t.dtype)
    g.t.copy_(t)
    g._bits = g._as_int(g.buf).clone()
    return g


def ema_hyper(d, overwrite):
    h = torch.zeros(16, dtype=torch.float32)
    h[10], h[11], h[12] = d, 1.0 - d, 1.0 if overwrite else 0.0
    return h.to(DEV)


# ================================================================================================ kernels
@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("mode", [0, 1])
def test_grad_accumulate_matches_torch_path(mode, n):
    """mode 0: accum += g; mode 1: g = (accum + g) / n, accum = 0.  The reference is the CPU torch path (IEEE add and
    division, as the kernel's __fadd_rn / __fdiv_rn)."""
    e = _ops()
    g = gen(20 + mode)
    gr = torch.randn(OPT_N, device=DEV, generator=g)
    acc = torch.randn(OPT_N, device=DEV, generator=g) * 3
    G, A = guarded(gr), guarded(acc)
    e.grad_accumulate(G.t, A.t, n, mode)
    torch.cuda.synchronize()
    rg, ra = gr.cpu(), acc.cpu()
    if mode == 0:
        ra = ra + rg
    else:
        rg = (ra + rg) / n
        ra = torch.zeros_like(ra)
    check_equal(f"grad_accumulate mode {mode} g", G.t.cpu(), rg)
    check_equal(f"grad_accumulate mode {mode} accum", A.t.cpu(), ra)
    G.check_guards("g")
    A.check_guards("accum")


@pytest.mark.parametrize("with_p16", [True, False])
@pytest.mark.parametrize("d,overwrite", [(0.99, False), (0.0, False), (0.9, True)])
def test_ema_update_matches_torch_path(d, overwrite, with_p16):
    e = _ops()
    g = gen(30)
    p, ema = torch.randn(OPT_N, device=DEV, generator=g), torch.randn(OPT_N, device=DEV, generator=g)
    P, E = guarded(p), guarded(ema)
    p16 = Guarded((OPT_N,), BF)
    h = ema_hyper(d, overwrite)
    e.ema_update(P.t, E.t, p16.t if with_p16 else None, h)
    torch.cuda.synchronize()
    hc = h.cpu()
    ref = ema.cpu() * hc[10] + p.cpu() * hc[11]
    check_equal("ema", E.t.cpu(), ref)
    check_equal("p", P.t.cpu(), ref if overwrite else p.cpu())
    if with_p16 and overwrite:
        check_equal("p16", p16.t, P.t.to(BF))
    else:
        assert bool(p16.untouched().all()), "p16 written without an overwrite"
    for nm, t in (("p", P), ("ema", E), ("p16", p16)):
        t.check_guards(nm)


def test_malformed_calls_raise_before_any_launch():
    e = _ops()
    n = 1024
    g, acc, p, ema = (torch.zeros(n, device=DEV) for _ in range(4))
    p16 = torch.zeros(n, device=DEV, dtype=BF)
    h = torch.zeros(16, device=DEV)
    bad = [
        lambda: e.grad_accumulate(g, acc, 2, 2),                                   # mode
        lambda: e.grad_accumulate(g, acc, 0, 1),                                   # steps
        lambda: e.grad_accumulate(g.double(), acc, 2, 0),                          # dtype
        lambda: e.grad_accumulate(g, acc[:n - 4], 2, 0),                           # size
        lambda: e.grad_accumulate(g[:n - 2], acc[:n - 2], 2, 0),                   # n % 4
        lambda: e.grad_accumulate(torch.zeros(n + 4, device=DEV)[1:n + 1], acc, 2, 0),   # alignment
        lambda: e.grad_accumulate(g, g, 2, 0),                                     # aliasing
        lambda: e.grad_accumulate(g, torch.zeros(2, n // 2, device=DEV).t(), 2, 0),   # contiguity
        lambda: e.grad_accumulate(g.cpu(), acc.cpu(), 2, 0),                       # device
        lambda: e.ema_update(p, ema, p16, h[:8]),                                  # hyper < 16
        lambda: e.ema_update(p, ema, p16.float(), h),                              # p16 dtype
        lambda: e.ema_update(p, ema[:n - 4], None, h),                             # size
        lambda: e.ema_update(p, p, None, h),                                       # aliasing
        lambda: e.ema_update(p, ema, p.view(BF)[:n], h),                           # p16 inside p
        lambda: e.ema_update(p.double(), ema, None, h),                            # dtype
        lambda: e.ema_update(torch.zeros(n + 4, device=DEV)[1:n + 1], ema, None, h),   # alignment
    ]
    buf = torch.zeros(2 * n, device=DEV)
    bad.append(lambda: e.grad_accumulate(buf[:n], buf[n // 2:n // 2 + n], 2, 0))   # partial overlap
    torch.cuda.synchronize()
    before = e.launch_count()
    for i, f in enumerate(bad):
        with pytest.raises(RuntimeError):
            f()
        assert e.launch_count() == before, f"case {i} launched"


# ================================================================================================ optimizer
def _flat_opt(name="Adam", **kw):
    from b200ddl import optim

    return optim.get(name)(learning_rate=1e-2, weight_decay=1e-3, **kw)


def test_graph_replay_equals_eager_launches():
    """Adam with n = 3, EMA (overwrite every 2 updates) and clipnorm: one graph per variant, replayed as `is_update_step`
    selects, equals eager steps bit for bit."""
    n = 4 * 40000
    segs = [(0, 4096), (4096, 100000), (100000, n)]
    g0 = gen(40)
    p0 = torch.randn(n, device=DEV, generator=g0)
    grads = [torch.randn(n, device=DEV, generator=g0) for _ in range(8)]
    kw = dict(gradient_accumulation_steps=3, use_ema=True, ema_overwrite_frequency=2, clipnorm=5.0)
    out = []
    for use_graph in (False, True):
        p = p0.clone()
        gb = torch.zeros(n, device=DEV)
        w16 = torch.zeros(n, device=DEV, dtype=BF)
        opt = _flat_opt(**kw).attach(p, gb, w16, segments=segs)
        graphs = {}
        if use_graph:
            snap = {k: v.clone() for k, v in opt.state.items()}
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for u in (True, False):
                    opt.step(u)
            torch.cuda.current_stream().wait_stream(s)
            for u in (True, False):
                graphs[u] = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graphs[u]):
                    opt.step(u)
            torch.cuda.synchronize()
            p.copy_(p0)
            for k, v in opt.state.items():
                v.copy_(snap[k])
        for gr in grads:
            gb.copy_(gr)
            opt.begin_step()
            if use_graph:
                graphs[opt.is_update_step].replay()
            else:
                opt.step()
        torch.cuda.synchronize()
        out.append((p.clone(), w16.clone(), {k: v.clone() for k, v in opt.state.items()}))
    (pe, we, se), (pg, wg, sg) = out
    check_equal("params", pg, pe)
    check_equal("w16", wg, we)
    for k in se:
        check_equal(k, sg[k], se[k])
    assert not torch.equal(pe, p0)


# ================================================================================================ engines
def _images(batch, size, seed=1):
    g = gen(seed)
    x = torch.randint(0, 256, (batch, size, size, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (batch,), device=DEV, generator=g)
    return x, y


def _resnet(batch=8):
    from b200ddl.models.resnet_engine import ResNet50Engine

    return ResNet50Engine(batch=batch, num_classes=5, image_size=224, seed=0)


def _mobilenet(k, batch=8, batchnorm="inference", size=64):
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    return MobileNetV2Engine(batch=batch, num_classes=5, image_size=size, dropout=0.0, seed=0, fine_tune_at=k,
                             batchnorm=batchnorm)


def test_resnet_engine_accumulates_then_updates_from_both_gradients():
    """n = 2 (SGD with momentum): micro-batch 1 leaves the parameters unchanged and accum equals its gradient; micro-batch
    2 applies the torch-path update of (g1 + g2) / 2 from the engine's own gradient buffers.  The combine is bit-exact;
    the kernel's update is one fma where the torch path rounds twice: one rounding of the parameter and 2^-22 of the
    update."""
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    eng = _resnet()
    opt = optim.SGD(0.05, momentum=0.9, gradient_accumulation_steps=2)
    step = EngineTrainStep(eng, opt, use_graph=True)
    (x1, y1), (x2, y2) = _images(8, 224, seed=1), _images(8, 224, seed=2)
    step.load(x1, y1)
    step.run()                      # captures both variants, then replays the accumulation graph
    torch.cuda.synchronize()
    p0 = eng.params.clone()
    assert step.graph is not None and step.accum_graph is not None
    g1 = eng.grads.clone()
    check_equal("accum after micro-batch 1", opt.state["accum"], g1)
    P0 = p0.cpu()
    # micro-batch 2, eager (the same launches as the update graph), with its gradient read before the optimizer
    opt.begin_step()
    assert opt.is_update_step
    eng.set_input(x2, y2)
    eng.forward(training=True)
    eng.backward()
    torch.cuda.synchronize()
    G2 = eng.grads.cpu().clone()
    S = {k: v.cpu().clone() for k, v in opt.state.items()}
    opt.step()
    eng.refresh_derived_weights()
    torch.cuda.synchronize()
    assert int(opt.state["accum"].count_nonzero()) == 0
    cpu = optim.SGD(0.05, momentum=0.9, gradient_accumulation_steps=2)
    P = P0.clone()
    cpu.attach(P, G2, None, segments=opt.segments)
    cpu.t = 1
    for k, v in S.items():
        cpu.state[k].copy_(v)
    cpu.begin_step()
    cpu.step()
    got = eng.params.cpu().double()
    upd = (P.double() - P0.double()).abs()
    err = (got - P.double()).abs()
    bound = 2.0 ** -24 * P.double().abs() * 2 + 2.0 ** -22 * upd + 2.0 ** -30 * float(upd.max())
    assert bool((err <= bound).all()), f"max excess {float((err - bound).max()):.3e}"
    assert float(upd.max()) > 0


def test_resnet_update_graph_applies_the_torch_path_update():
    """n = 2, both micro-batches replayed from the captured graphs.  The optimizer copies the gradient it is handed
    into a side buffer first (a copy captured into both graphs), so the test sees each micro-batch's own gradient g1,
    g2 as the graphs computed them.  The update graph's combine leaves exactly (g1 + g2) / 2 in the gradient buffer and
    zeroes accum, and its parameters equal the torch path fed g1 (in accum) and g2 (bound as above)."""
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    class Snooping(optim.SGD):
        snap = None

        def step(self, update=None):
            self.snap.copy_(self.grads)
            super().step(update)

    eng = _resnet()
    opt = Snooping(0.05, momentum=0.9, gradient_accumulation_steps=2)
    step = EngineTrainStep(eng, opt, use_graph=True)
    opt.snap = torch.empty_like(eng.grads)   # allocated before capture
    (x1, y1), (x2, y2) = _images(8, 224, seed=1), _images(8, 224, seed=2)
    step.load(x1, y1)
    step.run()                      # captures both variants, then replays the accumulation graph
    torch.cuda.synchronize()
    assert step.graph is not None and step.accum_graph is not None
    g1 = opt.snap.cpu().clone()
    check_equal("accum after micro-batch 1", opt.state["accum"].cpu(), g1)
    P0 = eng.params.cpu().clone()
    S = {k: v.cpu().clone() for k, v in opt.state.items()}
    step.load(x2, y2)
    step.run()                      # t = 2: the update graph
    torch.cuda.synchronize()
    assert opt.t == 2 and opt.updates == 1
    g2 = opt.snap.cpu().clone()
    assert not torch.equal(g1, g2)
    check_equal("accum after the update", opt.state["accum"].cpu(), torch.zeros_like(g1))
    check_equal("combined gradient", eng.grads.cpu(), (g1 + g2) / 2)
    cpu = optim.SGD(0.05, momentum=0.9, gradient_accumulation_steps=2)
    P = P0.clone()
    cpu.attach(P, g2.clone(), None, segments=opt.segments)
    cpu.t = 1
    for k, v in S.items():
        cpu.state[k].copy_(v)
    cpu.begin_step()
    cpu.step()
    got = eng.params.cpu().double()
    upd = (P.double() - P0.double()).abs()
    err = (got - P.double()).abs()
    bound = 2.0 ** -24 * P.double().abs() * 2 + 2.0 ** -22 * upd + 2.0 ** -30 * float(upd.max())
    assert bool((err <= bound).all()), f"max excess {float((err - bound).max()):.3e}"
    assert float(upd.max()) > 0


def test_resnet_micro_batch_1_leaves_parameters_bit_identical():
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    eng = _resnet()
    opt = optim.Adam(1e-3, gradient_accumulation_steps=2, use_ema=True)
    step = EngineTrainStep(eng, opt, use_graph=True)
    step.capture()
    p_before, w_before = eng.params.clone(), eng.w16.clone()
    x, y = _images(8, 224, seed=3)
    step.load(x, y)
    step.run()
    torch.cuda.synchronize()
    check_equal("params after micro-batch 1", eng.params, p_before)
    check_equal("w16 after micro-batch 1", eng.w16, w_before)
    check_equal("accum after micro-batch 1", opt.state["accum"], eng.grads)
    check_equal("ema after micro-batch 1", opt.state["ema"], p_before)
    assert float(eng.grads.abs().max()) > 0


def test_mobilenet_head_accumulation_equals_the_double_batch():
    """fine_tune_at=19 (head only), dropout 0, SGD: n = 2 over x1 then x2 (batch 8 each) moves the parameters as one step
    of a batch-16 engine on their concatenation.  The head gradient comes from bf16 features, which the two batch shapes
    may round differently: one bf16 rounding (2^-8) of either side, so the bound is 2^-7 of the largest update."""
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    (x1, y1), (x2, y2) = _images(8, 64, seed=5), _images(8, 64, seed=6)
    a = _mobilenet(19, batch=8)
    sa = EngineTrainStep(a, optim.SGD(0.5, gradient_accumulation_steps=2), use_graph=True)
    p0 = a.params.clone()
    for x, y in ((x1, y1), (x2, y2)):
        sa.load(x, y)
        sa.run()
    b = _mobilenet(19, batch=16)
    sb = EngineTrainStep(b, optim.SGD(0.5), use_graph=True)
    check_equal("same initial weights", b.params, p0)
    sb.load(torch.cat([x1, x2]), torch.cat([y1, y2]))
    sb.run()
    torch.cuda.synchronize()
    ua, ub = (a.params - p0).double(), (b.params - p0).double()
    assert float(ub.abs().max()) > 0
    err = float((ua - ub).abs().max())
    assert err <= 2.0 ** -7 * float(ub.abs().max()), f"{err:.3e} vs update {float(ub.abs().max()):.3e}"


def _padding_views(eng, flat, k):
    """Slices of a flat buffer that are padding in `eng`'s layout (pointwise cout/cin padding, fc rows, gaps)."""
    out = []
    for lay in eng._layers:
        if lay[0] == "pw" and lay[8] >= k:
            s = eng.spec[lay[1] + ".weight"]
            w = flat[s.offset:s.offset + s.numel].view(s.shape).clone()
            w[:lay[4], :lay[3]] = 0
            out.append((lay[1], w))
    s = eng.spec["fc.weight"]
    out.append(("fc rows", flat[s.offset:s.offset + s.numel].view(s.shape)[eng.num_classes:]))
    for s in eng.param_specs:
        lo, hi = s.offset + s.numel, -(-(s.offset + s.numel) // 64) * 64
        out.append(("gap after " + s.name, flat[lo:hi]))
    return out


def test_mobilenet_bn_training_partial_accumulation_evaluates_with_current_statistics():
    """fine_tune_at=14, batchnorm="training", n = 2: an accumulation step moves the running statistics and folds them
    into the inference affine, so evaluation right after it equals evaluation after an explicit re-derivation; accum
    and ema keep the padding at zero."""
    from b200ddl import optim
    from b200ddl.train import Trainer

    k = 14
    eng = _mobilenet(k, batchnorm="training")
    tr = Trainer(eng).compile(optim.Adam(1e-3, gradient_accumulation_steps=2, use_ema=True))
    x, y = _images(8, 64, seed=7)
    xv, yv = _images(8, 64, seed=8)
    before = tr.evaluate([(xv, yv)])
    r0 = eng.running.clone()
    tr.backend.train_batch(x, y)           # micro-batch 1: accumulation only
    tr.backend.pop_results()
    torch.cuda.synchronize()
    assert not torch.equal(eng.running, r0), "running statistics did not move"
    after = tr.evaluate([(xv, yv)])
    logits = tr.predict(xv.cpu().numpy())
    eng.sync_weights()                     # re-derive every inference weight from params + running statistics
    logits2 = tr.predict(xv.cpu().numpy())
    assert after != before
    assert (logits == logits2).all(), "evaluation after accumulation used stale statistics"
    for _ in range(2):                     # t = 3: one update applied, one micro-batch accumulated
        tr.backend.train_batch(x, y)
    tr.backend.pop_results()
    torch.cuda.synchronize()
    for st in ("accum", "ema"):
        for nm, v in _padding_views(eng, tr.optimizer.state[st], k):
            assert int(v.count_nonzero()) == 0, f"{st}: padding of {nm} is no longer zero"


@pytest.mark.parametrize("arch", ["resnet50", "mobilenetv2"])
def test_ema_overwrite_and_fit_end_on_both_engines(arch):
    """use_ema, ema_overwrite_frequency=3, n = 1: the parameters equal the average after steps 1 (d = 0), 3 and 6 only;
    after `fit` evaluation equals a fresh engine loaded with the EMA weights."""
    from b200ddl import optim
    from b200ddl.train import Callback, Trainer

    make = (lambda: _resnet()) if arch == "resnet50" else (lambda: _mobilenet(14, batchnorm="training"))
    size = 224 if arch == "resnet50" else 64
    eng = make()
    tr = Trainer(eng).compile(optim.SGD(0.05, momentum=0.9, use_ema=True, ema_momentum=0.8, ema_overwrite_frequency=3))
    equal = []

    class Watch(Callback):
        def on_train_batch_end(self, batch, logs=None):
            torch.cuda.synchronize()
            equal.append(torch.equal(eng.params, tr.optimizer.state["ema"]))

    data = [_images(8, size, seed=10 + i) for i in range(7)]
    tr.fit(data, epochs=1, verbose=0, callbacks=[Watch()])
    assert equal == [True, False, True, False, False, True, False], equal
    torch.cuda.synchronize()
    check_equal("params after fit", eng.params, tr.optimizer.state["ema"])
    xv, yv = _images(8, size, seed=99)
    got = tr.evaluate([(xv, yv)])
    fresh = make()
    fresh.load_state_dict(tr.get_weights())
    ref = Trainer(fresh).compile(optim.SGD(0.05)).evaluate([(xv, yv)])
    assert got[0] == pytest.approx(ref[0], rel=1e-6, abs=1e-6) and got[1] == ref[1]


# ================================================================================================ launch counts
# Eager launches of one ResNet-50 step at batch 32 with SGD and the defaults (tests/test_augment.py
# PARENT_STEP_LAUNCHES).  Accumulation adds the combine pass to an update step and replaces clip + update (+ EMA) by
# one accumulation pass on every other step; EMA adds one pass to an update step; clipnorm is three passes.
BASE = 395


@pytest.mark.parametrize("kw,update,accumulate", [
    ({}, BASE, None),
    ({"gradient_accumulation_steps": 2}, BASE + 1, BASE),
    ({"use_ema": True}, BASE + 1, None),
    ({"gradient_accumulation_steps": 2, "use_ema": True}, BASE + 2, BASE),
    ({"gradient_accumulation_steps": 2, "use_ema": True, "clipnorm": 1.0}, BASE + 5, BASE),
])
def test_step_launch_counts(kw, update, accumulate):
    from b200ddl import ops, optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    eng = _resnet(batch=32)
    x, y = _images(32, 224)
    opt = optim.SGD(0.01, **kw)
    step = EngineTrainStep(eng, opt, use_graph=False)
    step.capture()
    counts = {}
    for _ in range(2):
        step.load(x, y)
        torch.cuda.synchronize()
        n0 = ops.kernel_launches()
        step.run()
        torch.cuda.synchronize()
        counts.setdefault(opt.is_update_step, ops.kernel_launches() - n0)
    assert counts[True] == update
    assert counts.get(False) == accumulate


# ================================================================================================ two GPUs
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_accumulation_and_ema_stay_identical_and_turn_fused_update_off():
    from b200ddl.parallel import Runner

    def fn():
        import torch
        import b200ddl.parallel as hvd
        from b200ddl import optim
        from b200ddl.models.resnet_engine import ResNet50Engine
        from b200ddl.train import Trainer
        from b200ddl.utils import checksum_across_ranks

        hvd.init()
        dev = torch.device("cuda", hvd.local_rank())
        g = torch.Generator(device=dev).manual_seed(hvd.rank())
        data = [(torch.randint(0, 256, (8, 224, 224, 3), device=dev, dtype=torch.uint8, generator=g),
                 torch.randint(0, 5, (8,), device=dev, generator=g)) for _ in range(5)]
        opt = hvd.DistributedOptimizer(optim.SGD(0.05, momentum=0.9, gradient_accumulation_steps=2, use_ema=True),
                                       fused_update=True)
        eng = ResNet50Engine(batch=8, num_classes=5, image_size=224, seed=0, device=dev)
        tr = Trainer(eng, device=dev).compile(opt)
        tr.broadcast_state(0)
        h = tr.fit(data, epochs=1, verbose=0)
        torch.cuda.synchronize()
        return (checksum_across_ranks(eng.params), checksum_across_ranks(opt.opt.state["ema"]), opt.fused_update,
                h.history["loss"][-1])

    out = Runner(np=2, driver_log_verbosity="none").run(fn)
    assert out[0] and out[1], "replicas diverged"
    assert out[2] is False and math.isfinite(out[3])
