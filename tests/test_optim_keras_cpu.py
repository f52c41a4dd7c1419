"""RMSprop / Adagrad / Adamax / AdamW / Lamb and Keras's gradient clipping on the flat optimizers' CPU path: the update
rules against torch.optim (Lamb against a float64 reimplementation), clipping against torch.nn.utils, validation,
name lookup, checkpoints and two gloo ranks."""
import math

import pytest
import torch

from b200ddl import optim
from b200ddl.parallel import Runner


def _run(ours, theirs_factory, steps=5, n=4096, seed=0, segments=None, grad_scale=1.0):
    """`steps` steps of `ours` on one flat buffer and of the torch optimizer `theirs_factory` returns (None: skipped),
    which gets grad_scale * g (clipping, when `theirs_factory` wants it, is its business)."""
    g = torch.Generator().manual_seed(seed)
    p0 = torch.randn(n, generator=g)
    p = p0.clone()
    grads = torch.zeros(n)
    w16 = torch.zeros(n, dtype=torch.bfloat16)
    ours.grad_scale = grad_scale
    ours.attach(p, grads, w16, segments=segments)
    ref = torch.nn.Parameter(p0.clone())
    theirs = theirs_factory([ref]) if theirs_factory is not None else None
    for _ in range(steps):
        gr = torch.randn(n, generator=g)
        grads.copy_(gr)
        ours.begin_step()
        ours.step()
        if theirs is not None:
            ref.grad = gr * grad_scale
            theirs.step()
    return p, ref.detach(), w16


RMS_CASES = [(0.0, False, 0.0), (0.0, False, 1e-3), (0.9, False, 0.0), (0.9, False, 1e-3), (0.0, True, 0.0),
             (0.0, True, 1e-3), (0.9, True, 1e-3)]


@pytest.mark.parametrize("momentum,centered,wd", RMS_CASES)
def test_rmsprop_matches_torch(momentum, centered, wd):
    p, ref, w16 = _run(optim.RMSprop(1e-2, rho=0.9, momentum=momentum, epsilon=1e-7, centered=centered, weight_decay=wd),
                       lambda ps: torch.optim.RMSprop(ps, lr=1e-2, alpha=0.9, eps=1e-7, momentum=momentum,
                                                      centered=centered, weight_decay=wd))
    assert torch.allclose(p, ref, rtol=1e-5, atol=1e-6)
    assert torch.equal(w16, p.to(torch.bfloat16))


@pytest.mark.parametrize("wd", [0.0, 1e-3])
def test_adagrad_matches_torch(wd):
    p, ref, w16 = _run(optim.Adagrad(1e-1, initial_accumulator_value=0.1, epsilon=1e-7, weight_decay=wd),
                       lambda ps: torch.optim.Adagrad(ps, lr=1e-1, initial_accumulator_value=0.1, eps=1e-7,
                                                      weight_decay=wd))
    assert torch.allclose(p, ref, rtol=1e-5, atol=1e-6)
    assert torch.equal(w16, p.to(torch.bfloat16))


@pytest.mark.parametrize("wd", [0.0, 1e-3])
def test_adamax_matches_torch(wd):
    p, ref, w16 = _run(optim.Adamax(1e-2, beta_1=0.9, beta_2=0.999, epsilon=1e-7, weight_decay=wd),
                       lambda ps: torch.optim.Adamax(ps, lr=1e-2, betas=(0.9, 0.999), eps=1e-7, weight_decay=wd))
    assert torch.allclose(p, ref, rtol=1e-5, atol=1e-6)
    assert torch.equal(w16, p.to(torch.bfloat16))


def test_adamw_matches_torch():
    p, ref, w16 = _run(optim.AdamW(1e-2, beta_1=0.9, beta_2=0.999, epsilon=1e-7, weight_decay=0.05),
                       lambda ps: torch.optim.AdamW(ps, lr=1e-2, betas=(0.9, 0.999), eps=1e-7, weight_decay=0.05))
    assert torch.allclose(p, ref, rtol=1e-4, atol=1e-6)
    assert torch.equal(w16, p.to(torch.bfloat16))


def test_keras_defaults():
    r, a, x, w, l = optim.RMSprop(), optim.Adagrad(), optim.Adamax(), optim.AdamW(), optim.Lamb()
    assert (r.learning_rate, r.rho, r.momentum, r.epsilon, r.centered, r.weight_decay) == (1e-3, 0.9, 0.0, 1e-7, False, 0)
    assert (a.learning_rate, a.initial_accumulator_value, a.epsilon) == (1e-3, 0.1, 1e-7)
    assert (x.beta_1, x.beta_2, x.epsilon) == (0.9, 0.999, 1e-7)
    assert (w.weight_decay, w.epsilon) == (0.004, 1e-7) and l.weight_decay == 0.0
    for o in (r, a, x, w, l):
        assert o.clipnorm is None and o.clipvalue is None and o.global_clipnorm is None and o.clip_mode is None


def lamb_reference(p0, grads, segments, lr, b1, b2, eps, wd):
    """float64 LAMB over the gradient sequence: per segment r = m_hat / (sqrt(v_hat) + eps) + wd p, phi = |p| / |r|
    (1 when either is 0), p -= lr phi r."""
    p = p0.double().clone()
    m = torch.zeros_like(p)
    v = torch.zeros_like(p)
    for t, g in enumerate(grads, 1):
        g = g.double()
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        r = (m / (1 - b1 ** t)) / ((v / (1 - b2 ** t)).sqrt() + eps) + wd * p
        for lo, hi in segments:
            pn, rn = float(p[lo:hi].norm()), float(r[lo:hi].norm())
            phi = pn / rn if pn > 0 and rn > 0 else 1.0
            p[lo:hi] -= lr * phi * r[lo:hi]
    return p


def test_lamb_matches_float64_reference_with_a_zero_segment():
    """3 segments; the middle one has all-zero parameters and gradients, so its phi is 1 and it stays 0."""
    n = 4096
    segs = [(0, 1024), (1024, 2048), (2048, 4096)]
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(n, generator=g)
    p0[1024:2048] = 0
    grads = [torch.randn(n, generator=g) for _ in range(5)]
    for gr in grads:
        gr[1024:2048] = 0
    p = p0.clone()
    gb = torch.zeros(n)
    w16 = torch.zeros(n, dtype=torch.bfloat16)
    o = optim.Lamb(1e-2, weight_decay=0.01).attach(p, gb, w16, segments=segs)
    for gr in grads:
        gb.copy_(gr)
        o.begin_step()
        o.step()
    ref = lamb_reference(p0, grads, segs, 1e-2, 0.9, 0.999, 1e-7, 0.01)
    assert torch.allclose(p.double(), ref, rtol=1e-5, atol=1e-6)
    assert int(p[1024:2048].count_nonzero()) == 0
    assert torch.equal(w16, p.to(torch.bfloat16))
    # the trust ratio matters: a whole-buffer LAMB moves the parameters differently
    whole = lamb_reference(p0, grads, [(0, n)], 1e-2, 0.9, 0.999, 1e-7, 0.01)
    assert not torch.allclose(ref, whole, rtol=1e-4, atol=1e-5)


def _clipped_sgd(clip_kw, torch_clip, grad_scale, segments=None, n=4096):
    p, ref, _ = _run(optim.SGD(0.05, momentum=0.9, weight_decay=1e-3, **clip_kw), None, n=n, segments=segments,
                     grad_scale=grad_scale)
    # the same steps with torch: clip (grad_scale * g), then torch.optim.SGD (coupled weight decay after the clip)
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(n, generator=g)
    par = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([par], lr=0.05, momentum=0.9, weight_decay=1e-3)
    for _ in range(5):
        par.grad = torch.randn(n, generator=g) * grad_scale
        torch_clip(par)
        opt.step()
    return p, par.detach()


@pytest.mark.parametrize("c", [2.0, 1e6])   # the norm is ~64 * grad_scale: the second threshold never clips
def test_global_clipnorm_matches_clip_grad_norm(c):
    p, ref = _clipped_sgd({"global_clipnorm": c}, lambda par: torch.nn.utils.clip_grad_norm_([par], c), 0.5)
    assert torch.allclose(p, ref, rtol=1e-5, atol=1e-6)
    if c > 1e5:
        plain, _, _ = _run(optim.SGD(0.05, momentum=0.9, weight_decay=1e-3), None, grad_scale=0.5)
        assert torch.equal(p, plain)


@pytest.mark.parametrize("c", [3.0, 1e6])
def test_clipnorm_is_per_segment(c):
    segs = [(0, 64), (64, 1088), (1088, 4096)]

    def per_segment(par):
        for lo, hi in segs:
            x = par.grad[lo:hi]
            x.mul_(c / max(float(x.norm()), c))

    p, ref = _clipped_sgd({"clipnorm": c}, per_segment, 2.0, segments=segs)
    assert torch.allclose(p, ref, rtol=1e-5, atol=1e-6)
    if c > 1e5:
        plain, _, _ = _run(optim.SGD(0.05, momentum=0.9, weight_decay=1e-3), None, grad_scale=2.0, segments=segs)
        assert torch.allclose(p, plain, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("c", [0.5, 1e6])
def test_clipvalue_matches_clip_grad_value(c):
    p, ref = _clipped_sgd({"clipvalue": c}, lambda par: torch.nn.utils.clip_grad_value_([par], c), 0.5)
    assert torch.allclose(p, ref, rtol=1e-5, atol=1e-6)
    if c > 1e5:
        plain, _, _ = _run(optim.SGD(0.05, momentum=0.9, weight_decay=1e-3), None, grad_scale=0.5)
        assert torch.allclose(p, plain, rtol=1e-6, atol=1e-7)


def test_clip_options_are_validated():
    with pytest.raises(ValueError):
        optim.Adam(clipnorm=1.0, global_clipnorm=1.0)
    with pytest.raises(ValueError):
        optim.SGD(clipvalue=1.0, clipnorm=2.0)
    for bad in (0.0, -1.0):
        for k in ("clipnorm", "clipvalue", "global_clipnorm"):
            with pytest.raises(ValueError):
                optim.RMSprop(**{k: bad})
    o = optim.SGD(0.1, global_clipnorm=1.0)
    with pytest.raises(ValueError):
        o.clipnorm = 1.0           # a second option
    with pytest.raises(ValueError):
        o.global_clipnorm = 0.0
    o.attach(torch.zeros(8), torch.zeros(8))
    with pytest.raises(ValueError):
        o.global_clipnorm = None   # the mode is fixed once attached
    with pytest.raises(ValueError):
        optim.SGD().attach(torch.zeros(16), torch.zeros(16), segments=[(0, 8), (4, 16)])


def test_threshold_change_takes_effect_at_next_begin_step():
    o = optim.SGD(1.0, global_clipnorm=1.0)
    p, g = torch.zeros(4), torch.full((4,), 2.0)   # |g| = 4
    o.attach(p, g)
    o.begin_step(); o.step()
    assert torch.allclose(p, torch.full((4,), -0.5))
    o.global_clipnorm = 2.0
    o.step()                                        # no begin_step: still the old threshold
    assert torch.allclose(p, torch.full((4,), -1.0))
    o.begin_step(); o.step()
    assert torch.allclose(p, torch.full((4,), -2.0))


def test_repeated_step_does_not_compound_the_global_clip():
    o = optim.SGD(1.0, global_clipnorm=1.0)
    o.grad_scale = 0.5
    p, g = torch.zeros(4), torch.full((4,), 4.0)    # |0.5 g| = 4
    o.attach(p, g)
    o.begin_step()
    for k in range(1, 4):
        o.step()
        assert torch.allclose(p, torch.full((4,), -0.5 * k))


def test_padding_stays_zero_under_every_optimizer_and_clip():
    """A segment's alignment tail (zero parameter, zero gradient) stays exactly zero."""
    segs = [(0, 64), (64, 192)]
    for make in (optim.RMSprop, lambda **k: optim.RMSprop(momentum=0.9, centered=True, **k), optim.Adagrad,
                 optim.Adamax, optim.AdamW, optim.Lamb):
        for clip in ({}, {"clipnorm": 0.1}, {"clipvalue": 0.01}, {"global_clipnorm": 0.1}):
            p = torch.randn(192)
            g = torch.randn(192)
            p[50:64] = 0
            g[50:64] = 0
            o = make(learning_rate=0.1, weight_decay=0.01, **clip).attach(p, g, segments=segs)
            for _ in range(3):
                o.begin_step(); o.step()
            assert int(p[50:64].count_nonzero()) == 0, (o.name, clip)


def test_get_resolves_every_name_and_compile_accepts_a_string():
    from b200ddl.train import Trainer

    for cls in (optim.RMSprop, optim.Adagrad, optim.Adamax, optim.AdamW, optim.Lamb):
        assert optim.get(cls.name) is cls and optim.get(cls.name.lower()) is cls
    model = torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * 4 * 4, 3))
    tr = Trainer(model, device="cpu").compile("adamw")
    assert isinstance(tr.optimizer, optim.AdamW) and tr.optimizer.weight_decay == 0.004
    g = torch.Generator().manual_seed(0)
    y = torch.randint(0, 3, (8,), generator=g)
    x = (torch.randint(0, 20, (8, 4, 4, 3), generator=g) + (y * 80)[:, None, None, None]).to(torch.uint8)
    h = Trainer(model, device="cpu").compile("rmsprop").fit([(x, y)] * 10, epochs=2, verbose=0)
    assert h.history["loss"][-1] < h.history["loss"][0]
    assert len(tr.backend.optimizer.segments) == 2   # one segment per parameter tensor


def test_autolog_records_the_new_optimizer_names(tmp_path):
    from b200ddl import tracking
    from b200ddl.train import Trainer

    tracking.set_tracking_uri(str(tmp_path / "mlruns"))
    tracking.set_experiment("optimizers")
    model = torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * 4 * 4, 3))
    x = torch.zeros(4, 4, 4, 3, dtype=torch.uint8)
    y = torch.zeros(4, dtype=torch.int64)
    tracking.autolog(log_models=False)
    try:
        for name in ("RMSprop", "Adagrad", "Adamax", "AdamW", "Lamb"):
            tr = Trainer(model, device="cpu").compile(optim.get(name)(global_clipnorm=1.0))
            with tracking.start_run() as run:
                tr.fit([(x, y)], epochs=1, verbose=0)
            assert tracking.get_run(run.info.run_id).data.params["optimizer_name"] == name
    finally:
        tracking.autolog(disable=True)


@pytest.mark.parametrize("name", ["Adagrad", "Lamb"])
def test_save_load_round_trips_the_state(name, tmp_path):
    """Trainer.save / load restores the state (Adagrad's accumulator starts at 0.1, not 0): the resumed run continues
    exactly as the uninterrupted one."""
    from b200ddl.train import Trainer

    def make():
        torch.manual_seed(0)
        return torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * 4 * 4, 8), torch.nn.ReLU(),
                                   torch.nn.Linear(8, 3))

    g = torch.Generator().manual_seed(1)
    data = [(torch.randint(0, 255, (4, 4, 4, 3), generator=g).to(torch.uint8), torch.randint(0, 3, (4,), generator=g))
            for _ in range(6)]
    a = Trainer(make(), device="cpu").compile(optim.get(name)(1e-2))
    assert name != "Adagrad" or float(a.optimizer.state["acc"].min()) == pytest.approx(0.1)
    a.fit(data[:3], epochs=1, verbose=0)
    a.save(str(tmp_path / "ck.pt"))
    a.fit(data[3:], epochs=1, verbose=0)
    b = Trainer(make(), device="cpu").compile(optim.get(name)(1e-2))
    b.load(str(tmp_path / "ck.pt"))
    assert b.optimizer.t == 3
    b.fit(data[3:], epochs=1, verbose=0)
    assert torch.equal(a.backend.flat.params, b.backend.flat.params)
    for k, v in a.optimizer.state.items():
        assert torch.equal(v, b.optimizer.state[k]), k


def test_two_ranks_lamb_with_global_clipnorm_equals_one_process_on_the_mean_gradient():
    """Module backend, DistributedOptimizer(Lamb(global_clipnorm)) on 2 gloo ranks with different data: identical
    replicas, equal to one process that steps Lamb on the mean of the two ranks' gradients."""
    def make_model():
        torch.manual_seed(0)
        return torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * 4 * 4, 8), torch.nn.ReLU(),
                                   torch.nn.Linear(8, 3))

    def batches(rank):
        g = torch.Generator().manual_seed(10 + rank)
        return [(torch.randint(0, 255, (4, 4, 4, 3), generator=g).to(torch.uint8),
                 torch.randint(0, 3, (4,), generator=g)) for _ in range(4)]

    def fn():
        import b200ddl.parallel as hvd
        from b200ddl.train import Trainer
        from b200ddl.utils import checksum_across_ranks

        hvd.init()
        opt = hvd.DistributedOptimizer(optim.Lamb(1e-2, weight_decay=0.01, global_clipnorm=0.05), bucket_mb=0.0001)
        tr = Trainer(make_model(), device="cpu").compile(optimizer=opt)
        tr.fit(batches(hvd.rank()), epochs=1, verbose=0)
        return {"same": checksum_across_ranks(tr.backend.flat.params), "params": tr.backend.flat.params.clone()}

    out = Runner(np=2, driver_log_verbosity="none", force_cpu=True).run(fn)
    assert out["same"], "replicas diverged"

    # one process: the same Lamb on the mean gradient of the two ranks' batches
    from b200ddl.train.flat import FlatParams

    model = make_model()
    flat = FlatParams(model)
    opt = optim.Lamb(1e-2, weight_decay=0.01, global_clipnorm=0.05).attach(flat.params, flat.grads,
                                                                            segments=flat.ranges)
    from b200ddl.models.preprocess import preprocess_tensor

    for (x0, y0), (x1, y1) in zip(batches(0), batches(1)):
        opt.begin_step()
        mean = torch.zeros_like(flat.grads)
        for x, y in ((x0, y0), (x1, y1)):
            flat.zero_grad()
            torch.nn.functional.cross_entropy(model(preprocess_tensor(x)).float(), y).backward()
            mean += flat.grads / 2
        flat.grads.copy_(mean)
        opt.step()
    assert torch.allclose(out["params"], flat.params, rtol=1e-5, atol=1e-6), \
        float((out["params"] - flat.params).abs().max())
    assert math.isfinite(float(flat.params.sum()))
