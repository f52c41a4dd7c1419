"""Keras's gradient accumulation and weight EMA on the flat optimizers' CPU path: validation, the accumulation / EMA
rules against a hand-written loop for every optimizer and clip mode, the overwrite schedule, the end of `fit`, and
checkpoints.

The reference loop writes out the new rules (sum the micro-batch gradients in order, divide by n, count updates
u = t // n, average the weights with d = 0 at u = 1, overwrite every f updates) and delegates the update itself to an
optimizer without either option, whose rules `test_optim_cpu.py` / `test_optim_keras_cpu.py` check against torch.optim.
It repeats the fp32 operations in the kernels' order, so the comparison is bit for bit."""
import pytest
import torch

from b200ddl import optim
from b200ddl.optim.fused import EMA_DECAY, EMA_OVERWRITE, EMA_REST, HYPER_SLOTS
from b200ddl.train import Trainer

NAMES = ["SGD", "Adam", "Adadelta", "RMSprop", "Adagrad", "Adamax", "AdamW", "Lamb"]
CLIPS = [{}, {"clipnorm": 0.5}, {"clipvalue": 0.01}, {"global_clipnorm": 0.5}]
SEGS = [(0, 64), (64, 448), (448, 1024)]
N = 1024


def make_opt(name, **kw):
    extra = {"momentum": 0.9} if name == "SGD" else {}
    return optim.get(name)(learning_rate=1e-2, weight_decay=1e-3, **extra, **kw)


def grads_seq(steps, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(N, generator=g), [torch.randn(N, generator=g) for _ in range(steps)]


def reference(name, clip, n, p0, grads, momentum=0.99, freq=None):
    """(params, accum, ema) after the micro-batch gradients `grads`, from the rules written out."""
    p = p0.clone()
    w16 = torch.zeros(N, dtype=torch.bfloat16)
    g = torch.zeros(N)
    inner = make_opt(name, **clip).attach(p, g, w16, segments=SEGS)
    acc = torch.zeros(N)
    ema = p0.clone()
    d_f32 = torch.tensor(momentum, dtype=torch.float32)
    for t, gr in enumerate(grads, 1):
        if t % n:
            acc = acc + gr
            continue
        g.copy_((acc + gr) / n)
        acc = torch.zeros(N)
        inner.begin_step()            # inner.t == u = t // n: the bias corrections count updates
        assert inner.t == t // n
        inner.step()
        u = t // n
        d = d_f32 if u > 1 else torch.tensor(0.0)
        d1 = torch.tensor(1.0 - (momentum if u > 1 else 0.0), dtype=torch.float32)
        ema = ema * d + p * d1
        if freq is not None and u % freq == 0:
            p.copy_(ema)
            w16.copy_(p)
    return p, acc, ema, w16


def run(opt, p0, grads):
    p = p0.clone()
    g = torch.zeros(N)
    w16 = torch.zeros(N, dtype=torch.bfloat16)
    opt.attach(p, g, w16, segments=SEGS)
    for gr in grads:
        g.copy_(gr)
        opt.begin_step()
        opt.step()
    return p, w16


# ------------------------------------------------------------------------------------------------ arguments
def test_defaults_and_validation():
    o = optim.Adam()
    assert (o.gradient_accumulation_steps, o.use_ema, o.ema_momentum, o.ema_overwrite_frequency) == (None, False, 0.99,
                                                                                                      None)
    for bad in (1, 0, -2, 2.0, True, "2"):
        with pytest.raises(ValueError):
            optim.SGD(gradient_accumulation_steps=bad)
    for bad in (-0.1, 1.01, float("nan")):
        with pytest.raises(ValueError):
            optim.SGD(use_ema=True, ema_momentum=bad)
    for bad in (0, -1, 1.5, False):
        with pytest.raises(ValueError):
            optim.SGD(use_ema=True, ema_overwrite_frequency=bad)
    for ok in (0.0, 1.0):
        assert optim.SGD(use_ema=True, ema_momentum=ok).ema_momentum == ok
    # as Keras, the EMA arguments are only checked with use_ema
    o = optim.SGD(ema_momentum=2.0, ema_overwrite_frequency=0)
    assert not o.use_ema and "ema" not in o.attach(torch.zeros(8), torch.zeros(8)).state
    o = optim.SGD(gradient_accumulation_steps=2)
    o.attach(torch.zeros(8), torch.zeros(8))
    o.begin_step()
    assert not o.is_update_step
    o.begin_step()
    assert o.is_update_step and o.updates == 1
    with pytest.raises(ValueError):
        optim.SGD().attach(torch.zeros(8), torch.zeros(8)).step(update=False)


@pytest.mark.parametrize("name", sorted(set(optim.OPTIMIZERS)))
def test_get_round_trips_the_arguments(name):
    o = optim.get(name)(gradient_accumulation_steps=3, use_ema=True, ema_momentum=0.9, ema_overwrite_frequency=2,
                        clipnorm=1.0)
    assert (o.gradient_accumulation_steps, o.use_ema, o.ema_momentum, o.ema_overwrite_frequency) == (3, True, 0.9, 2)
    assert o.accumulation_steps == 3 and o.clip_mode == "clipnorm"
    o.attach(torch.ones(16), torch.zeros(16))
    assert torch.equal(o.state["accum"], torch.zeros(16)) and torch.equal(o.state["ema"], torch.ones(16))


# ------------------------------------------------------------------------------------------------ the rules
@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("clip", CLIPS, ids=["noclip", "clipnorm", "clipvalue", "global_clipnorm"])
@pytest.mark.parametrize("name", NAMES)
def test_accumulation_and_ema_match_the_rules(name, clip, n):
    """7 micro-batches: two updates at n = 3 (and a partial accumulation of one), three at n = 2."""
    p0, grads = grads_seq(7)
    opt = make_opt(name, gradient_accumulation_steps=n, use_ema=True, **clip)
    p, w16 = run(opt, p0, grads)
    rp, racc, rema, rw16 = reference(name, clip, n, p0, grads)
    assert opt.t == 7 and opt.updates == 7 // n
    assert torch.equal(p, rp)
    assert torch.equal(w16, rw16)
    assert torch.equal(opt.state["accum"], racc)
    assert torch.equal(opt.state["ema"], rema)
    assert not torch.equal(p, p0) and not torch.equal(rema, rp)


@pytest.mark.parametrize("name", NAMES)
def test_defaults_are_the_plain_optimizer(name):
    """n = 1 and use_ema=False: no new state, hyper slots 10-12 untouched, and step(update=None) / step(update=True)
    are the optimizer's plain step."""
    p0, grads = grads_seq(4, seed=1)
    plain = make_opt(name)
    p, w16 = run(plain, p0, grads)
    assert set(plain.state) == set(make_opt(name).attach(torch.zeros(8), torch.zeros(8)).state)
    assert "accum" not in plain.state and "ema" not in plain.state
    assert torch.equal(plain._hyper[EMA_DECAY:EMA_OVERWRITE + 1], torch.zeros(3))
    explicit = make_opt(name, gradient_accumulation_steps=None, use_ema=False)
    q = p0.clone()
    g = torch.zeros(N)
    explicit.attach(q, g, torch.zeros(N, dtype=torch.bfloat16), segments=SEGS)
    for gr in grads:
        g.copy_(gr)
        explicit.begin_step()
        explicit.step(update=True)
    assert torch.equal(p, q)
    # bias corrections at n = 1 count steps as before
    if name in ("Adam", "Adamax", "AdamW", "Lamb"):
        assert float(plain._hyper[6]) == pytest.approx(1 - 0.9 ** 4)


def test_ema_with_n1_is_keras_and_the_overwrite_schedule():
    """SGD, n = 2, f = 3: the parameters become the average at updates 3 and 6 (t = 6, 12); at n = 1 the average
    moves every step."""
    p0, grads = grads_seq(14, seed=2)
    opt = make_opt("SGD", gradient_accumulation_steps=2, use_ema=True, ema_momentum=0.9, ema_overwrite_frequency=3)
    p = p0.clone()
    g = torch.zeros(N)
    w16 = torch.zeros(N, dtype=torch.bfloat16)
    opt.attach(p, g, w16, segments=SEGS)
    replaced = []
    for t, gr in enumerate(grads, 1):
        g.copy_(gr)
        opt.begin_step()
        assert float(opt._hyper[EMA_OVERWRITE]) == (1.0 if t in (6, 7, 12, 13) else 0.0)
        assert float(opt._hyper[EMA_DECAY]) == (0.0 if t < 4 else pytest.approx(0.9))
        assert float(opt._hyper[EMA_DECAY] + opt._hyper[EMA_REST]) == pytest.approx(1.0)
        opt.step()
        if torch.equal(p, opt.state["ema"]):
            replaced.append(t)
    # the average starts as the parameters (t = 1), the first update sets it to them (d = 0, t = 2), accumulation steps
    # change neither (t = 3, 7, 13), and the overwrites at updates 3 and 6 make them equal again
    assert replaced == [1, 2, 3, 6, 7, 12, 13]
    rp, _, rema, rw16 = reference("SGD", {}, 2, p0, grads, momentum=0.9, freq=3)
    assert torch.equal(p, rp) and torch.equal(opt.state["ema"], rema) and torch.equal(w16, rw16)
    # at n = 1 the average moves on every step, as Keras's does
    opt1 = make_opt("SGD", use_ema=True, ema_momentum=0.9)
    run(opt1, p0, grads[:3])
    ema = p0.clone()
    q = p0.clone()
    inner = make_opt("SGD").attach(q, torch.zeros(N), segments=SEGS)
    for t, gr in enumerate(grads[:3], 1):
        inner.grads.copy_(gr)
        inner.begin_step()
        inner.step()
        d = 0.9 if t > 1 else 0.0
        ema = ema.double() * d + q.double() * (1 - d)
    assert torch.allclose(opt1.state["ema"].double(), ema, rtol=1e-6, atol=1e-7)


# ------------------------------------------------------------------------------------------------ Trainer
def make_model():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * 4 * 4, 8), torch.nn.ReLU(),
                               torch.nn.Linear(8, 3))


def make_data(k, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, 255, (4, 4, 4, 3), generator=g).to(torch.uint8), torch.randint(0, 3, (4,), generator=g))
            for _ in range(k)]


def test_fit_ends_with_the_moving_average():
    data = make_data(5)
    tr = Trainer(make_model(), device="cpu").compile(optim.Adam(1e-2, use_ema=True, ema_momentum=0.5,
                                                                gradient_accumulation_steps=2))
    opt = tr.optimizer
    seen = []
    orig = opt.finalize_variable_values

    def spy():
        seen.append((tr.backend.flat.params.clone(), opt.state["ema"].clone()))
        orig()

    opt.finalize_variable_values = spy
    tr.fit(data, epochs=1, verbose=0)
    assert len(seen) == 1
    live, ema = seen[0]
    assert not torch.equal(live, ema)
    assert torch.equal(tr.backend.flat.params, ema)
    # the module's own parameters are views of the flat buffer: evaluation sees the average
    lin = tr.model[3]
    assert torch.equal(lin.bias.detach(), ema[:3])


def test_on_train_end_sees_the_moving_average():
    """As Keras's fit: the weights are the average before `on_train_end`, so a callback that saves or logs the model
    there gets the weights the trainer keeps."""
    from b200ddl.train import Callback

    data = make_data(4)
    tr = Trainer(make_model(), device="cpu").compile(optim.SGD(0.1, use_ema=True, ema_momentum=0.5))
    seen = {}

    class AtEnd(Callback):
        def on_train_batch_end(self, batch, logs=None):
            seen["live differs"] = not torch.equal(tr.backend.flat.params, tr.optimizer.state["ema"])

        def on_train_end(self, logs=None):
            seen["params"] = tr.backend.flat.params.clone()
            seen["ema"] = tr.optimizer.state["ema"].clone()
            seen["weights"] = tr.get_weights()

    tr.fit(data, epochs=1, verbose=0, callbacks=[AtEnd()])
    assert seen["live differs"]
    assert torch.equal(seen["params"], seen["ema"])
    own = tr.get_weights()
    assert all(torch.equal(seen["weights"][k], own[k]) for k in own)


def test_checkpoint_mid_accumulation_resumes_bit_for_bit(tmp_path):
    """n = 3, saved at t = 4 (one micro-batch in accum): the resumed run equals the uninterrupted one."""
    data = make_data(7)
    make_opt3 = lambda: optim.Adam(1e-2, gradient_accumulation_steps=3, clipnorm=0.5)
    a = Trainer(make_model(), device="cpu").compile(make_opt3())
    a.fit(data, epochs=1, verbose=0)
    b = Trainer(make_model(), device="cpu").compile(make_opt3())
    b.fit(data[:4], epochs=1, verbose=0)
    assert b.optimizer.t == 4 and bool(b.optimizer.state["accum"].abs().sum() > 0)
    b.save(str(tmp_path / "ck.pt"))
    c = Trainer(make_model(), device="cpu").compile(make_opt3())
    c.load(str(tmp_path / "ck.pt"))
    assert torch.equal(c.optimizer.state["accum"], b.optimizer.state["accum"])
    c.fit(data[4:], epochs=1, verbose=0)
    assert c.optimizer.t == 7
    assert torch.equal(a.backend.flat.params, c.backend.flat.params)
    for k, v in a.optimizer.state.items():
        assert torch.equal(v, c.optimizer.state[k]), k


def test_ema_checkpoint_round_trip_and_reseeding(tmp_path):
    data = make_data(4)
    a = Trainer(make_model(), device="cpu").compile(optim.SGD(0.1, use_ema=True))
    a.fit(data, epochs=1, verbose=0)
    a.backend.train_batch(*data[0])   # outside fit: the average and the weights differ again
    a.save(str(tmp_path / "ema.pt"))
    b = Trainer(make_model(), device="cpu").compile(optim.SGD(0.1, use_ema=True))
    b.load(str(tmp_path / "ema.pt"))
    assert torch.equal(b.optimizer.state["ema"], a.optimizer.state["ema"])
    assert not torch.equal(b.optimizer.state["ema"], b.backend.flat.params)
    # a checkpoint without an average: it starts from the loaded weights
    plain = Trainer(make_model(), device="cpu").compile(optim.SGD(0.1))
    plain.fit(data, epochs=1, verbose=0)
    plain.save(str(tmp_path / "plain.pt"))
    plain.save_weights(str(tmp_path / "w.pt"))
    for load in ("load", "load_weights"):
        c = Trainer(make_model(), device="cpu").compile(optim.SGD(0.1, use_ema=True))
        c.fit(data[:2], epochs=1, verbose=0)
        getattr(c, load)(str(tmp_path / ("plain.pt" if load == "load" else "w.pt")))
        assert torch.equal(c.backend.flat.params, plain.backend.flat.params)
        assert torch.equal(c.optimizer.state["ema"], c.backend.flat.params), load
    # an average in the checkpoint, resumed without EMA: ignored
    d = Trainer(make_model(), device="cpu").compile(optim.SGD(0.1))
    d.load(str(tmp_path / "ema.pt"))
    assert "ema" not in d.optimizer.state


def test_hyper_slots_fit_the_array():
    assert EMA_OVERWRITE < HYPER_SLOTS
