"""Knowledge distillation without a GPU: `train.losses.Distillation`'s validation, the torch reference
`distillation_reference` against float64 and autograd, and training with a torch teacher on the module backend
(frozen teacher, logged terms, evaluate, checkpoints, the teacher broadcast on two gloo ranks)."""
from __future__ import annotations

import math

import pytest
import torch

from b200ddl import optim
from b200ddl.models.augment import (Augmentation, augment_key, distillation_head_reference, distillation_reference,
                                     mix_params_reference, soft_head_reference)
from b200ddl.parallel import Runner
from b200ddl.train import CategoricalCrossentropy, Distillation, Trainer

U32 = 2.0 ** -24   # fp32 unit roundoff


def _net(seed, S=8, K=5, hidden=16):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * S * S, hidden), torch.nn.ReLU(),
                               torch.nn.Linear(hidden, K))


def _data(n_batches=4, B=8, S=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_batches):
        y = torch.randint(0, 5, (B,), generator=g)
        x = (torch.randint(0, 60, (B, S, S, 3), generator=g) + (y * 45).view(B, 1, 1, 1)).to(torch.uint8)
        out.append((x, y))
    return out


class _FakeEngine:
    """Just enough of a native engine for `Distillation`'s checks (they read attributes only)."""
    param_specs = ()

    def __init__(self, batch=8, image_size=224, num_classes=5, device="cuda:0"):
        self.batch, self.image_size, self.num_classes, self.device = batch, image_size, num_classes, torch.device(device)

    def forward_logits(self, *a, **k):
        pass

    def bind_grad_buffer(self, *a):
        pass


# ------------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("field, bad", [("alpha", -0.1), ("alpha", 1.5), ("alpha", float("nan")), ("alpha", True),
                                        ("alpha", "0.5"), ("temperature", 0.0), ("temperature", -1.0),
                                        ("temperature", float("inf")), ("temperature", float("nan")),
                                        ("temperature", False), ("label_smoothing", 1.5),
                                        ("label_smoothing", float("nan")), ("label_smoothing", True)])
def test_validation_names_the_field(field, bad):
    with pytest.raises(ValueError, match=field):
        Distillation(_net(0), **{field: bad})


def test_defaults_are_the_keras_examples():
    d = Distillation(_net(0))
    assert (d.alpha, d.temperature, d.label_smoothing) == (0.1, 3.0, 0.0)
    Distillation(_net(0), alpha=0, temperature=1e-3)   # closed at alpha = 0 and 1, open at T = 0
    Distillation(_net(0), alpha=1)


def test_teacher_checks():
    with pytest.raises(ValueError, match="teacher"):
        Distillation("resnet50")
    student = _net(0)
    with pytest.raises(ValueError, match="teacher is the student"):
        Trainer(student, device="cpu").compile(optim.SGD(0.1), loss=Distillation(student))
    with pytest.raises(ValueError, match="native engines or both torch modules"):
        Trainer(student, device="cpu").compile(optim.SGD(0.1), loss=Distillation(_FakeEngine()))
    with pytest.raises(ValueError, match="native engines or both torch modules"):
        Distillation(student).check_student(_FakeEngine())
    s = _FakeEngine()
    Distillation(_FakeEngine()).check_student(s)
    for field, v in (("batch", 16), ("image_size", 192), ("num_classes", 1000), ("device", "cuda:1")):
        with pytest.raises(ValueError, match=field):
            Distillation(_FakeEngine(**{field: v})).check_student(s)


def test_compile_accepts_distillation_with_mixing_and_keeps_eps():
    from b200ddl.models import build_model

    mixed = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", augmentation=Augmentation(cutmix=1.0))
    tr = Trainer(mixed, device="cpu").compile(optim.SGD(0.1), loss=Distillation(_net(1, S=32), label_smoothing=0.2))
    assert tr.backend.label_smoothing == 0.2 and tr.distillation is not None


# ------------------------------------------------------------------------------------------------ reference
def _logits(B, K, seed, spread=4.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, K, generator=g) * spread).float()


def _mix_rows(B, mode, seed=3):
    if mode is None:
        return None
    aug = Augmentation(**{mode: 0.4})
    return mix_params_reference(aug, B, 16, 16, augment_key(seed, 0), 5)


@pytest.mark.parametrize("mode", [None, "mixup", "cutmix"])
@pytest.mark.parametrize("T", [1.0, 3.0, 10.0])
@pytest.mark.parametrize("alpha", [0.0, 0.1, 1.0])
def test_reference_autograd_matches_float64(mode, T, alpha):
    """The fp32 reference's autograd gradient and losses against the float64 closed form.  Bound: every fp32 log-softmax
    entry is off by at most c u (|z|max + log K + 2) with c = 8 (subtraction of the max, log, the sum of K exps each
    within 2u, the division by T); exp turns that into a relative error of the same size on p, q, r, so
    |d dlogit_k| <= c u (|z|max / min(T, 1) + log K + 2) (alpha (p_k + t_k) + (1 - alpha) T (q_k + r_k)) + a few u, and
    each loss term is off by that times its size plus its own K-term sum (K u |terms|)."""
    B, K, eps = 7, 10, 0.1
    s, t = _logits(B, K, 1), _logits(B, K, 2)
    y = torch.randint(0, K, (B,), generator=torch.Generator().manual_seed(4))
    mix = _mix_rows(B, mode)
    s_ = s.clone().requires_grad_(True)
    loss, ce, kd = distillation_reference(s_, t, y, mix, eps, alpha, T)
    (loss.sum() / B).backward()
    L, CE, KD, D, _ = distillation_head_reference(s, t, y, mix, eps, alpha, T, 1.0 / B)
    zmax = float(torch.cat([s, t]).abs().max())
    c = 8 * U32 * (2 * zmax / min(T, 1.0) + math.log(K) + 2)
    p, q, r = torch.softmax(s.double(), 1), torch.softmax(s.double() / T, 1), torch.softmax(t.double() / T, 1)
    from b200ddl.models.augment import soft_targets

    tg = soft_targets(y, K, mix, eps, torch.float64)
    bound = (c * (alpha * (p + tg) + (1 - alpha) * T * (q + r)) + 4 * U32 * D.abs()) / B + 1e-30
    err = (s_.grad.double() - D).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    for name, got, want in (("loss", loss, L), ("student", ce, CE), ("distill", kd, KD)):
        lb = c * (want.abs() + 1) * (K + 4) * max(T * T, 1.0) + 1e-30
        assert bool(((got.double() - want).abs() <= lb).all()), name
    # float64 autograd equals the float64 closed form to float64 rounding
    z = s.double().requires_grad_(True)
    distillation_reference(z, t.double(), y, mix, eps, alpha, T)[0].sum().div(B).backward()
    assert torch.allclose(z.grad, D, rtol=1e-12, atol=1e-15)


def test_kl_matches_torch_kl_div_and_is_zero_for_equal_logits():
    s, t = _logits(5, 7, 8), _logits(5, 7, 9)
    y = torch.zeros(5, dtype=torch.long)
    _, _, kd = distillation_reference(s.double(), t.double(), y, None, 0.0, 0.5, 2.0)
    want = torch.nn.functional.kl_div(torch.log_softmax(s.double() / 2, 1), torch.log_softmax(t.double() / 2, 1),
                                      reduction="none", log_target=True).sum(1) * 4
    assert torch.allclose(kd, want, rtol=1e-13, atol=1e-15)
    _, _, kd0 = distillation_reference(s.double(), s.double(), y, None, 0.0, 0.5, 2.0)
    assert float(kd0.abs().max()) < 1e-14


@pytest.mark.parametrize("mode", [None, "mixup", "cutmix"])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_alpha_one_is_the_categorical_reference(mode, eps):
    B, K = 9, 6
    s, t = _logits(B, K, 5), _logits(B, K, 6)
    y = torch.randint(0, K, (B,), generator=torch.Generator().manual_seed(7))
    mix = _mix_rows(B, mode)
    loss, student, _, d, correct = distillation_head_reference(s, t, y, mix, eps, 1.0, 3.0, 0.25)
    want_loss, want_d, want_correct = soft_head_reference(s, y, mix, eps, 0.25)
    assert torch.equal(loss, want_loss) and torch.equal(student, want_loss)
    assert torch.equal(d, want_d) and correct == want_correct


# ------------------------------------------------------------------------------------------------ module backend
def _fit_trainer(teacher, alpha=0.5, T=2.0, lr=3e-2):
    return Trainer(_net(0), device="cpu").compile(optim.Adam(lr), loss=Distillation(teacher, alpha, T))


def test_fit_freezes_teacher_logs_terms_and_learns():
    teacher = _net(11)
    teacher.train()   # fit must run it in inference mode regardless
    before = {k: v.clone() for k, v in teacher.state_dict().items()}
    tr = _fit_trainer(teacher)
    data = _data(4)
    h = tr.fit(data, epochs=6, verbose=0)
    for k, v in teacher.state_dict().items():
        assert torch.equal(v, before[k]), k
    assert not any(p.grad is not None for p in teacher.parameters())
    logs = h.history
    for key in ("loss", "accuracy", "student_loss", "distillation_loss"):
        assert len(logs[key]) == 6 and all(math.isfinite(v) for v in logs[key]), key
    assert logs["loss"][-1] < logs["loss"][0]
    for lo, ce, kd in zip(logs["loss"], logs["student_loss"], logs["distillation_loss"]):
        assert lo == pytest.approx(0.5 * ce + 0.5 * kd, rel=1e-5)


def test_first_step_loss_is_the_reference():
    from b200ddl.models.preprocess import preprocess_tensor

    teacher, data = _net(11), _data(1)
    tr = _fit_trainer(teacher, alpha=0.3, T=4.0)
    x, y = data[0]
    with torch.no_grad():
        want = [float(v.mean()) for v in distillation_reference(
            tr.model(preprocess_tensor(x)).float(), teacher(preprocess_tensor(x)).float(), y, None, 0.0, 0.3, 4.0)]
    h = tr.fit(data, epochs=1, verbose=0).history
    got = [h["loss"][0], h["student_loss"][0], h["distillation_loss"][0]]
    assert got == pytest.approx(want, rel=1e-6)


def test_evaluate_and_checkpoints_see_the_student_alone(tmp_path):
    teacher, data = _net(11), _data(3)
    tr = Trainer(_net(0), device="cpu").compile(optim.Adam(1e-2), loss=Distillation(teacher, label_smoothing=0.1))
    tr.fit(data, epochs=1, verbose=0)
    plain = Trainer(tr.model, device="cpu").compile(optim.Adam(1e-2),
                                                    loss=CategoricalCrossentropy(from_logits=True, label_smoothing=0.1))
    assert tr.evaluate(data) == plain.evaluate(data)
    tr.save(str(tmp_path / "ck.pt"))
    tr.save_weights(str(tmp_path / "w.pt"))
    keys = set(tr.model.state_dict())
    assert set(torch.load(str(tmp_path / "ck.pt"))["weights"]) == keys
    assert set(torch.load(str(tmp_path / "w.pt"))) == keys
    assert tr.predict(data[0][0].numpy()).shape == (8, 5)


def test_teacher_broadcast_on_two_ranks():
    """Rank-dependent teacher seeds, the same data on both ranks: after BroadcastGlobalVariablesCallback both ranks
    hold rank 0's teacher, report identical losses and keep identical students."""
    def fn():
        import torch

        import b200ddl.parallel as hvd
        from b200ddl import optim
        from b200ddl.train import Distillation, Trainer
        from b200ddl.utils import checksum_across_ranks

        def net(seed):
            torch.manual_seed(seed)
            return torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * 8 * 8, 16), torch.nn.ReLU(),
                                       torch.nn.Linear(16, 5))

        g = torch.Generator().manual_seed(0)
        data = [(torch.randint(0, 256, (8, 8, 8, 3), generator=g).to(torch.uint8), torch.randint(0, 5, (8,), generator=g))
                for _ in range(3)]
        hvd.init()
        teacher = net(100 + hvd.rank())
        tr = Trainer(net(0), device="cpu").compile(optim.SGD(0.05), loss=Distillation(teacher, 0.2, 2.0))
        h = tr.fit(data, epochs=1, verbose=0, callbacks=[hvd.callbacks.BroadcastGlobalVariablesCallback(0)])
        flat = torch.cat([v.flatten() for v in teacher.state_dict().values()])
        losses = torch.tensor([h.history[k][0] for k in ("loss", "student_loss", "distillation_loss")],
                              dtype=torch.float64)
        return {"teacher_same": checksum_across_ranks(flat), "losses_same": checksum_across_ranks(losses),
                "student_same": checksum_across_ranks(tr.backend.flat.params),
                "teacher_is_rank0s": torch.equal(flat, torch.cat([v.flatten() for v in net(100).state_dict().values()]))}

    out = Runner(np=2, driver_log_verbosity="none", force_cpu=True).run(fn)
    assert out == {"teacher_same": True, "losses_same": True, "student_same": True, "teacher_is_rank0s": True}
