"""MixUp, CutMix and label smoothing without a GPU: the configuration, the Beta quantile table, the reference mix rows
and mixing warp, the soft-target reference, `Trainer.compile`'s loss check and training on the module backend."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from b200ddl.models.augment import (CUT_MIX, MIX_UP, Augmentation, augment_key, augment_reference, beta_quantiles,
                                     mix_params_reference, mix_warp_reference, params_reference, soft_head_reference,
                                     soft_targets, target_argmax, warp_reference)


def _img(N=5, H=9, W=13, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g)


# ------------------------------------------------------------------------------------------------ configuration
@pytest.mark.parametrize("kw", [dict(mixup=-0.1), dict(mixup=100.5), dict(cutmix=float("inf")), dict(cutmix=float("nan")),
                                dict(mixup=True), dict(cutmix="1"), dict(mixup=0.2, cutmix=1.0)])
def test_validation_errors(kw):
    with pytest.raises(ValueError):
        Augmentation(**kw)


def test_both_on_names_both():
    with pytest.raises(ValueError, match="mixup.*cutmix"):
        Augmentation(mixup=0.2, cutmix=0.5)


def test_dict_round_trip_and_old_dicts():
    a = Augmentation("horizontal", 0.1, cutmix=1.0)
    d = a.to_dict()
    assert d["cutmix"] == 1.0 and d["mixup"] == 0.0
    assert Augmentation.from_dict(d) == a
    old = {k: v for k, v in Augmentation("vertical", 0.2).to_dict().items() if k not in ("mixup", "cutmix")}
    b = Augmentation.from_dict(old)
    assert b.mixup == 0.0 and b.cutmix == 0.0 and b.mix_mode == 0
    assert Augmentation(mixup=0.2).mix_mode == MIX_UP and Augmentation(cutmix=2).mix_mode == CUT_MIX


def test_tracking_round_trip(tmp_path):
    from b200ddl.models import build_model
    from b200ddl.tracking.models import load_model, save_model

    a = Augmentation("horizontal", mixup=0.4)
    save_model(build_model(32, 32, 3, 5, arch="mobilenetv2_torch", augmentation=a, seed=2), str(tmp_path / "m"))
    assert load_model(str(tmp_path / "m")).model.augmentation == a


# ------------------------------------------------------------------------------------------------ lambda table
@pytest.mark.parametrize("alpha", [0.1, 0.2, 0.4, 1.0, 2.0, 8.0])
def test_lambda_table_matches_scipy(alpha):
    """Each Q16 entry is the nearest integer to 65536 x scipy's quantile (within 1e-6 of the rounding boundary), the
    table is exactly symmetric and monotone, and the sqrt column follows the lambda column."""
    from scipy.special import betaincinv

    n = 4096
    ref = betaincinv(alpha, alpha, (np.arange(n) + 0.5) / n)
    assert np.abs(beta_quantiles(alpha) - ref).max() < 1e-12
    tab = Augmentation(mixup=alpha).lambda_table().numpy().astype(np.int64)
    assert tab.shape == (n, 2)
    assert np.abs(tab[:, 0] - ref * 65536).max() <= 0.5 + 1e-6
    assert np.abs(tab[:, 1] - np.sqrt(1 - ref) * 65536).max() <= 0.5 + 1e-6
    assert np.array_equal(tab[:, 0] + tab[::-1, 0], np.full(n, 65536))
    assert (np.diff(tab[:, 0]) >= 0).all() and (np.diff(tab[:, 1]) <= 0).all()
    assert np.array_equal(Augmentation(cutmix=alpha).lambda_table().numpy(), tab)


def test_package_does_not_import_scipy():
    import subprocess
    import sys

    code = ("import sys; from b200ddl.models.augment import Augmentation; Augmentation(mixup=0.2).lambda_table(); "
            "print('scipy' in sys.modules)")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "False"


# ------------------------------------------------------------------------------------------------ mix rows
@pytest.mark.parametrize("N", [2, 3, 7, 256])
def test_partner_map_is_a_rotation(N):
    """At every step the partner map is a permutation without a fixed point, and it changes over the steps."""
    aug = Augmentation(mixup=0.2)
    maps = set()
    for t in range(1, 41):
        p = mix_params_reference(aug, N, 8, 8, augment_key(3, 1), t)[:, 0].long()
        assert sorted(p.tolist()) == list(range(N))
        assert bool((p != torch.arange(N)).all())
        s = int(p[0])
        assert torch.equal(p, (torch.arange(N) + s) % N)
        maps.add(s)
    if N > 2:
        assert len(maps) > 1
    assert mix_params_reference(aug, 1, 8, 8, 1, 5)[0, 0] == 0


def test_mixup_rows():
    aug = Augmentation(mixup=0.4)
    m = mix_params_reference(aug, 2000, 20, 30, augment_key(1, 0), 9).long()
    w = m[:, 1]
    assert bool(((w >= 0) & (w <= 256)).all())
    assert torch.equal(m[:, 6], 256 - w) and bool((m[:, 7] == 256).all())
    assert bool((m[:, 2:6] == 0).all())
    # Beta(0.4, 0.4) is U-shaped: weights pile up near both ends
    assert float(((w < 26) | (w > 230)).float().mean()) > 0.4


def test_cutmix_rows():
    aug = Augmentation(cutmix=1.0)
    H, W = 20, 30
    m = mix_params_reference(aug, 2000, H, W, augment_key(1, 0), 9).long()
    x0, y0, x1, y1 = m[:, 2], m[:, 3], m[:, 4], m[:, 5]
    assert bool(((0 <= x0) & (x0 <= x1) & (x1 <= W) & (0 <= y0) & (y0 <= y1) & (y1 <= H)).all())
    assert torch.equal(m[:, 6], (x1 - x0) * (y1 - y0)) and bool((m[:, 7] == H * W).all())
    assert bool((m[:, 1] == 0).all())
    # Beta(1, 1): the area fraction before clipping is uniform, so the mean clipped fraction is below 1/2 but not 0
    mu = (m[:, 6].double() / m[:, 7].double()).mean()
    assert 0.15 < float(mu) < 0.5


def test_geometric_params_are_the_same_with_mixing():
    base = dict(flip="horizontal_and_vertical", rotation=0.2, zoom=0.3, translation=0.1)
    for mix in (dict(), dict(mixup=0.2), dict(cutmix=1.0)):
        assert torch.equal(params_reference(Augmentation(**base, **mix), 50, 16, 24, 77, 3),
                           params_reference(Augmentation(**base), 50, 16, 24, 77, 3))


# ------------------------------------------------------------------------------------------------ mixing warp
@pytest.mark.parametrize("mode", [MIX_UP, CUT_MIX])
def test_mixing_a_batch_with_itself_is_the_geometric_warp(mode):
    aug = Augmentation("horizontal", 0.2, 0.2, 0.1, mixup=0.2 if mode == MIX_UP else 0.0,
                       cutmix=1.0 if mode == CUT_MIX else 0.0)
    x = _img()
    N, H, W, _ = x.shape
    p = params_reference(aug, N, H, W, 5, 2)
    m = mix_params_reference(aug, N, H, W, 5, 2)
    m[:, 0] = torch.arange(N)
    assert torch.equal(mix_warp_reference(x, p, m, mode), warp_reference(x, p))
    one = x[:1]
    assert torch.equal(augment_reference(aug, one, 5, 2), warp_reference(one, params_reference(aug, 1, H, W, 5, 2)))


def test_mixup_blend():
    x = _img()
    N, H, W, _ = x.shape
    aug = Augmentation(mixup=1.0)
    p = params_reference(aug, N, H, W, 1, 4)
    m = mix_params_reference(aug, N, H, W, 1, 4)
    own = warp_reference(x, p).long()
    w = m[:, 1].long().view(N, 1, 1, 1)
    want = (w * own + (256 - w) * own[m[:, 0].long()] + 128) >> 8
    assert torch.equal(mix_warp_reference(x, p, m, MIX_UP).long(), want)


def test_cutmix_box_comes_from_the_partner():
    """Inside the box every pixel is the partner's warped pixel, outside the image's own; mu = box area / (H W)."""
    x = _img(N=6, H=24, W=32, seed=3)
    N, H, W, _ = x.shape
    aug = Augmentation("horizontal", 0.1, cutmix=1.0)
    p = params_reference(aug, N, H, W, 11, 7)
    m = mix_params_reference(aug, N, H, W, 11, 7).long()
    own = warp_reference(x, p)
    out = mix_warp_reference(x, p, m, CUT_MIX)
    assert bool((m[:, 6] > 0).any())
    for n in range(N):
        q, x0, y0, x1, y1 = (int(v) for v in m[n, [0, 2, 3, 4, 5]])
        inside = torch.zeros(H, W, dtype=torch.bool)
        inside[y0:y1, x0:x1] = True
        assert torch.equal(out[n][inside], own[q][inside])
        assert torch.equal(out[n][~inside], own[n][~inside])
        assert int(inside.sum()) == int(m[n, 6]) and int(m[n, 7]) == H * W


# ------------------------------------------------------------------------------------------------ soft targets
def _logits(B=9, K=7, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, K, generator=g, dtype=torch.float64) * 3, torch.randint(0, K, (B,), generator=g)


@pytest.mark.parametrize("eps", [0.0, 0.1, 0.5, 1.0])
def test_soft_reference_without_mixing_is_label_smoothing(eps):
    z, y = _logits()
    loss, d, correct = soft_head_reference(z, y, None, eps, grad_scale=0.5)
    want = F.cross_entropy(z, y, label_smoothing=eps, reduction="none")
    assert torch.allclose(loss, want, rtol=1e-12, atol=1e-12)
    zz = z.clone().requires_grad_(True)
    F.cross_entropy(zz, y, label_smoothing=eps, reduction="sum").backward()
    assert torch.allclose(d, 0.5 * zz.grad, rtol=1e-12, atol=1e-12)
    assert correct == int((z.argmax(1) == y).sum())   # smoothing never enters the accuracy, as in Keras


@pytest.mark.parametrize("mode", [MIX_UP, CUT_MIX])
def test_soft_reference_without_smoothing_is_the_weighted_sum(mode):
    z, y = _logits(B=64, K=5, seed=1)
    aug = Augmentation(mixup=0.3) if mode == MIX_UP else Augmentation(cutmix=1.0)
    m = mix_params_reference(aug, 64, 16, 16, 3, 2)
    loss, _, _ = soft_head_reference(z, y, m, 0.0)
    mu = m[:, 6].double() / m[:, 7].double()
    p = m[:, 0].long()
    ce = lambda t: F.cross_entropy(z, t, reduction="none")  # noqa: E731
    assert torch.allclose(loss, (1 - mu) * ce(y) + mu * ce(y[p]), rtol=1e-12, atol=1e-12)


def test_target_argmax_rule():
    y = torch.tensor([3, 1, 4, 2])
    mix = torch.tensor([[1, 0, 0, 0, 0, 0, 100, 256], [2, 0, 0, 0, 0, 0, 200, 256],
                        [3, 0, 0, 0, 0, 0, 128, 256], [0, 0, 0, 0, 0, 0, 128, 256]], dtype=torch.int32)
    # row 0: mu < 1/2 -> own label 3; row 1: mu > 1/2 -> partner's 4; rows 2, 3: tie -> lower of (4, 2) and (2, 3)
    assert target_argmax(y, mix).tolist() == [3, 4, 2, 2]
    for eps in (0.0, 0.1, 0.9):
        t = soft_targets(y, 5, mix, eps, torch.float64)
        assert torch.equal(t.argmax(1), target_argmax(y, mix))


# ------------------------------------------------------------------------------------------------ compile
def test_compile_accepts_and_refuses_losses():
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.train import Trainer
    from b200ddl.train.losses import CategoricalCrossentropy, SparseCategoricalCrossentropy

    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch")
    for loss, eps in (("sparse_categorical_crossentropy", 0.0), (SparseCategoricalCrossentropy(from_logits=True), 0.0),
                      ("categorical_crossentropy", 0.0), (CategoricalCrossentropy(from_logits=True), 0.0),
                      (CategoricalCrossentropy(from_logits=True, label_smoothing=0.2), 0.2)):
        tr = Trainer(m, device="cpu").compile(optim.SGD(0.1), loss=loss)
        assert tr.backend.label_smoothing == eps
    for bad in ("mse", "binary_crossentropy"):
        with pytest.raises(ValueError):
            Trainer(m, device="cpu").compile(optim.SGD(0.1), loss=bad)
    for kw in (dict(), dict(from_logits=True, label_smoothing=1.5), dict(from_logits=True, label_smoothing=-0.1),
               dict(from_logits=True, label_smoothing=float("nan"))):
        with pytest.raises(ValueError):
            CategoricalCrossentropy(**kw)
    mixed = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", augmentation=Augmentation(mixup=0.2))
    with pytest.raises(ValueError, match="soft targets"):
        Trainer(mixed, device="cpu").compile(optim.SGD(0.1))
    Trainer(mixed, device="cpu").compile(optim.SGD(0.1), loss="categorical_crossentropy")


@pytest.mark.parametrize("mix", [dict(mixup=0.4), dict(cutmix=1.0)], ids=["mixup", "cutmix"])
def test_mixing_model_predicts_and_serves(tmp_path, mix):
    """A model whose augmentation mixes predicts on an uncompiled Trainer and after save_model / load_model, with the
    logits of the same weights without the augmentation."""
    from b200ddl.models import build_model
    from b200ddl.tracking.models import load_model, save_model
    from b200ddl.train import Trainer

    aug = Augmentation("horizontal", **mix)
    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", augmentation=aug, seed=3)
    x = _img(N=4, H=32, W=32, seed=5).numpy()
    p = Trainer(m, device="cpu").predict(x)
    save_model(m, str(tmp_path / "m"))
    tr = load_model(str(tmp_path / "m"))
    assert tr.model.augmentation == aug
    plain = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", seed=3)
    plain.load_state_dict(m.state_dict())
    want = Trainer(plain, device="cpu").predict(x)
    assert np.array_equal(p, want) and np.array_equal(tr.predict(x), want)
    assert tr.evaluate([(torch.from_numpy(x), torch.tensor([0, 1, 2, 3]))])


def test_eval_accuracy_ignores_smoothing():
    """evaluate at label_smoothing = 1 reports the accuracy against the labels, not against class 0."""
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.train import Trainer
    from b200ddl.train.losses import CategoricalCrossentropy

    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", seed=2)
    data = _data(2)
    acc = [Trainer(m, device="cpu").compile(optim.SGD(0.0), loss=loss).evaluate(data)[1]
           for loss in ("sparse_categorical_crossentropy", CategoricalCrossentropy(from_logits=True, label_smoothing=1.0))]
    assert acc[0] == acc[1]


def test_resnet50_torch_takes_label_smoothing_but_no_augmentation():
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.train import Trainer
    from b200ddl.train.losses import CategoricalCrossentropy

    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="resnet50_torch", augmentation=Augmentation(cutmix=1.0))
    m = build_model(32, 32, 3, 5, arch="resnet50_torch")
    tr = Trainer(m, device="cpu").compile(optim.SGD(0.0), loss=CategoricalCrossentropy(True, 0.3))
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, 256, (4, 32, 32, 3), dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (4,), generator=g)
    loss = tr.evaluate([(x, y)])[0]
    from b200ddl.models.preprocess import preprocess_tensor

    m.eval()
    with torch.no_grad():
        want = F.cross_entropy(m(preprocess_tensor(x)).float(), y, label_smoothing=0.3)
    assert loss == pytest.approx(float(want), rel=1e-6)


# ------------------------------------------------------------------------------------------------ module backend
def _data(n_batches=4, B=8, S=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_batches):
        y = torch.randint(0, 5, (B,), generator=g)
        x = (torch.randint(0, 60, (B, S, S, 3), generator=g) + (y * 45).view(B, 1, 1, 1)).to(torch.uint8)
        out.append((x, y))
    return out


AUG = Augmentation("horizontal", 0.1, 0.1, 0.1, cutmix=1.0)


def _trainer(eps=0.1):
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.train import Trainer
    from b200ddl.train.losses import CategoricalCrossentropy

    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", dropout=0.0, fine_tune_at=16, augmentation=AUG, seed=1)
    tr = Trainer(m, device="cpu")
    tr.compile(optim.Adam(1e-2), loss=CategoricalCrossentropy(from_logits=True, label_smoothing=eps))
    return tr


def test_first_loss_is_the_reference():
    """The first training loss of a CutMix + eps = 0.1 fit is the soft-target loss of the module on the reference
    mixed batch, before the update."""
    from b200ddl.models.preprocess import preprocess_tensor

    data = _data(1)
    tr = _trainer()
    x, y = data[0]
    key = augment_key(1, 0)
    xm = augment_reference(AUG, x, key, 1)
    m = mix_params_reference(AUG, x.shape[0], 32, 32, key, 1)
    assert not torch.equal(xm, augment_reference(Augmentation("horizontal", 0.1, 0.1, 0.1), x, key, 1))
    tr.model.train()
    with torch.no_grad():
        z = tr.model(preprocess_tensor(xm)).float()
    want = F.cross_entropy(z, soft_targets(y, 5, m, 0.1))
    ref_loss, _, _ = soft_head_reference(z, y, m, 0.1)
    assert float(want) == pytest.approx(float(ref_loss.mean()), rel=1e-6)
    tr.fit(data, epochs=1, verbose=0)
    assert tr.history.history["loss"][0] == pytest.approx(float(want), rel=1e-6)


def test_resume_repeats_the_uninterrupted_run(tmp_path):
    data = _data(3)
    h_full = _trainer().fit(data, epochs=4, verbose=0).history["loss"]
    first = _trainer()
    h1 = first.fit(data, epochs=2, verbose=0).history["loss"]
    first.save(str(tmp_path / "ck.pt"))
    second = _trainer()
    second.load(str(tmp_path / "ck.pt"))
    h2 = second.fit(data, epochs=4, initial_epoch=2, verbose=0).history["loss"]
    assert h1 + h2 == pytest.approx(h_full, rel=0, abs=0)
