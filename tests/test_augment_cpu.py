"""Random augmentation without a GPU: the reference implementation's semantics, the configuration's validation, routing
through `build_model`, tracking, and training with it on the module backend."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from b200ddl.models.augment import (Augmentation, augment_key, augment_reference, hash_u32, params_reference,
                                     warp_reference)

O = 65536


def _rows(N, a00, a01, b0, a10, a11, b1):
    return torch.tensor([[a00, a01, b0, a10, a11, b1, 0, 0]] * N, dtype=torch.int32)


def _img(N=3, H=6, W=9, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g)


def test_identity_flip_and_rot90_matrices():
    x = _img()
    N, H, W, _ = x.shape
    assert torch.equal(warp_reference(x, _rows(N, O, 0, 0, 0, O, 0)), x)
    assert torch.equal(warp_reference(x, _rows(N, -O, 0, (W - 1) * O, 0, O, 0)), torch.flip(x, [2]))
    assert torch.equal(warp_reference(x, _rows(N, O, 0, 0, 0, -O, (H - 1) * O)), torch.flip(x, [1]))
    sq = _img(H=7, W=7)
    # out[y, x] = in[x, S-1-y]
    assert torch.equal(warp_reference(sq, _rows(N, 0, -O, 6 * O, O, 0, 0)), torch.rot90(sq, 1, (1, 2)))


@pytest.mark.parametrize("dx,dy", [(2, 0), (-3, 1), (0, -4), (11, 0)])
@pytest.mark.parametrize("fill", ["reflect", "constant"])
def test_integer_translation_is_a_filled_shift(dx, dy, fill):
    """sx = x - dx: the content moves by (dx, dy); "reflect" equals numpy's symmetric padding, "constant" fills."""
    x = _img(N=2, H=6, W=9, seed=1)
    N, H, W, _ = x.shape
    out = warp_reference(x, _rows(N, O, 0, -dx * O, 0, O, -dy * O), fill, 77)
    p = 2 * max(H, W)
    if fill == "reflect":
        padded = np.pad(x.numpy(), ((0, 0), (p, p), (p, p), (0, 0)), mode="symmetric")
    else:
        padded = np.pad(x.numpy(), ((0, 0), (p, p), (p, p), (0, 0)), mode="constant", constant_values=77)
    want = padded[:, p - dy:p - dy + H, p - dx:p - dx + W]
    assert np.array_equal(out.numpy(), want)


def test_draws_cover_their_ranges():
    """Over 10^4 draws: each allowed axis flips with rate ~1/2, and the matrix entries stay inside the bounds the
    rotation, zoom and translation ranges imply."""
    aug = Augmentation("horizontal_and_vertical", rotation=0.1, zoom=0.25, translation=0.2)
    N, H, W = 10_000, 40, 60
    p = params_reference(aug, N, H, W, augment_key(3, 1), 17).long()
    hf, vf = (p[:, 6] & 1).float().mean(), ((p[:, 6] >> 1) & 1).float().mean()
    for rate in (hf, vf):
        assert abs(float(rate) - 0.5) < 4 * math.sqrt(0.25 / N)
    a00, a01, a10, a11 = (p[:, i].double() / O for i in (0, 1, 3, 4))
    det = (a00 * a11 - a01 * a10).abs().sqrt()           # = the zoom s (up to rounding)
    assert float(det.min()) >= 0.75 - 1e-3 and float(det.max()) <= 1.25 + 1e-3
    assert float(det.min()) < 0.77 and float(det.max()) > 1.23
    ang = torch.atan2(a10.abs(), a11.abs())             # |rotation angle| (flips only change signs)
    assert float(ang.max()) <= 2 * math.pi * 0.1 + 1e-3 and float(ang.max()) > 2 * math.pi * 0.1 * 0.98
    # translation: the centre pixel maps to centre - A t, |t| <= f * side
    cx, cy = (W - 1) / 2, (H - 1) / 2
    sx = (p[:, 0].double() * cx + p[:, 1].double() * cy + p[:, 2].double()) / O - cx
    assert float(sx.abs().max()) <= 1.25 * math.sqrt(2) * 0.2 * max(H, W) + 1
    only_flip = params_reference(Augmentation("horizontal"), N, H, W, augment_key(3, 1), 17)
    assert set(only_flip[:, 6].unique().tolist()) == {0, 1}
    assert set(params_reference(Augmentation("vertical"), N, H, W, 1, 2)[:, 6].unique().tolist()) == {0, 2}
    assert set(params_reference(Augmentation(), 100, H, W, 1, 2)[:, 6].unique().tolist()) == {0}


def test_draws_depend_on_seed_rank_step_and_image():
    aug = Augmentation("horizontal", rotation=0.2, zoom=0.2, translation=0.2)
    base = params_reference(aug, 64, 32, 32, augment_key(1, 0), 5)
    assert torch.equal(base, params_reference(aug, 64, 32, 32, augment_key(1, 0), 5))
    for key, step in ((augment_key(2, 0), 5), (augment_key(1, 1), 5), (augment_key(1, 0), 6)):
        assert not torch.equal(base, params_reference(aug, 64, 32, 32, key, step))
    assert len({tuple(r) for r in base.tolist()}) == 64
    assert torch.equal(base[:10], params_reference(aug, 10, 32, 32, augment_key(1, 0), 5))


def test_hash_matches_dropout_reference():
    """The shared hash (csrc/hash.cuh) on uint32 corner values, against an independent numpy uint32 evaluation."""
    def np_hash(a, b, c):
        a, b, c = (np.asarray(v, dtype=np.uint64) for v in (a, b, c))
        m = np.uint64(0xFFFFFFFF)
        h = ((a * np.uint64(0x9E3779B1)) & m) ^ ((((b + np.uint64(0x7F4A7C15)) & m) * np.uint64(0x85EBCA77)) & m) ^ \
            ((((c + np.uint64(0x165667B1)) & m) * np.uint64(0xC2B2AE3D)) & m)
        h ^= h >> np.uint64(15)
        h = (h * np.uint64(0x2C1B3C6D)) & m
        h ^= h >> np.uint64(12)
        h = (h * np.uint64(0x297A2D39)) & m
        h ^= h >> np.uint64(15)
        return h
    vals = [0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 123456789]
    for a in vals:
        for b in vals:
            c = torch.tensor(vals, dtype=torch.int64)
            assert hash_u32(a, b, c).tolist() == np_hash(a, b, np.array(vals)).tolist()


@pytest.mark.parametrize("kw", [dict(flip="diagonal"), dict(rotation=-0.1), dict(rotation=0.6), dict(zoom=1.0),
                                dict(zoom=-0.1), dict(translation=1.5), dict(fill_mode="nearest"), dict(fill_value=256),
                                dict(fill_value=-1), dict(fill_value=1.5), dict(rotation=float("nan")),
                                dict(zoom=True), dict(rotation="0.1")])
def test_validation_errors(kw):
    with pytest.raises(ValueError):
        Augmentation(**kw)


def test_round_trip_and_frozen():
    a = Augmentation("horizontal_and_vertical", 0.2, 0.1, 0.3, "constant", 9)
    assert Augmentation.from_dict(a.to_dict()) == a
    assert Augmentation.from_dict(None) is None
    with pytest.raises(Exception):
        a.zoom = 0.5
    with pytest.raises(ValueError):
        augment_reference(a, torch.zeros(2, 8, 8, 3), 0, 1)


def test_build_model_routing():
    from b200ddl.models import Augmentation as Exported, build_model
    from b200ddl.models.mobilenet import FrozenBaseClassifier

    a = Exported(flip="horizontal", rotation=0.2)
    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", augmentation=a, seed=4)
    assert isinstance(m, FrozenBaseClassifier) and m.augmentation == a and m.augmentation_seed == 4
    assert build_model(32, 32, 3, 5, arch="mobilenetv2_torch").augmentation is None
    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", fine_tune_at=15, augmentation=a.to_dict())
    assert m.augmentation == a and m.fine_tune_at == 15
    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="resnet50_torch", augmentation=a)
    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="mobilenetv2_torch", augmentation="flip")


def test_tracking_round_trip(tmp_path):
    from b200ddl.models import build_model
    from b200ddl.tracking.models import load_model, save_model

    a = Augmentation("vertical", 0.05, 0.1, 0.1, "constant", 3)
    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", fine_tune_at=17, augmentation=a, seed=6)
    save_model(m, str(tmp_path / "m"))
    tr = load_model(str(tmp_path / "m"))
    assert tr.model.augmentation == a and tr.model.fine_tune_at == 17 and tr.model.augmentation_seed == 6
    plain = build_model(32, 32, 3, 5, arch="mobilenetv2_torch")
    save_model(plain, str(tmp_path / "p"))
    assert load_model(str(tmp_path / "p")).model.augmentation is None


def _data(n_batches=6, B=8, S=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_batches):
        y = torch.randint(0, 5, (B,), generator=g)
        # class-dependent colour so the head can learn it through the augmentation
        x = (torch.randint(0, 60, (B, S, S, 3), generator=g) + (y * 45).view(B, 1, 1, 1)).to(torch.uint8)
        out.append((x, y))
    return out


def _trainer(aug, lr=1e-2):
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.train import Trainer

    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", dropout=0.0, fine_tune_at=16, augmentation=aug,
                    seed=1)
    tr = Trainer(m, device="cpu")
    tr.compile(optim.Adam(lr))
    return tr


def test_fit_with_augmentation_lowers_the_loss():
    aug = Augmentation("horizontal", 0.1, 0.1, 0.1)
    data = _data()
    tr = _trainer(aug)
    hist = tr.fit(data, epochs=6, verbose=0)
    losses = hist.history["loss"]
    assert losses[-1] < losses[0] - 0.05, losses
    with pytest.raises(ValueError):
        tr.fit([(data[0][0].float(), data[0][1])], epochs=1, verbose=0)


def test_training_batches_are_augmented_and_eval_is_not():
    """The module sees the reference-augmented batch at the optimizer's step in training, the raw batch in evaluate."""
    aug = Augmentation("horizontal", 0.2, 0.2, 0.2)
    tr = _trainer(aug)
    seen = []
    h = tr.model.register_forward_pre_hook(lambda mod, inp: seen.append(inp[0].detach().clone()))
    data = _data(2)
    tr.fit(data, epochs=1, verbose=0)
    tr.evaluate(data[:1], verbose=0)
    h.remove()
    from b200ddl.models.preprocess import preprocess_tensor

    for t, (x, _) in enumerate(data, start=1):
        want = preprocess_tensor(augment_reference(aug, x, augment_key(1, 0), t))
        assert torch.equal(seen[t - 1], want)
    assert torch.equal(seen[-1], preprocess_tensor(data[0][0]))


def test_resume_repeats_the_uninterrupted_run(tmp_path):
    aug = Augmentation("horizontal_and_vertical", 0.1, 0.2, 0.1)
    data = _data(4)
    full = _trainer(aug)
    h_full = full.fit(data, epochs=4, verbose=0).history["loss"]
    first = _trainer(aug)
    h1 = first.fit(data, epochs=2, verbose=0).history["loss"]
    first.save(str(tmp_path / "ck.pt"))
    second = _trainer(aug)
    second.load(str(tmp_path / "ck.pt"))
    h2 = second.fit(data, epochs=4, initial_epoch=2, verbose=0).history["loss"]
    assert h1 + h2 == pytest.approx(h_full, rel=0, abs=0)
