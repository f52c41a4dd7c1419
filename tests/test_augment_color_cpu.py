"""Color augmentation without a GPU: the configuration, the draws, the integer reference `color_reference` and its
stages, and the module backend's training step."""
from __future__ import annotations

import itertools

import pytest
import torch

from b200ddl.models import augment as A
from b200ddl.models.augment import (GRAY_Q16, GRAY_WEIGHTS, Q8_MAX, Augmentation, augment_batch_reference, augment_key,
                                     augment_reference, color_apply_reference, color_draws_reference, color_key,
                                     color_reference, mix_params_reference, params_reference)

COLOR = dict(brightness=0.2, contrast=0.4, saturation=0.6, hue=0.15, grayscale=0.3)
STAGES = ("brightness", "contrast", "saturation", "hue", "grayscale")


def _img(N=6, H=9, W=13, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g)


def _varied(seed=0):
    """Random images, plus images of near-gray pixels (dl of a few levels), saturated pixels, ties between channels and
    flat images: the places where the HSV stages and the clamps have their edge cases."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (12, 7, 11, 3), dtype=torch.int64, generator=g)
    base = torch.randint(0, 256, (4, 7, 11, 1), dtype=torch.int64, generator=g)
    x[:4] = (base + torch.randint(-3, 4, (4, 7, 11, 3), generator=g)).clamp(0, 255)
    x[4] = torch.randint(0, 2, (7, 11, 3), generator=g) * 255
    x[5, ..., 1] = x[5, ..., 0]                       # R == G
    x[6, ..., 2] = x[6, ..., 1] = x[6, ..., 0]        # gray
    x[7] = 200
    return x.to(torch.uint8)


# ------------------------------------------------------------------------------------------------ configuration
@pytest.mark.parametrize("kw", [dict(brightness=-0.1), dict(brightness=1.5), dict(contrast=float("nan")),
                                dict(saturation=float("inf")), dict(hue=0.6), dict(grayscale=1.01), dict(hue=True),
                                dict(contrast="0.2"), dict(saturation=None), dict(brightness=(0.1, 0.2)),
                                dict(contrast=[0.5, 1.5])])
def test_validation_errors(kw):
    with pytest.raises(ValueError):
        Augmentation(**kw)


def test_tuple_forms_are_named_in_the_error():
    with pytest.raises(ValueError, match="lower, upper"):
        Augmentation(hue=(-0.1, 0.1))


def test_fields_accept_their_ranges():
    a = Augmentation(brightness=1, contrast=1.0, saturation=0, hue=0.5, grayscale=1)
    assert (a.brightness, a.contrast, a.saturation, a.hue, a.grayscale) == (1.0, 1.0, 0.0, 0.5, 1.0)
    assert isinstance(a.brightness, float)
    assert a.color_quantised() == (Q8_MAX, 65536, 0, 3 * 65536, 65536)
    assert not Augmentation().color_on and Augmentation(grayscale=0.1).color_on


def test_dict_round_trip_and_old_dicts():
    a = Augmentation("horizontal", 0.1, cutmix=1.0, **COLOR)
    d = a.to_dict()
    assert all(d[k] == COLOR[k] for k in COLOR)
    assert Augmentation.from_dict(d) == a
    old = {k: v for k, v in Augmentation("vertical", 0.2, mixup=0.3).to_dict().items() if k not in STAGES}
    b = Augmentation.from_dict(old)
    assert not b.color_on and all(getattr(b, k) == 0.0 for k in STAGES)
    assert b == Augmentation("vertical", 0.2, mixup=0.3)


def test_tracking_round_trip(tmp_path):
    from b200ddl.models import build_model
    from b200ddl.tracking.models import load_model, save_model

    a = Augmentation("horizontal", **COLOR)
    save_model(build_model(32, 32, 3, 5, arch="mobilenetv2_torch", augmentation=a, seed=2), str(tmp_path / "m"))
    assert load_model(str(tmp_path / "m")).model.augmentation == a


def test_launch_plan():
    """The params + warp launches run unless color is the only thing on; the identity configuration keeps them."""
    assert Augmentation().warp_on
    assert Augmentation("horizontal").warp_on and Augmentation(cutmix=1.0).warp_on
    assert Augmentation("horizontal", **COLOR).warp_on and Augmentation(mixup=0.2, hue=0.1).warp_on
    assert not Augmentation(**COLOR).warp_on and not Augmentation(grayscale=0.5).warp_on


# ------------------------------------------------------------------------------------------------ draws
def test_color_leaves_the_geometric_and_mix_rows_unchanged():
    geo = dict(flip="horizontal_and_vertical", rotation=0.2, zoom=0.3, translation=0.1)
    key = augment_key(5, 2)
    for mix in (dict(), dict(mixup=0.2), dict(cutmix=1.0)):
        plain, colored = Augmentation(**geo, **mix), Augmentation(**geo, **mix, **COLOR)
        for t in (1, 7, 100_000):
            assert torch.equal(params_reference(colored, 40, 16, 24, key, t), params_reference(plain, 40, 16, 24, key, t))
            if mix:
                assert torch.equal(mix_params_reference(colored, 40, 16, 24, key, t),
                                   mix_params_reference(plain, 40, 16, 24, key, t))
                x = _img(N=4, H=16, W=24)
                assert torch.equal(augment_batch_reference(colored, x, key, t)[1], augment_batch_reference(plain, x, key, t)[1])
    assert color_key(key) != key


def test_draws_cover_their_ranges():
    a = Augmentation(**COLOR)
    bq, cq, sq, hq, pq = a.color_quantised()
    d = torch.cat([color_draws_reference(a, 4000, augment_key(1, 0), t) for t in (1, 2)])
    for col, lo, hi in ((0, -bq, bq), (1, 65536 - cq, 65536 + cq), (2, 65536 - sq, 65536 + sq), (3, -hq, hq)):
        v = d[:, col]
        assert int(v.min()) >= lo and int(v.max()) < hi
        assert int(v.min()) < lo + (hi - lo) // 50 and int(v.max()) > hi - (hi - lo) // 50
    assert set(d[:, 4].tolist()) == {0, 1}
    assert abs(float(d[:, 4].double().mean()) - COLOR["grayscale"]) < 0.03
    off = color_draws_reference(Augmentation(), 50, 3, 4)
    assert torch.equal(off, torch.tensor([0, 65536, 65536, 0, 0]).expand(50, 5))
    assert not torch.equal(color_draws_reference(a, 50, 3, 4), color_draws_reference(a, 50, 3, 5))
    assert not torch.equal(color_draws_reference(a, 50, 3, 4), color_draws_reference(a, 50, 4, 4))


# ------------------------------------------------------------------------------------------------ stages
def test_stages_at_zero_are_skipped(monkeypatch):
    """A field at 0 skips its stage: no color field returns the batch as it is, the chain with one field at 0 is the
    chain without that stage, and the HSV helpers are never called for a stage that is off."""
    x = _varied()
    assert torch.equal(color_reference(Augmentation(), x, 1, 1), x)
    for name in STAGES:
        others = {k: v for k, v in COLOR.items() if k != name}
        want = color_apply_reference(x, color_draws_reference(Augmentation(**others), x.shape[0], 7, 3),
                                     [k != name for k in STAGES])
        with monkeypatch.context() as m:
            if name == "saturation":
                m.setattr(A, "_saturate", lambda *a: pytest.fail("saturation ran at 0"))
            if name == "hue":
                m.setattr(A, "_rotate_hue", lambda *a: pytest.fail("hue ran at 0"))
            assert torch.equal(color_reference(Augmentation(**others), x, 7, 3), want)


def test_unit_factors_are_exact_identities():
    x = _varied(1)
    N = x.shape[0]
    ones = torch.tensor([0, 65536, 65536, 0, 0]).expand(N, 5)
    for stages in ((True, False, False, False, False), (False, True, False, False, False),
                   (False, False, True, False, False), (True, True, True, False, False)):
        assert torch.equal(color_apply_reference(x, ones, stages), x), stages


def test_saturation_keeps_the_max_and_the_order_and_hue_keeps_max_and_min():
    """Saturation keeps each pixel's max (HSV value) exactly and never reorders its channels; hue rotation keeps each
    pixel's max and min exactly (so value and saturation are unchanged)."""
    x = _varied(2)
    N = x.shape[0]
    for t in range(1, 6):
        d = color_draws_reference(Augmentation(saturation=1.0, hue=0.5), N, 11, t)
        xs = color_apply_reference(x, d, (False, False, True, False, False)).long()
        xh = color_apply_reference(x, d, (False, False, False, True, False)).long()
        xl = x.long()
        assert torch.equal(xs.amax(-1), xl.amax(-1))
        for i, j in itertools.permutations(range(3), 2):
            assert bool((xs[..., i] >= xs[..., j])[xl[..., i] >= xl[..., j]].all())
        assert torch.equal(xh.amax(-1), xl.amax(-1)) and torch.equal(xh.amin(-1), xl.amin(-1))
        gray = (xl.amax(-1) == xl.amin(-1)).unsqueeze(-1).expand_as(xl)
        assert torch.equal(xs[gray], xl[gray]) and torch.equal(xh[gray], xl[gray])
    # S = 2 saturates every pixel as far as it goes: min -> 0 where dl >= mx / 2
    d = torch.tensor([0, 65536, 131072, 0, 0]).expand(N, 5)
    xs = color_apply_reference(x, d, (False, False, True, False, False)).long()
    xl = x.long()
    sat = (2 * (xl.amax(-1) - xl.amin(-1)) >= xl.amax(-1)) & (xl.amax(-1) > 0)
    assert bool((xs.amin(-1)[sat] == 0).all())


def test_hue_turns():
    """A shift of 1/3 of a turn moves pure red to pure green, and a full +-1/2 turn is the complement hue."""
    x = torch.tensor([[[[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0]]]], dtype=torch.uint8)
    d = torch.tensor([[0, 65536, 65536, 2 * 65536, 0]])
    out = color_apply_reference(x, d, (False, False, False, True, False))
    assert out[0, 0].tolist() == [[0, 255, 0], [0, 0, 255], [255, 0, 0], [0, 255, 255]]
    d = torch.tensor([[0, 65536, 65536, -3 * 65536, 0]])
    out = color_apply_reference(x, d, (False, False, False, True, False))
    assert out[0, 0].tolist() == [[0, 255, 255], [255, 0, 255], [255, 255, 0], [0, 0, 255]]


def test_grayscale_output_has_equal_channels():
    assert GRAY_Q16 == tuple(round(w * 65536) for w in GRAY_WEIGHTS)
    x = _img(N=64, seed=4)
    out = color_reference(Augmentation(grayscale=1.0), x, 2, 9)
    assert torch.equal(out[..., 0], out[..., 1]) and torch.equal(out[..., 1], out[..., 2])
    half = color_reference(Augmentation(grayscale=0.5), x, 2, 9)
    flat = (half[..., 0] == half[..., 1]).all((1, 2)) & (half[..., 1] == half[..., 2]).all((1, 2))
    drawn = color_draws_reference(Augmentation(grayscale=0.5), 64, 2, 9)[:, 4].bool()
    assert torch.equal(flat, drawn) and 0 < int(drawn.sum()) < 64
    assert torch.equal(half[drawn], out[drawn]) and torch.equal(half[~drawn], x[~drawn])


# ------------------------------------------------------------------------------------------------ float64 agreement
def _float_stage(name, x, d):
    """float64 implementation of one stage's formula on the uint8 batch x, with the draws d: the exact values the
    integer stage approximates, in levels (0 .. 255)."""
    N = x.shape[0]
    p = x.double()
    col = lambda k: d[:, k].double().view(N, 1, 1, 1)   # noqa: E731
    if name == "brightness":
        return (p + col(0) / 256).clamp(0, 255)
    if name == "contrast":
        m = p.mean((1, 2), keepdim=True)
        return (m + (p - m) * col(1) / 65536).clamp(0, 255)
    if name == "grayscale":
        y = sum(w * p[..., c] for c, w in enumerate(GRAY_WEIGHTS)).unsqueeze(-1).expand_as(p)
        return torch.where(col(4) != 0, y, p)
    r, g, b = p.unbind(-1)
    mx, mn = p.amax(-1), p.amin(-1)
    dl = mx - mn
    dls = torch.where(dl > 0, dl, torch.ones_like(dl))
    if name == "saturation":
        S = d[:, 2].double().view(N, 1, 1) / 65536
        k = torch.minimum(S, mx / dls)
        return torch.stack([mx - (mx - v) * k for v in (r, g, b)], -1)
    P = torch.where(r == mx, (g - b) / dls, torch.where(g == mx, 2 + (b - r) / dls, 4 + (r - g) / dls))
    P = torch.remainder(P + d[:, 3].double().view(N, 1, 1) / 65536, 6)
    s, f = torch.floor(P), P - torch.floor(P)
    rise, fall = mn + f * dl, mx - f * dl
    opts = [(mx, rise, mn), (fall, mx, mn), (mn, mx, rise), (mn, fall, mx), (rise, mn, mx), (mx, mn, fall)]
    out = torch.zeros_like(p)
    for i, o in enumerate(opts):
        out = torch.where((s == i).unsqueeze(-1), torch.stack(o, -1), out)
    return torch.where((dl > 0).unsqueeze(-1), out, p)


def _q8_bound(name, x, d):
    """Largest error of the integer stage's Q8 value (before the final rounding), per element, in Q8 units:
    - brightness: 256 p + delta is exact: 0.
    - contrast: the mean is rounded to Q8 (<= 1/2) and enters with weight 1 - f; the product rounds once (<= 1/2):
      1/2 |1 - f| + 1/2.  Clamping is 1-Lipschitz.
    - saturation: k = min(S, floor(mx 2^16 / dl)) is at most one Q16 unit below the exact min(S, mx / dl), which
      (mx - v) scales by (mx - v) / 2^16; the product rounds once: (mx - v) / 2^16 + 1/2.
    - hue: the fraction (a 2^16 + floor(dl / 2)) // dl is within 1/2 + 1 / (2 dl) <= 1 Q16 unit of a 2^16 / dl, and
      the rebuilt channel moves by dl per sixth (continuously across sectors and the wrap): dl / 2^16; one rounding of
      the part: + 1/2.
    - grayscale: each Q16 weight is within 1/2 unit of Keras's weight: sum_c |w_q,c / 2^16 - w_c| v_c; one rounding: + 1/2.
    Every bound is below 2 Q8 units, so with the final rounding (v + 128) >> 8 (<= 1/2 level) the uint8 result is
    within 1/2 + 2/256 < 1 level of the float64 value."""
    N = x.shape[0]
    v = x.double() * 256
    if name == "brightness":
        return torch.zeros_like(v)
    if name == "contrast":
        return (0.5 * (1 - d[:, 1].double() / 65536).abs() + 0.5).view(N, 1, 1, 1).expand_as(v)
    mx = v.amax(-1, keepdim=True)
    dl = mx - v.amin(-1, keepdim=True)
    if name == "saturation":
        return (mx - v) / 65536 + 0.5
    if name == "hue":
        return (dl / 65536 + 0.5).expand_as(v)
    err = sum(abs(q / 65536 - w) * v[..., c] for c, (q, w) in enumerate(zip(GRAY_Q16, GRAY_WEIGHTS)))
    return (err + 0.5).unsqueeze(-1).expand_as(v)


@pytest.mark.parametrize("name", STAGES)
def test_each_stage_agrees_with_float64(name):
    """Each stage alone, on random and edge-case images over several draws (hue over its whole range, contrast and
    saturation up to factor 2), against the float64 formula: within 1/2 level + the stage's Q8 bound (`_q8_bound`), which
    is below 1 level."""
    x = _varied(3)
    N = x.shape[0]
    aug = Augmentation(brightness=1.0, contrast=1.0, saturation=1.0, hue=0.5, grayscale=0.5)
    stages = [k == name for k in STAGES]
    worst = 0.0
    for t in range(1, 9):
        d = color_draws_reference(aug, N, augment_key(t, 0), t)
        got = color_apply_reference(x, d, stages).double()
        want = _float_stage(name, x, d)
        bound = 0.5 + _q8_bound(name, x, d) / 256
        assert float(bound.max()) < 1.0
        err = (got - want).abs()
        bad = (err > bound + 1e-9).nonzero()
        assert bad.numel() == 0, f"{name} step {t}: {bad.shape[0]} values off, first {bad[0].tolist()}: got " \
                                 f"{got[tuple(bad[0])]}, want {want[tuple(bad[0])]}, bound {bound[tuple(bad[0])]}"
        worst = max(worst, float(err.max()))
    assert worst < 1.0


def test_chain_order_and_clamps():
    """The whole chain clips after brightness and after contrast, and the output stays uint8 at the extremes."""
    x = _varied(5)
    aug = Augmentation(brightness=1.0, contrast=1.0, saturation=1.0, hue=0.5, grayscale=0.5)
    for t in range(1, 5):
        out = color_reference(aug, x, 9, t)
        assert out.dtype == torch.uint8 and out.shape == x.shape
    white = torch.full((1, 4, 4, 3), 255, dtype=torch.uint8)
    d = torch.tensor([[Q8_MAX, 65536, 65536, 0, 0]])
    assert torch.equal(color_apply_reference(white, d, (True, False, False, False, False)), white)
    d = torch.tensor([[-Q8_MAX, 65536, 65536, 0, 0]])
    assert int(color_apply_reference(white, d, (True, False, False, False, False)).max()) == 0


def test_mixed_images_take_their_own_color_draws():
    """Color comes after mixing: the batch is the mixed warp colored with image n's draws."""
    from b200ddl.models.augment import mix_warp_reference

    aug = Augmentation("horizontal", 0.1, cutmix=1.0, **COLOR)
    x = _img(N=5, H=16, W=20, seed=6)
    key = augment_key(4, 0)
    out, mix = augment_batch_reference(aug, x, key, 3)
    p = params_reference(aug, 5, 16, 20, key, 3)
    assert torch.equal(out, color_reference(aug, mix_warp_reference(x, p, mix, aug.mix_mode), key, 3))


# ------------------------------------------------------------------------------------------------ module backend
def _data(n_batches=2, B=8, S=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_batches):
        y = torch.randint(0, 5, (B,), generator=g)
        x = (torch.randint(0, 60, (B, S, S, 3), generator=g) + (y * 45).view(B, 1, 1, 1)).to(torch.uint8)
        out.append((x, y))
    return out


@pytest.mark.parametrize("aug", [Augmentation("horizontal", 0.1, **COLOR), Augmentation(**COLOR)], ids=["geo+color", "color"])
def test_module_training_step_feeds_the_reference_batch(aug):
    """mobilenetv2_torch on the module backend: every training step's module input is the reference batch of its
    optimizer step (color included), and evaluate sees the raw batch."""
    from b200ddl import optim
    from b200ddl.models import build_model
    from b200ddl.models.preprocess import preprocess_tensor
    from b200ddl.train import Trainer

    m = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", dropout=0.0, fine_tune_at=16, augmentation=aug, seed=1)
    tr = Trainer(m, device="cpu")
    tr.compile(optim.Adam(1e-2))
    seen = []
    h = tr.model.register_forward_pre_hook(lambda mod, inp: seen.append(inp[0].detach().clone()))
    data = _data()
    tr.fit(data, epochs=1, verbose=0)
    tr.evaluate(data[:1], verbose=0)
    h.remove()
    for t, (x, _) in enumerate(data, start=1):
        xa = augment_reference(aug, x, augment_key(1, 0), t)
        assert not torch.equal(xa, augment_reference(Augmentation("horizontal", 0.1) if aug.warp_on else
                                                     Augmentation(), x, augment_key(1, 0), t))
        assert torch.equal(seen[t - 1], preprocess_tensor(xa))
    assert torch.equal(seen[-1], preprocess_tensor(data[0][0]))
