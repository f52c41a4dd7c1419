"""`fine_tune_at` on the torch module and through `build_model` / tracking, without a GPU."""
from __future__ import annotations

import pytest
import torch

from b200ddl.models import build_model
from b200ddl.models.mobilenet import FrozenBaseClassifier, MobileNetV2Base


def _module(k, dropout=0.0):
    return build_model(32, 32, 3, 5, dropout=dropout, arch="mobilenetv2_torch", fine_tune_at=k)


def _expected_trainable(k):
    base = MobileNetV2Base()
    return sum(p.numel() for p in base.features[k:].parameters()) + 1280 * 5 + 5


@pytest.mark.parametrize("k", range(20))
def test_trainable_count(k):
    m = _module(k)
    n = sum(p.numel() for p in m.parameters() if p.requires_grad)
    assert n == _expected_trainable(k)
    if k == 19:
        assert n == 6405
    names = {n for n, p in m.named_parameters() if p.requires_grad}
    for n in names - {"fc.weight", "fc.bias"}:
        assert int(n.split(".")[2]) >= k, n


def test_engine_trainable_count_formula_matches_module():
    """MobileNetV2Engine.trainable_parameters() without building (or needing) a GPU: the same per-layer formula."""
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    eng = MobileNetV2Engine.__new__(MobileNetV2Engine)
    eng.num_classes, eng.feat_channels = 5, 1280
    eng._layers = MobileNetV2Engine._describe(eng)
    for k in (0, 1, 4, 14, 18, 19):
        eng._k = k
        assert eng.trainable_parameters() == _expected_trainable(k), k


def test_batchnorm_stays_in_eval_mode():
    m = _module(4)
    m.train()
    bns = [mod for mod in m.base.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    assert bns and not any(bn.training for bn in bns)
    stats = {n: v.clone() for n, v in m.state_dict().items() if "running" in n or "num_batches" in n}
    x = torch.randn(2, 3, 32, 32)
    m(x).sum().backward()
    for n, v in m.state_dict().items():
        if n in stats:
            assert torch.equal(v, stats[n]), n


@pytest.mark.parametrize("k", [0, 5, 18, 19])
def test_gradients_only_in_trainable_blocks(k):
    m = _module(k)
    m.train()
    torch.nn.functional.cross_entropy(m(torch.randn(2, 3, 32, 32)), torch.tensor([0, 3])).backward()
    for n, p in m.named_parameters():
        if n.startswith("base."):
            trainable = int(n.split(".")[2]) >= k
            assert (p.grad is not None) == trainable, n
            if trainable and n.endswith("weight"):
                assert float(p.grad.abs().sum()) > 0, n
        else:
            assert p.grad is not None


def test_build_model_validation():
    for bad in (-1, 20, 2.0, "3", True):
        with pytest.raises(ValueError):
            build_model(32, 32, 3, 5, arch="mobilenetv2_torch", fine_tune_at=bad)
    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="mobilenetv2", freeze_base=False, fine_tune_at=3)
    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="resnet50", fine_tune_at=3)
    with pytest.raises(ValueError):
        FrozenBaseClassifier(MobileNetV2Base(), 1280, 5, 0.5, False, 3)


def test_fine_tune_at_none_leaves_constructions_unchanged():
    for freeze in (True, False):
        a = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", freeze_base=freeze)
        b = build_model(32, 32, 3, 5, arch="mobilenetv2_torch", freeze_base=freeze, fine_tune_at=None)
        assert a.fine_tune_at is None and a.freeze_base is freeze
        assert [(n, p.requires_grad) for n, p in a.named_parameters()] == \
            [(n, p.requires_grad) for n, p in b.named_parameters()]
        sa, sb = a.state_dict(), b.state_dict()
        assert all(torch.equal(sa[n], sb[n]) for n in sa)
        a.train()
        assert all(mod.training != freeze for mod in a.base.modules() if isinstance(mod, torch.nn.BatchNorm2d))
        n_train = sum(p.numel() for p in a.parameters() if p.requires_grad)
        assert (n_train == 6405) == freeze


def test_describe_and_load_model_round_trip(tmp_path):
    from b200ddl.tracking.models import _describe, load_model, save_model

    m = _module(12, dropout=0.25)
    with torch.no_grad():
        m.base.features[15].conv[0][0].weight.mul_(1.5)
    d = _describe(m)
    assert d["fine_tune_at"] == 12 and d["freeze_base"] is True
    assert _describe(_module(None))["fine_tune_at"] is None
    save_model(m, str(tmp_path / "m"))
    tr = load_model(str(tmp_path / "m"), device="cpu")
    assert isinstance(tr.model, FrozenBaseClassifier) and tr.model.fine_tune_at == 12
    a, b = m.state_dict(), tr.model.state_dict()
    assert sorted(a) == sorted(b) and all(torch.equal(a[n], b[n]) for n in a)
    assert [n for n, p in tr.model.named_parameters() if p.requires_grad] == \
        [n for n, p in m.named_parameters() if p.requires_grad]
