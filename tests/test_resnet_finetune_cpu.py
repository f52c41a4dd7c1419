"""`arch="resnet50_head"` (ResNet-50 transfer learning): validation, the torch module and tracking, without a GPU."""
from __future__ import annotations

import pytest
import torch
import torchvision

from b200ddl.models import build_model
from b200ddl.models.resnet import ResNet50Head


def _module(k, batchnorm="inference", dropout=0.0, num_classes=5):
    return build_model(32, 32, 3, num_classes, dropout=dropout, arch="resnet50_head", fine_tune_at=k,
                       batchnorm=batchnorm, device="cpu")


def _block_of(name):
    """Feature block of a torchvision parameter name, counted independently of the module under test."""
    if name.startswith("fc."):
        return 17
    if name.startswith("layer"):
        stage, idx = name.split(".")[:2]
        return 1 + [0, 3, 7, 13][int(stage[5:]) - 1] + int(idx)
    return 0


def test_validation():
    for bad in (-1, 18, 2.0, "3", True):
        with pytest.raises(ValueError):
            _module(bad)
    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="resnet50_head", freeze_base=False, device="cpu")
    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="resnet50_head", batchnorm="training", device="cpu")
    with pytest.raises(ValueError):
        _module(4, batchnorm="frozen")
    with pytest.raises(ValueError):
        build_model(32, 32, 3, 5, arch="resnet50", fine_tune_at=3)
    a = build_model(32, 32, 3, 5, arch="resnet50_head", device="cpu")
    b = _module(17, dropout=0.5)
    assert isinstance(a, ResNet50Head) and a.fine_tune_at == b.fine_tune_at == 17
    assert [(n, p.requires_grad) for n, p in a.named_parameters()] == [(n, p.requires_grad) for n, p in b.named_parameters()]
    sa, sb = a.state_dict(), b.state_dict()
    assert all(torch.equal(sa[n], sb[n]) for n in sa)


@pytest.mark.parametrize("k,count,tensors,bns", [(17, 10_245, 2, 0), (14, 14_974_981, 32, 10), (4, 23_292_933, 128, None),
                                                 (0, 23_518_277, 161, 53)])
def test_trainable_counts(k, count, tensors, bns):
    m = _module(k)
    ref = torchvision.models.resnet50(weights=None, num_classes=5)
    expect = [(n, p.numel()) for n, p in ref.named_parameters() if _block_of(n) >= k]
    got = [(n, p.numel()) for n, p in m.named_parameters() if p.requires_grad]
    assert got == expect
    assert sum(n for _, n in got) == count and len(got) == tensors
    if bns is not None:
        trainable_bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d) and mod.weight.requires_grad]
        assert len(trainable_bns) == bns
    assert list(m.state_dict()) == list(ref.state_dict())


@pytest.mark.parametrize("k", [0, 8, 17])
def test_batchnorm_modes_after_train(k):
    for mode in ("inference", "training"):
        m = _module(k, batchnorm=mode).train()
        for name, mod in m.named_modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                assert mod.training == (mode == "training" and _block_of(name) >= k), (mode, name)
        m.eval()
        assert not any(mod.training for mod in m.modules())


def test_logits_match_torchvision_in_inference_mode():
    torch.manual_seed(0)
    m = _module(8)
    ref = torchvision.models.resnet50(weights=None, num_classes=5)
    with torch.no_grad():   # non-trivial running statistics
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.5, 1.5)
    ref.load_state_dict(m.state_dict())
    ref.eval()
    x = torch.randn(2, 3, 64, 64)
    m.train()   # inference-mode BatchNorm and dropout 0: training logits equal eval logits
    assert torch.equal(m(x), ref(x))


def _data(n_batches=4, b=4, size=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, 256, (b, size, size, 3), dtype=torch.uint8, generator=g),
             torch.randint(0, 5, (b,), generator=g)) for _ in range(n_batches)]


@pytest.mark.parametrize("k,mode", [(14, "inference"), (14, "training"), (0, "inference"), (17, "inference")])
@pytest.mark.parametrize("opt_kind", ["adamw_ema", "sgd_accum"])
def test_fit_changes_trainable_only(k, mode, opt_kind):
    from b200ddl import optim
    from b200ddl.train import Trainer

    m = _module(k, batchnorm=mode, dropout=0.2)
    before = {n: v.clone() for n, v in m.state_dict().items()}
    trainable = {n for n, p in m.named_parameters() if p.requires_grad}
    if opt_kind == "adamw_ema":
        opt = optim.AdamW(1e-3, weight_decay=0.05, use_ema=True)
    else:
        opt = optim.SGD(0.05, momentum=0.9, gradient_accumulation_steps=2)
    tr = Trainer(m, device="cpu").compile(opt)
    tr.fit(_data(), steps_per_epoch=4, epochs=1, verbose=0)
    after = m.state_dict()
    for n, v in after.items():
        blk = _block_of(n)
        if n in trainable:
            assert not torch.equal(v, before[n]), n
        elif "running" in n or "num_batches" in n:
            if mode == "inference" or blk < k:
                assert torch.equal(v, before[n]), n
        else:
            assert torch.equal(v, before[n]), n
    if mode == "training" and k < 17:
        moved = [n for n in after if "running_mean" in n and not torch.equal(after[n], before[n])]
        assert moved and all(_block_of(n) >= k for n in moved)


def test_tracking_round_trip(tmp_path):
    from b200ddl.tracking.models import _describe, load_model, save_model

    m = _module(14, batchnorm="training", dropout=0.25)
    with torch.no_grad():
        m.layer4[1].conv2.weight.mul_(1.5)
        m.layer1[0].bn1.running_var.fill_(2.0)
    d = _describe(m)
    assert (d["arch"], d["fine_tune_at"], d["batchnorm"]) == ("resnet50_head", 14, "training")
    save_model(m, str(tmp_path / "m"))
    tr = load_model(str(tmp_path / "m"), device="cpu")
    got = tr.model
    assert isinstance(got, ResNet50Head) and (got.fine_tune_at, got.batchnorm, got.dropout.p) == (14, "training", 0.25)
    a, b = m.state_dict(), got.state_dict()
    assert list(a) == list(b) and all(torch.equal(a[n], b[n]) for n in a)
    assert [(n, p.requires_grad) for n, p in got.named_parameters()] == \
        [(n, p.requires_grad) for n, p in m.named_parameters()]


def test_engine_layout_prefix_without_gpu():
    """The engine's trainable tensors for every k are a prefix of its flat layout, with the module's counts."""
    from b200ddl.models.resnet_engine import ResNet50Engine, resnet50_blocks

    for k in (0, 1, 4, 8, 14, 16, 17):
        eng = ResNet50Engine.__new__(ResNet50Engine)
        eng.num_classes, eng.blocks, eng._k = 5, resnet50_blocks(224), k
        ResNet50Engine._layout_params(eng)
        expect = sum(p.numel() for p in _module(k).parameters() if p.requires_grad)
        assert eng.trainable_parameters() == expect, k
        assert eng.trainable_numel == sum(-(-s.numel // 64) * 64 for s in eng.trainable_specs)
        names = {s.name for s in eng.trainable_specs}
        assert names == {n for n, p in _module(k).named_parameters() if p.requires_grad}
