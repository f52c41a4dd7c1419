"""`batchnorm="training"` (MobileNetV2 `fine_tune_at` with batch-statistics BatchNorm) on the torch module, through
`build_model`, tracking and checkpoints, without a GPU."""
from __future__ import annotations

import pytest
import torch

from b200ddl.models import build_model
from b200ddl.models.mobilenet import FrozenBaseClassifier, MobileNetV2Base


def _module(k, batchnorm="training", dropout=0.0):
    return build_model(32, 32, 3, 5, dropout=dropout, arch="mobilenetv2_torch", fine_tune_at=k, batchnorm=batchnorm)


def _bns(mod):
    return [m for m in mod.modules() if isinstance(m, torch.nn.BatchNorm2d)]


def _data(n_batches=4, batch=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randint(0, 256, (batch, 32, 32, 3), dtype=torch.uint8, generator=g),
             torch.randint(0, 5, (batch,), generator=g)) for _ in range(n_batches)]


def test_validation():
    for bad in ("train", "eval", None, True, "Training"):
        with pytest.raises(ValueError):
            build_model(32, 32, 3, 5, arch="mobilenetv2_torch", fine_tune_at=3, batchnorm=bad)
    with pytest.raises(ValueError, match="freeze_base=False"):
        build_model(32, 32, 3, 5, arch="mobilenetv2_torch", batchnorm="training")
    with pytest.raises(ValueError, match="freeze_base=False"):
        FrozenBaseClassifier(MobileNetV2Base(), 1280, 5, 0.5, True, None, batchnorm="training")
    for arch in ("resnet50", "resnet50_torch"):
        with pytest.raises(ValueError):
            build_model(32, 32, 3, 5, arch=arch, batchnorm="training")
        with pytest.raises(ValueError):
            build_model(32, 32, 3, 5, arch=arch, fine_tune_at=3, batchnorm="training")
    with pytest.raises(ValueError):   # fine_tune_at and freeze_base=False still exclude each other
        build_model(32, 32, 3, 5, arch="mobilenetv2_torch", freeze_base=False, fine_tune_at=3, batchnorm="training")
    # the defaults are unchanged
    assert _module(5, "inference").batchnorm == "inference"
    assert build_model(32, 32, 3, 5, arch="mobilenetv2_torch").batchnorm == "inference"


def test_routing_without_gpu():
    """Without an H100 (or at a size the engine does not take) the option builds the torch module."""
    for size in (32, 30):
        m = build_model(size, size, 3, 5, arch="mobilenetv2", fine_tune_at=14, batchnorm="training")
        assert isinstance(m, FrozenBaseClassifier) and m.batchnorm == "training" and m.fine_tune_at == 14


@pytest.mark.parametrize("k", [0, 7, 18, 19])
def test_train_mode_switches_only_trainable_blocks(k):
    m = _module(k)
    m.train()
    for i, f in enumerate(m.base.features):
        assert all(bn.training == (i >= k) for bn in _bns(f)), i
    m.eval()
    assert not any(bn.training for bn in _bns(m))
    m.train()
    m.train(False)
    assert not any(bn.training for bn in _bns(m))


def test_fit_updates_running_statistics_of_trainable_blocks_only():
    from b200ddl import optim
    from b200ddl.train import Trainer

    k = 12
    m = _module(k)
    sd0 = {n: v.clone() for n, v in m.state_dict().items()}
    tr = Trainer(m, device="cpu")
    tr.compile(optim.SGD(0.01, momentum=0.9))
    data = _data(3)
    tr.fit(data, epochs=1, verbose=0)
    sd1 = m.state_dict()
    stats = [n for n in sd0 if "running" in n or "num_batches" in n]
    assert stats
    for n in stats:
        feat = int(n.split(".")[2])
        if feat >= k:
            assert not torch.equal(sd1[n], sd0[n]), n
            if n.endswith("num_batches_tracked"):
                assert int(sd1[n]) == 3, n
        else:
            assert torch.equal(sd1[n], sd0[n]), n
    # eval() normalises with the running statistics: a sample's logits do not depend on the rest of the batch
    m.eval()
    x = data[0][0].permute(0, 3, 1, 2).float() / 127.5 - 1.0
    with torch.no_grad():
        full, alone = m(x), m(x[:1])
    torch.testing.assert_close(full[:1], alone, rtol=1e-5, atol=1e-5)
    m.train()
    with torch.no_grad():
        assert not torch.allclose(m(x)[:2], m(x[:2]), rtol=1e-3, atol=1e-3)   # batch statistics


def test_tracking_round_trip(tmp_path):
    from b200ddl import optim
    from b200ddl.tracking.models import _describe, load_model, save_model
    from b200ddl.train import Trainer

    m = _module(15)
    tr = Trainer(m, device="cpu")
    tr.compile(optim.SGD(0.01))
    tr.fit(_data(2), epochs=1, verbose=0)
    d = _describe(m)
    assert d["batchnorm"] == "training" and d["fine_tune_at"] == 15
    assert _describe(_module(15, "inference"))["batchnorm"] == "inference"
    save_model(m, str(tmp_path / "m"))
    back = load_model(str(tmp_path / "m"), device="cpu").model
    assert isinstance(back, FrozenBaseClassifier) and back.batchnorm == "training" and back.fine_tune_at == 15
    a, b = m.state_dict(), back.state_dict()
    assert sorted(a) == sorted(b) and all(torch.equal(a[n], b[n]) for n in a)


def test_resume_repeats_the_loss_curve(tmp_path):
    """4 steps in one run equal 2 steps, save, a fresh trainer loading the checkpoint, 2 more steps: the running
    statistics (which the next steps' losses do not read, but evaluation does) and the weights travel together."""
    from b200ddl import optim
    from b200ddl.train import Trainer

    data = _data(4)

    def trainer():
        t = Trainer(_module(10), device="cpu")
        t.compile(optim.SGD(0.05, momentum=0.9))
        return t

    full = trainer()
    losses_full = full.fit(data, epochs=1, verbose=0).history["loss"]
    per_step_full = [full.evaluate([b], verbose=0)[0] for b in data]
    a = trainer()
    a.fit(data[:2], epochs=1, verbose=0)
    a.save(str(tmp_path / "ck.pt"))
    b = trainer()
    b.load(str(tmp_path / "ck.pt"))
    b.fit(data[2:], epochs=1, verbose=0)
    sa, sb = full.model.state_dict(), b.model.state_dict()
    for n in sa:
        if "num_batches" in n:
            assert int(sb[n]) == int(sa[n]), n
        else:
            torch.testing.assert_close(sb[n], sa[n], rtol=1e-5, atol=1e-6, msg=n)
    per_step_b = [b.evaluate([x], verbose=0)[0] for x in data]
    assert per_step_b == pytest.approx(per_step_full, rel=1e-5, abs=1e-6)
    assert len(losses_full) == 1
