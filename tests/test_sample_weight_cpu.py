"""Keras loss weighting without a GPU: `fit(class_weight=...)` and `(x, y, sample_weight)` batches.  Validation, the
module backend against a float64 reference of (1/B) sum_n w_n l_n (MixUp rows weighted at their target argmax, both
distillation terms weighted), `InMemoryDataset(weight_column=...)` and autolog's record of class_weight."""
from __future__ import annotations

import copy

import numpy as np
import pytest
import torch

from b200ddl import optim
from b200ddl.models.augment import (Augmentation, augment_batch_reference, augment_key, distillation_reference,
                                     soft_targets, target_argmax)
from b200ddl.models.preprocess import preprocess_tensor
from b200ddl.train import CategoricalCrossentropy, Distillation, Trainer
from b200ddl.train.trainer import class_weight_table

K = 5


def _net(seed, S=8, hidden=16):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * S * S, hidden), torch.nn.ReLU(),
                               torch.nn.Linear(hidden, K))


def _data(n_batches=3, B=8, S=8, seed=0, weights=False):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_batches):
        y = torch.randint(0, K, (B,), generator=g)
        x = (torch.randint(0, 60, (B, S, S, 3), generator=g) + (y * 45).view(B, 1, 1, 1)).to(torch.uint8)
        out.append((x, y, torch.rand(B, generator=g) * 3) if weights else (x, y))
    return out


def _trainer(seed=0, loss="sparse_categorical_crossentropy", net=None):
    return Trainer(net if net is not None else _net(seed), device="cpu").compile(optim.SGD(0.05), loss=loss)


# ------------------------------------------------------------------------------------------------ validation
def test_class_weight_table_defaults_missing_classes_to_one():
    t = class_weight_table({0: 2.0, 3: 0.0, np.int64(4): np.float32(0.5)}, K)
    assert t.dtype == torch.float32 and t.tolist() == [2.0, 1.0, 1.0, 0.0, 0.5]


@pytest.mark.parametrize("cw", [{5: 1.0}, {-1: 1.0}, {1.0: 2.0}, {True: 2.0}, {"1": 2.0}, {0: -0.5},
                                {0: float("nan")}, {0: float("inf")}, {0: "2"}, {0: True}, [1.0, 2.0]])
def test_bad_class_weight_is_refused_before_the_first_step(cw):
    tr = _trainer()
    before = copy.deepcopy(tr.model.state_dict())
    with pytest.raises(ValueError, match="class_weight"):
        tr.fit(_data(1), epochs=1, verbose=0, class_weight=cw)
    for k, v in tr.model.state_dict().items():
        assert torch.equal(v, before[k]), k


def test_class_weight_with_sample_weight_batches_is_refused():
    with pytest.raises(ValueError, match="class_weight and sample_weight"):
        _trainer().fit(_data(1, weights=True), epochs=1, verbose=0, class_weight={0: 2.0})


def test_sample_weight_keyword_is_refused():
    with pytest.raises(ValueError, match="sample_weight"):
        _trainer().fit(_data(1), epochs=1, verbose=0, sample_weight=torch.ones(8))


@pytest.mark.parametrize("bad", [lambda b: (b[0],), lambda b: (*b, torch.ones(8), torch.ones(8)),
                                 lambda b: (*b, torch.ones(7)), lambda b: (*b, torch.ones(8, dtype=torch.int64)),
                                 lambda b: (*b, torch.ones(8, 1))])
def test_malformed_batches_are_refused(bad):
    with pytest.raises(ValueError, match="batches|sample_weight"):
        _trainer().fit([bad(_data(1)[0])], epochs=1, verbose=0)


# ------------------------------------------------------------------------------------------------ module backend
def _grads(tr):
    """The module's gradients of the last step (views into the flat gradient buffer), in parameter order, float64."""
    return torch.cat([p.grad.reshape(-1) for p in tr.model.parameters()]).double()


def test_all_ones_weights_train_exactly_as_unweighted():
    """All-ones class and sample weights give the unweighted run's gradients and weights bit for bit (the row product
    by 1 is exact and the mean's backward gives every row 1/B either way); the logged loss is the same up to the
    order of the batch sum."""
    data = _data(3)
    runs = []
    for kind in ("plain", "class", "sample"):
        tr = _trainer(0)
        if kind == "sample":
            h = tr.fit([(x, y, torch.ones(len(y))) for x, y in data], epochs=2, verbose=0).history
        else:
            h = tr.fit(data, epochs=2, verbose=0,
                       class_weight={c: 1.0 for c in range(K)} if kind == "class" else None).history
        runs.append((h["loss"], tr.backend.flat.params.clone(), tr.backend.flat.grads.clone()))
    for loss, params, grads in runs[1:]:
        assert torch.equal(params, runs[0][1]) and torch.equal(grads, runs[0][2])
        assert loss == pytest.approx(runs[0][0], rel=1e-6)


def _reference(net, x, y, w, target=None):
    """float64 (1/B) sum_n w_n l_n of ``net`` on the batch and its gradient with respect to every parameter."""
    net64 = copy.deepcopy(net).double()
    logits = net64(preprocess_tensor(x).double())
    logp = torch.log_softmax(logits, 1)
    t = torch.nn.functional.one_hot(y, K).double() if target is None else target.double()
    loss = (-(t * logp).sum(1) * w.double()).mean()
    loss.backward()
    return loss.item(), torch.cat([p.grad.reshape(-1) for p in net64.parameters()])


@pytest.mark.parametrize("kind", ["class", "sample"])
def test_weighted_loss_and_gradients_match_float64(kind):
    x, y = _data(1)[0]
    cw = {0: 2.5, 1: 0.0, 3: 0.25}
    g = torch.Generator().manual_seed(3)
    w = class_weight_table(cw, K)[y] if kind == "class" else torch.rand(len(y), generator=g) * 4
    tr = _trainer(0)
    ref_loss, ref_grad = _reference(tr.model, x, y, w)
    if kind == "class":
        h = tr.fit([(x, y)], epochs=1, verbose=0, class_weight=cw).history
    else:
        h = tr.fit([(x, y, w)], epochs=1, verbose=0).history
    # the gradient was taken before the SGD step moved the parameters; fp32 forward/backward against float64
    assert h["loss"][0] == pytest.approx(ref_loss, rel=1e-5)
    assert torch.allclose(_grads(tr), ref_grad, rtol=1e-4, atol=1e-6)


def test_weight_zero_rows_contribute_nothing():
    x, y = _data(1)[0]
    keep = y != y[0]
    w = keep.float()
    tr_w, tr_sub = _trainer(0), _trainer(0)
    tr_w.fit([(x, y, w)], epochs=1, verbose=0)
    _, g_sub = _reference(tr_sub.model, x[keep], y[keep], torch.ones(int(keep.sum())))
    g_sub = g_sub * keep.sum().double() / len(y)   # (1/B) over the kept rows
    assert torch.allclose(_grads(tr_w), g_sub, rtol=1e-4, atol=1e-6)


def test_mixup_rows_take_the_weight_of_their_target_argmax():
    net = _net(0)
    net.augmentation = Augmentation(mixup=0.4)
    net.augmentation_seed = 7
    tr = _trainer(net=net, loss=CategoricalCrossentropy(from_logits=True, label_smoothing=0.1))
    x, y = _data(1)[0]
    cw = {0: 3.0, 2: 0.5, 4: 0.0}
    xm, mix = augment_batch_reference(net.augmentation, x, augment_key(7, 0), 1)   # step 1: the first fit step
    assert mix is not None
    w = class_weight_table(cw, K)[target_argmax(y, mix)]
    ref_loss, ref_grad = _reference(net, xm, y, w, target=soft_targets(y, K, mix, 0.1))
    h = tr.fit([(x, y)], epochs=1, verbose=0, class_weight=cw).history
    assert h["loss"][0] == pytest.approx(ref_loss, rel=1e-5)
    assert torch.allclose(_grads(tr), ref_grad, rtol=1e-4, atol=1e-6)


def test_distillation_weights_both_terms():
    teacher = _net(11)
    x, y = _data(1)[0]
    w = torch.tensor([0.0, 1.0, 2.0, 0.5, 4.0, 1.0, 0.25, 3.0])
    tr = Trainer(_net(0), device="cpu").compile(optim.SGD(0.05), loss=Distillation(teacher, 0.3, 4.0))
    with torch.no_grad():
        rows = distillation_reference(tr.model(preprocess_tensor(x)).float(), teacher(preprocess_tensor(x)).float(), y,
                                      None, 0.0, 0.3, 4.0)
    want = [float((r.double() * w.double()).mean()) for r in rows]
    h = tr.fit([(x, y, w)], epochs=1, verbose=0).history
    got = [h["loss"][0], h["student_loss"][0], h["distillation_loss"][0]]
    assert got == pytest.approx(want, rel=1e-5)
    assert got[0] == pytest.approx(0.3 * got[1] + 0.7 * got[2], rel=1e-5)


def test_evaluate_weights_loss_only_with_sample_weights_and_never_accuracy():
    tr = _trainer(0)
    x, y = _data(1)[0]
    w = torch.linspace(0.0, 2.0, len(y))
    with torch.no_grad():
        logits = tr.model(preprocess_tensor(x)).float()
        rows = torch.nn.functional.cross_entropy(logits, y, reduction="none")
        acc = float((logits.argmax(1) == y).float().mean())
    loss_w, acc_w = tr.evaluate([(x, y, w)])
    loss, acc_u = tr.evaluate([(x, y)])
    assert loss_w == pytest.approx(float((rows * w).mean()), rel=1e-6)
    assert loss == pytest.approx(float(rows.mean()), rel=1e-6)
    assert acc_w == acc_u == pytest.approx(acc)
    tr.fit([(x, y)], epochs=1, verbose=0, class_weight={0: 5.0},
           validation_data=[(x, y)])   # class_weight never reaches validation
    with torch.no_grad():
        plain = float(torch.nn.functional.cross_entropy(tr.model(preprocess_tensor(x)).float(), y))
    assert tr.history.history["val_loss"][0] == pytest.approx(plain, rel=1e-6)


# ------------------------------------------------------------------------------------------------ loader, tracking
def _jpeg_table(n=6):
    import io

    import pandas as pd
    from PIL import Image

    rows = []
    for i in range(n):
        buf = io.BytesIO()
        Image.fromarray(np.full((8, 8, 3), 20 * i, np.uint8)).save(buf, format="JPEG")
        rows.append({"content": buf.getvalue(), "label_idx": i % K, "w": 0.5 * i})
    return pd.DataFrame(rows)


def test_in_memory_dataset_weight_column():
    from b200ddl.loader import InMemoryDataset

    pdf = _jpeg_table()
    plain = list(InMemoryDataset(pdf, 4, image_size=(8, 8), drop_last=False))
    weighted = list(InMemoryDataset(pdf, 4, image_size=(8, 8), drop_last=False, weight_column="w"))
    assert all(len(b) == 2 for b in plain) and all(len(b) == 3 for b in weighted)
    for (x, y), (xw, yw, w) in zip(plain, weighted):
        assert torch.equal(x, xw) and torch.equal(y, yw) and w.dtype == torch.float32
    assert torch.cat([b[2] for b in weighted]).tolist() == [0.5 * i for i in range(6)]
    with pytest.raises(ValueError, match="weight_column"):
        InMemoryDataset(pdf, 4, image_size=(8, 8), weight_column="missing")


def test_autolog_records_class_weight(tmp_path):
    from b200ddl import tracking

    tracking.set_tracking_uri(str(tmp_path / "mlruns"))
    tracking.set_experiment("weights")
    tracking.autolog(log_models=False)
    try:
        tr = _trainer(0)
        with tracking.start_run() as run:
            tr.fit(_data(1), epochs=1, verbose=0, class_weight={1: 2.0})
        assert tracking.get_run(run.info.run_id).data.params["class_weight"] == str({1: 2.0})
        with tracking.start_run() as run:
            tr.fit(_data(1), epochs=1, verbose=0)
        assert "class_weight" not in tracking.get_run(run.info.run_id).data.params
    finally:
        tracking.autolog(disable=True)
