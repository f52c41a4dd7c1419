"""Knowledge distillation on the GPU: softmax_kd_head (csrc/head_stem.cu) against the float64 reference
`distillation_head_reference`, and every native student engine with every native teacher engine.

The head is held to the float64 reference within bounds derived like test_mix.soft_bounds, and to softmax_ce_soft_head
/ softmax_ce_head bit for bit at alpha = 1.  The teacher's logits inside the student's training step are compared bit for
bit with the teacher's own evaluation step on the batch the student's stem read.
"""
from __future__ import annotations

import itertools

import pytest
import torch

from exact_util import DEV, U, Guarded, check_equal
from test_augment import AUG, _pix
from test_elementwise_exact import BF, NAN, RCP_ULP, bf, check_bound, f32, head_data
from test_mix import soft_bounds

pytestmark = pytest.mark.gpu


def _ops():
    from b200ddl import ops

    return ops.ext("_b200_ops")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _aug(**k):
    from b200ddl.models.augment import Augmentation

    return Augmentation(**k)


# ================================================================================================ softmax_kd_head
def _softmax_T_errors(z, T):
    """Per-entry error bounds of the kernel's fast-math log-softmax and softmax of z / T (fp32 logits z, float64): the
    argument (z - max) / T rounds twice after the correctly rounded 1 / T (3 u |x|); exp as in soft_bounds; the sum of
    K exps over ceil(K / 32) + 5 additions; __logf of the sum; the reciprocal."""
    K = z.shape[1]
    x = (z - z.max(1, keepdim=True).values) / T
    ex = torch.exp(x)
    se = ex.sum(1, keepdim=True)
    e_arg = 3 * U * x.abs()
    e_exp = (2 + torch.floor(1.173 * (x.abs() + e_arg))) * 2.0 ** -23 + U * x.abs() + e_arg
    depth = -(-K // 32) + 5
    rel_se = ((ex * e_exp).sum(1, keepdim=True) + depth * U * se) / se
    lg = torch.log(se)
    e_log = 2.0 ** -21.41 + 3 * 2.0 ** -23 * lg.abs()
    logp = x - lg
    e_logp = e_arg + (rel_se + e_log) * 1.001 + U * (x.abs() + logp.abs())
    p = ex / se
    e_p = p * (e_exp + rel_se + RCP_ULP + U) * 1.001
    return logp, e_logp, p, e_p


def kd_bounds(logit, tlogit, labels, mix, eps, alpha, T, grad_scale):
    """Float64 per-row (loss, student term, distillation term) and dlogits of softmax_kd_head on fp32 logits, with bounds.

    The student term and its dlogits are soft_bounds'.  KL = sum_k r_k (log r_k - log q_k): each log-softmax entry
    within _softmax_T_errors, r_k within its bound, the difference and the product round once each, the K-term sum has
    depth ceil(K / 32) + 5; T^2 KL rounds twice more.  dlogits: T (q - r) grad_scale from the two softmax bounds, the
    subtraction and two products.  alpha x + (1 - alpha) y: one rounding per product and one for the sum (the kernel
    uses uncontracted __fmul_rn / __fadd_rn).  Fast math flushes every result below 2^-126 to zero: p, q and r (q and r
    then scaled by T grad_scale <= T), the student dlogit, the distillation dlogit, the two weighted terms and their
    sum, so the dlogit bound has a floor of (6 + 2 T) 2^-126."""
    B, K = logit.shape
    ce, ceb, ds, dsb = soft_bounds(logit, labels, mix, eps, grad_scale)
    lq, e_lq, q, e_q = _softmax_T_errors(logit, T)
    lr, e_lr, r, e_r = _softmax_T_errors(tlogit, T)
    diff = lr - lq
    terms = r * diff
    depth = -(-K // 32) + 5
    kl = terms.sum(1)
    klb = (e_r * diff.abs() + r * (e_lq + e_lr) + 2 * U * terms.abs()).sum(1) * 1.001 + depth * U * terms.abs().sum(1)
    kd = T * T * kl
    kdb = T * T * (klb + 2 * U * kl.abs())
    beta = 1.0 - alpha
    loss = alpha * ce + beta * kd
    lb = alpha * ceb + beta * kdb + 2 * U * (alpha * ce.abs() + beta * kd.abs()) + U * loss.abs()
    dk = T * (q - r) * grad_scale
    dkb = T * (e_q + e_r + 3 * U * (q - r).abs()) * grad_scale
    d = alpha * ds + beta * dk
    db = (alpha * dsb + beta * dkb + 2 * U * (alpha * ds.abs() + beta * dk.abs()) + U * d.abs()
          + (6 + 2 * T) * 2.0 ** -126)
    return loss, lb, ce, ceb, kd, kdb, d, db


def _mix(mode, B):
    from b200ddl.models.augment import augment_key, mix_params_reference

    if mode is None:
        return None
    return mix_params_reference(_aug(**{mode: 0.4 if mode == "mixup" else 1.0}), B, 32, 32, augment_key(3, 0), 7,
                                device=DEV)


@pytest.mark.parametrize("B", [1, 7, 256, 513])
@pytest.mark.parametrize("K,ld,tld", [(5, 8, 64), (10, 64, 16), (1000, 1024, 1152)])
def test_kd_head(K, ld, tld, B):
    """softmax_kd_head for T in {1, 3, 10}, alpha in {0, 0.1, 1}, eps in {0, 0.1}, without mix rows and with MixUp and
    CutMix rows: logits32 exact, the accuracy count exact, padded dlogits exactly 0, the guards intact; loss rows, the
    four stats and dlogits within kd_bounds.  At alpha = 1 every output is softmax_ce_soft_head's bit for bit, and
    softmax_ce_head's at eps = 0 without mix rows."""
    from b200ddl.models.augment import distillation_head_reference, target_argmax

    e = _ops()
    g = gen(K * B + 1)
    l16, bias, labels = head_data(B, K, g)
    t16, tbias, _ = head_data(B, K, g)
    lg16 = torch.full((B, ld), NAN, device=DEV, dtype=BF)
    lg16[:, :K] = bf(l16)
    tg16 = torch.full((B, tld), NAN, device=DEV, dtype=BF)
    tg16[:, :K] = bf(t16)
    logit, tlogit = (l16 + bias).float().double(), (t16 + tbias).float().double()
    gs = 1.0 / 256
    for T, alpha, eps, mode in itertools.product((1.0, 3.0, 10.0), (0.0, 0.1, 1.0), (0.0, 0.1), (None, "mixup", "cutmix")):
        mix = _mix(mode, B)
        logits32, dl16 = Guarded((B, K), torch.float32), Guarded((B, ld), BF)
        loss_rows, stats = Guarded((B,), torch.float32, guard=64), Guarded((4,), torch.float32, 0.0, guard=64)
        e.softmax_kd_head(lg16, f32(bias), tg16, f32(tbias), labels, mix, eps, alpha, T, logits32.t, dl16.t,
                          loss_rows.t, stats.t, gs)
        torch.cuda.synchronize()
        name = f"softmax_kd_head K={K} ld={ld} tld={tld} B={B} T={T} alpha={alpha} eps={eps} mix={mode}"
        for gd, nm in ((logits32, "logits32"), (dl16, "dlogits16"), (loss_rows, "loss_rows"), (stats, "stats")):
            gd.check_guards(f"{name} {nm}")
        check_equal(name + " logits32", logits32.t, logit, lambda b, k: f"[warp {b} lane {k % 32}]")
        want = int((torch.from_numpy(logit.cpu().numpy().argmax(1)).to(DEV) == target_argmax(labels, mix)).sum())
        assert int(stats.t[1].item()) == want, f"{name}: accuracy count"
        check_equal(name + " padded dlogits", dl16.t[:, K:], torch.zeros(B, ld - K, device=DEV))
        loss, lb, ce, ceb, kd, kdb, d, db = kd_bounds(logit, tlogit, labels, mix, eps, alpha, T, gs)
        ref = distillation_head_reference(logit.float(), tlogit.float(), labels, mix, eps, alpha, T, gs)
        assert float((ref[0] - loss).abs().max()) <= 1e-9 * (1 + float(loss.abs().max())), name + " reference"
        check_bound(name + " loss", loss_rows.t, loss, lb)
        for i, (v, b_) in enumerate(((loss, lb), (ce, ceb), (kd, kdb))):
            check_bound(f"{name} stats[{(0, 2, 3)[i]}]", stats.t[(0, 2, 3)[i]:(0, 2, 3)[i] + 1], v.sum().view(1),
                        (b_.sum() + B * U * v.abs().sum()).view(1))
        check_bound(name + " dlogits", dl16.t[:, :K], d, db + 2.0 ** -8 * (d.abs() + db))
        if alpha != 1.0:
            continue
        kd_out = [torch.zeros(B, K, device=DEV), torch.zeros(B, ld, device=DEV, dtype=BF), torch.zeros(B, device=DEV),
                  torch.zeros(4, device=DEV)]
        soft = [torch.zeros_like(t) for t in kd_out[:3]] + [torch.zeros(2, device=DEV)]
        e.softmax_kd_head(lg16, f32(bias), tg16, f32(tbias), labels, mix, eps, 1.0, T, *kd_out, gs)
        e.softmax_ce_soft_head(lg16, f32(bias), labels, mix, eps, *soft, gs)
        others = [("softmax_ce_soft_head", soft)]
        if eps == 0.0 and mix is None:
            plain = [torch.zeros_like(t) for t in soft]
            e.softmax_ce_head(lg16, f32(bias), labels, *plain, gs)
            others.append(("softmax_ce_head", plain))
        torch.cuda.synchronize()
        for other, outs in others:
            for nm, a, b in zip(("logits32", "dlogits16", "loss rows"), kd_out, outs):
                check_equal(f"{name}: {nm} vs {other}", a, b)
            assert float(kd_out[3][1]) == float(outs[3][1]), f"{name}: accuracy vs {other}"
            check_bound(f"{name}: loss sum vs {other}", kd_out[3][:1], outs[3][:1].double(),
                        B * U * outs[2].double().abs().sum().view(1))


def test_kd_head_argument_checks():
    e = _ops()
    N = 4
    lg16, tg16 = torch.zeros(N, 8, device=DEV, dtype=BF), torch.zeros(N, 16, device=DEV, dtype=BF)
    bias, labels = torch.zeros(5, device=DEV), torch.zeros(N, device=DEV, dtype=torch.int64)
    mix = torch.zeros(N, 8, device=DEV, dtype=torch.int32)
    mix[:, 7] = 1
    stats = torch.zeros(4, device=DEV)
    ok = dict(logits16=lg16, bias=bias, tlogits16=tg16, tbias=bias.clone(), labels=labels, mix=mix,
              label_smoothing=0.1, alpha=0.5, temperature=2.0, stats=stats)
    bad = [dict(label_smoothing=1.5), dict(alpha=-0.1), dict(alpha=1.5), dict(alpha=float("nan")),
           dict(temperature=0.0), dict(temperature=-1.0), dict(temperature=float("inf")),
           dict(temperature=float("nan")), dict(tlogits16=tg16[:2].contiguous()), dict(tlogits16=tg16[:, :4].contiguous()),
           dict(tlogits16=tg16.float()), dict(tlogits16=tg16.cpu()), dict(tbias=torch.zeros(6, device=DEV)),
           dict(stats=stats[:2]), dict(mix=mix[:2].contiguous()), dict(labels=labels[:2]), dict(dlogits16=lg16),
           dict(tlogits16=lg16.clone(), dlogits16=None), dict(loss_rows=torch.zeros(N + 1, device=DEV)),
           dict(logits32=torch.zeros(N, 4, device=DEV))]
    e.softmax_kd_head(**ok)
    torch.cuda.synchronize()
    for b in bad:
        if b.get("dlogits16", 0) is None:   # the teacher's logits as the output
            b = {**b, "dlogits16": b["tlogits16"]}
        with pytest.raises(RuntimeError):
            e.softmax_kd_head(**{**ok, **b})
    torch.cuda.synchronize()


# ================================================================================================ engines
N_ENG, S_ENG = 16, 224
STUDENTS = [("resnet50", None), ("mobilenetv2", 19), ("mobilenetv2", 14)]
TEACHERS = [("resnet50", None), ("mobilenetv2", 14)]
PAIRS = [(s, t) for s in STUDENTS for t in TEACHERS]
IDS = [f"{s[0]}{'' if s[1] is None else s[1]}-from-{t[0]}{'' if t[1] is None else t[1]}" for s, t in PAIRS]


def _engine(arch, k, augmentation=None, seed=0):
    if arch == "resnet50":
        from b200ddl.models.resnet_engine import ResNet50Engine

        return ResNet50Engine(batch=N_ENG, num_classes=5, image_size=S_ENG, seed=seed, augmentation=augmentation)
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    return MobileNetV2Engine(batch=N_ENG, num_classes=5, image_size=S_ENG, dropout=0.0, seed=seed, fine_tune_at=k,
                             augmentation=augmentation)


def _batch(seed=1):
    g = gen(seed)
    x = torch.randint(0, 256, (N_ENG, S_ENG, S_ENG, 3), device=DEV, dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (N_ENG,), device=DEV, generator=g)
    return x, y


def _distilling(student, teacher, alpha=0.1, T=3.0, eps=0.0, accum=None, use_graph=True, seed=5):
    """A student engine with augmentation (+ CutMix) distilling from a fresh teacher engine, and its training step."""
    from b200ddl import optim
    from b200ddl.models.resnet_engine import EngineTrainStep
    from b200ddl.train.losses import Distillation

    s = _engine(*student, _aug(**AUG, cutmix=1.0), seed=seed)
    t = _engine(*teacher, None, seed=11)
    s.label_smoothing = eps
    s.set_distillation(Distillation(t, alpha, T, eps))
    opt = optim.SGD(0.01, momentum=0.9, gradient_accumulation_steps=accum)
    return s, t, EngineTrainStep(s, opt, use_graph=use_graph)


def _teacher_eval_logits16(t, x):
    from b200ddl.models.resnet_engine import EngineEvalStep

    if not hasattr(t, "_test_eval"):
        t._test_eval = EngineEvalStep(t, use_graph=True)
    t.set_input(x, None)
    t._test_eval.run()
    torch.cuda.synchronize()
    return t.logits16.clone()


@pytest.mark.parametrize("student,teacher", PAIRS, ids=IDS)
def test_graphed_step_teacher_logits_head_and_eager(student, teacher):
    """Graphed steps t = 1, 2: the teacher's logits16 equal the teacher's own EngineEvalStep on the uint8 batch the
    student's stem read, bit for bit; the student's loss rows, stats and dlogits are within kd_bounds of its own
    logits32 and the teacher's logits.  Eager steps give the same stem batches and teacher logits at both steps, and a
    MobileNetV2 student the same logits, dlogits and loss rows at step 1; the stats (sums by atomicAdd, in no fixed
    order) agree within 2 B u sum |term|.  Step 2's student outputs depend on weights updated by atomically accumulated
    gradients, and ResNet-50's training-mode BatchNorm statistics are atomically accumulated sums too."""
    from b200ddl.models.augment import augment_key, mix_params_reference

    x, y = _batch()
    runs = {}
    for use_graph in (True, False):
        s, t, step = _distilling(student, teacher, alpha=0.3, T=4.0, eps=0.1, use_graph=use_graph)
        out = []
        for it in (1, 2):
            step.load(x, y)
            step.run()
            torch.cuda.synchronize()
            name = f"{student} <- {teacher} graph={use_graph} step {it}"
            stem_in = s._stem_input(True).clone()
            tl = t.logits16.clone()
            out.append([stem_in, tl, s.logits.clone(), s.dlogits16.clone(), s.loss_rows.clone(), s.stats.clone()])
            K = s.num_classes
            tlogit = (tl[:, :K].float() + t.p("fc.bias")).double()
            rows = mix_params_reference(s.augmentation, N_ENG, S_ENG, S_ENG, augment_key(5, 0), it, device=DEV)
            check_equal(name + " mix rows", s._augmenter.mix, rows)
            loss, lb, ce, ceb, kd, kdb, d, db = kd_bounds(s.logits.double(), tlogit, y, rows, 0.1, 0.3, 4.0, 1.0 / N_ENG)
            check_bound(name + " loss rows", s.loss_rows, loss, lb)
            check_bound(name + " dlogits", s.dlogits16[:, :K], d, db + 2.0 ** -8 * (d.abs() + db))
            for i, (v, b_) in ((0, (loss, lb)), (2, (ce, ceb)), (3, (kd, kdb))):
                check_bound(f"{name} stats[{i}]", s.stats[i:i + 1], v.sum().view(1),
                            (b_.sum() + N_ENG * U * v.abs().sum()).view(1))
            check_equal(name + " teacher logits16 vs its EngineEvalStep", tl, _teacher_eval_logits16(t, stem_in))
        runs[use_graph] = out
    names = ("stem input", "teacher logits16", "logits32", "dlogits16", "loss rows")
    for it in range(2):
        exact = 5 if it == 0 and student[0] == "mobilenetv2" else 2
        for nm, a, b in list(zip(names, runs[True][it], runs[False][it]))[:exact]:
            check_equal(f"{student} <- {teacher}: eager vs graphed step {it + 1} {nm}", b, a,
                        _pix if nm == "stem input" else None)
    if student[0] == "mobilenetv2":
        rows, st_g, st_e = runs[True][0][4].double(), runs[True][0][5].double(), runs[False][0][5]
        assert float(st_g[1]) == float(st_e[1]), "eager vs graphed step 1: accuracy count"
        check_bound(f"{student} <- {teacher}: eager vs graphed step 1 loss sum", st_e[:1], st_g[:1],
                    (2 * N_ENG * U * rows.abs().sum()).view(1))


@pytest.mark.parametrize("student,teacher", PAIRS, ids=IDS)
def test_accumulation_runs_the_teacher_on_every_micro_batch(student, teacher):
    """gradient_accumulation_steps = 2 (two graphs): after each of four steps the teacher's logits are those of that
    step's stem input."""
    x, y = _batch(seed=2)
    s, t, step = _distilling(student, teacher, accum=2)
    prev = None
    for it in range(4):
        step.load(x, y)
        step.run()
        torch.cuda.synchronize()
        tl = t.logits16.clone()
        check_equal(f"{student} <- {teacher} accum step {it + 1}: teacher logits16", tl,
                    _teacher_eval_logits16(t, s._stem_input(True).clone()))
        assert prev is None or not torch.equal(prev, tl), "the augmented batch changes every step"
        prev = tl


@pytest.mark.parametrize("student,teacher", PAIRS, ids=IDS)
def test_launch_counts(student, teacher):
    """Launches per step of a distilling student = the same student's plain step + the teacher's logits launches (the
    head is swapped one for one); the teacher's weights and statistics never change."""
    from b200ddl import ops, optim
    from b200ddl.models.resnet_engine import EngineTrainStep

    def per_step(step):
        step.load(x, y)
        step.run()
        torch.cuda.synchronize()
        n0 = ops.kernel_launches()
        step.load(x, y)
        step.run()
        torch.cuda.synchronize()
        return ops.kernel_launches() - n0

    x, y = _batch()
    plain = per_step(EngineTrainStep(_engine(*student, _aug(**AUG, cutmix=1.0), seed=5), optim.SGD(0.01),
                                     use_graph=False))
    s, t, step = _distilling(student, teacher, use_graph=False)
    p0, r0 = t.params.clone(), t.running.clone()
    sd0 = t.state_dict()
    distilling = per_step(step)
    n0 = ops.kernel_launches()
    t.forward_logits(False, teacher=True)
    torch.cuda.synchronize()
    teacher_launches = ops.kernel_launches() - n0
    print(f"{student} <- {teacher}: plain {plain}, teacher {teacher_launches}, distilling {distilling}")
    assert distilling == plain + teacher_launches
    assert torch.equal(t.params, p0) and torch.equal(t.running, r0)
    for k, v in t.state_dict().items():
        assert torch.equal(v, sd0[k]), k


@pytest.mark.parametrize("student,teacher", [PAIRS[0], PAIRS[5]], ids=[IDS[0], IDS[5]])
def test_evaluate_and_predict_never_run_the_teacher(student, teacher):
    """Trainer.fit with Distillation logs the four terms; evaluate and predict call no teacher forward and equal those
    of the same student compiled with CategoricalCrossentropy(label_smoothing) alone."""
    from b200ddl import optim
    from b200ddl.train import Trainer
    from b200ddl.train.losses import CategoricalCrossentropy, Distillation

    x, y = _batch(seed=3)
    s = _engine(*student, _aug(**AUG), seed=5)
    t = _engine(*teacher, None, seed=11)
    tr = Trainer(s).compile(optim.SGD(0.01), loss=Distillation(t, 0.2, 2.0, 0.1))
    h = tr.fit([(x, y)], epochs=2, verbose=0).history
    for key in ("loss", "accuracy", "student_loss", "distillation_loss"):
        assert len(h[key]) == 2 and all(v == v for v in h[key]), key
    assert h["loss"][0] == pytest.approx(0.2 * h["student_loss"][0] + 0.8 * h["distillation_loss"][0], rel=1e-4)
    calls = []
    orig = t.forward_logits
    t.forward_logits = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    ev = tr.evaluate([(x, y)])
    pr = tr.predict(x.cpu().numpy())
    assert calls == []
    del t.forward_logits
    plain = Trainer(s).compile(optim.SGD(0.01), loss=CategoricalCrossentropy(from_logits=True, label_smoothing=0.1))
    ev_plain = plain.evaluate([(x, y)])   # the loss sum is accumulated by atomicAdd: equal up to its order
    assert ev_plain[1] == ev[1] and ev_plain[0] == pytest.approx(ev[0], rel=N_ENG * U * 4)
    assert (plain.predict(x.cpu().numpy()) == pr).all()
    assert set(tr.get_weights()) == set(s.state_dict())


def test_mobilenet_gradients_match_torch_module_with_a_resnet_teacher():
    """MobileNetV2 fine_tune_at=14 student, ResNet-50 teacher, CutMix, eps = 0.1, alpha = 0.3, T = 4: every trainable
    gradient against the fp32 `FrozenBaseClassifier` trained on `distillation_reference` with the engine teacher's
    logits, on the reference mixed batch, within the bound of test_mix's engine-vs-module check (4x the bf16-autocast
    distance, floor 2e-2)."""
    from b200ddl.models.augment import augment_key, augment_reference, distillation_reference, mix_params_reference
    from b200ddl.models.mobilenet import FrozenBaseClassifier, MobileNetV2Base
    from test_mobilenet_finetune import _grad_as_torch, _rel

    eps, alpha, T = 0.1, 0.3, 4.0
    s, t, _ = _distilling(("mobilenetv2", 14), ("resnet50", None), alpha, T, eps, seed=3)
    x, y = _batch(seed=14)
    s.set_input(x, y)
    s.set_augment_step(1)
    s.forward(training=True)
    s.backward()
    torch.cuda.synchronize()
    key = augment_key(3, 0)
    xm = augment_reference(s.augmentation, x, key, 1)
    rows = mix_params_reference(s.augmentation, N_ENG, S_ENG, S_ENG, key, 1, device=DEV)
    tlogit = t.logits16[:, :5].float() + t.p("fc.bias")
    base = MobileNetV2Base()
    mod = FrozenBaseClassifier(base, base.out_channels, 5, 0.0, True, 14).to(DEV)
    mod.load_state_dict({n: v.to(DEV) for n, v in s.state_dict().items()})
    mod.train()
    xin = xm.permute(0, 3, 1, 2).float() / 127.5 - 1.0
    grads = {}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    for mode in ("fp32", "autocast"):
        mod.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "autocast"):
            logits = mod(xin).float()
        distillation_reference(logits, tlogit, y, rows, eps, alpha, T)[0].mean().backward()
        grads[mode] = {n: p.grad.detach().float().cpu() for n, p in mod.named_parameters() if p.requires_grad}
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    names = [sp.name for sp in s.param_specs]
    assert sorted(names) == sorted(grads["fp32"])
    worst = sorted(((_rel(_grad_as_torch(s, n), grads["fp32"][n]) / max(4 * _rel(grads["autocast"][n],
                                                                                  grads["fp32"][n]), 2e-2), n)
                    for n in names), reverse=True)
    print("worst gradient distances (ratio to gate, name):", worst[:5])
    assert worst[0][0] <= 1.0, f"gradient off: {worst[:5]}"
