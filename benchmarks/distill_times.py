"""Knowledge distillation: softmax_kd_head against the head it replaces, and what a teacher adds to a training step.

    python benchmarks/distill_times.py [--batch 256] [--size 224] [--steps 20] [--pairs 2] [--iters 25] [--json OUT.json]

Kernel times at ``--batch`` rows (CUDA events around one launch, the L2 flushed before each by a 256 MB memset, the
median of ``--iters`` launches), at K = 5 and K = 1000 classes: softmax_ce_soft_head and softmax_kd_head (which also
reads the teacher's bf16 logits), both with dlogits and label smoothing 0.1.
Step times, ms: MobileNetV2 with fine_tune_at=14 (geometric augmentation, SGD with momentum, the whole step one CUDA
graph) without a teacher and with a ResNet-50 teacher (alpha 0.1, T 3), and the ResNet-50 teacher's evaluation step
alone (EngineEvalStep, graphed), in ``--pairs`` alternating rounds; each arm is the mean over ``--steps`` graph replays
after 3 warm-up steps.  The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import ops, optim
from b200ddl.models.augment import Augmentation
from b200ddl.models.mobilenet_engine import MobileNetV2Engine
from b200ddl.models.resnet_engine import EngineEvalStep, EngineTrainStep, ResNet50Engine
from b200ddl.train.losses import Distillation

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402

GEO = dict(flip="horizontal", rotation=0.2, zoom=0.2, translation=0.1)
ARMS = ("student", "student+teacher", "teacher eval")


def _batch(N, S):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 256, (N, S, S, 3), device="cuda", dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (N,), device="cuda", generator=g)
    return x, y


def _replays(run, steps):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        run()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def step_time(arm, N, S, steps):
    x, y = _batch(N, S)
    if arm == "teacher eval":
        t = ResNet50Engine(batch=N, num_classes=5, image_size=S)
        ev = EngineEvalStep(t, use_graph=True)
        t.set_input(x, y)
        return _replays(ev.run, steps)
    s = MobileNetV2Engine(batch=N, num_classes=5, image_size=S, fine_tune_at=14, augmentation=Augmentation(**GEO))
    if arm == "student+teacher":
        s.set_distillation(Distillation(ResNet50Engine(batch=N, num_classes=5, image_size=S), 0.1, 3.0))
    step = EngineTrainStep(s, optim.SGD(0.01, momentum=0.9), use_graph=True)
    step.load(x, y)
    return _replays(step.run, steps)


def kernel_rows(N, iters):
    e = ops.ext("_b200_ops")
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = []
    for K in (5, 1000):
        ld = 64 if K <= 64 else (K + 127) // 128 * 128
        g = torch.Generator(device="cuda").manual_seed(K)
        lg16 = (torch.randn(N, ld, device="cuda", generator=g) * 4).to(torch.bfloat16)
        tg16 = (torch.randn(N, ld, device="cuda", generator=g) * 4).to(torch.bfloat16)
        bias, tbias = torch.randn(K, device="cuda", generator=g), torch.randn(K, device="cuda", generator=g)
        labels = torch.randint(0, K, (N,), device="cuda", generator=g)
        logits32, dl16 = torch.empty(N, K, device="cuda"), torch.empty(N, ld, device="cuda", dtype=torch.bfloat16)
        loss_rows, stats = torch.empty(N, device="cuda"), torch.zeros(4, device="cuda")
        rows += [(f"softmax_ce_soft_head K={K}",
                  time_launch(lambda: e.softmax_ce_soft_head(lg16, bias, labels, None, 0.1, logits32, dl16, loss_rows,
                                                             stats, 1.0 / N), flush, iters)),
                 (f"softmax_kd_head K={K}",
                  time_launch(lambda: e.softmax_kd_head(lg16, bias, tg16, tbias, labels, None, 0.1, 0.1, 3.0, logits32,
                                                        dl16, loss_rows, stats, 1.0 / N), flush, iters))]
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=2)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    N, S = args.batch, args.size
    print("card:", card())
    out = {"card": card(), "batch": N, "size": S, "kernels": {}, "steps": {arm: [] for arm in ARMS}}
    print(f"\nheads alone, batch {N}, median of {args.iters} launches each, L2 flushed before each")
    for name, us in kernel_rows(N, args.iters):
        print(f"{name:32s} {us:9.1f} us")
        out["kernels"][name] = us
    torch.cuda.empty_cache()
    print(f"\nms per step (mean of {args.steps} graph replays per arm), {args.pairs} alternating rounds, batch {N} at "
          f"{S}x{S}: MobileNetV2 fine_tune_at=14 student, ResNet-50 teacher")
    for _ in range(args.pairs):
        for arm in ARMS:
            out["steps"][arm].append(step_time(arm, N, S, args.steps))
            torch.cuda.empty_cache()
    for arm in ARMS:
        print(f"{arm:16s} " + " ".join(f"{v:8.3f}" for v in out["steps"][arm]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
