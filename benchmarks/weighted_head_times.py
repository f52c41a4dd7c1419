"""Loss weighting: the weighted head kernels against the unweighted ones, and what class_weight adds to a training step.

    python benchmarks/weighted_head_times.py [--batch 256] [--size 224] [--steps 20] [--pairs 3] [--iters 25] [--json OUT]

Kernel times at ``--batch`` rows (CUDA events around one launch, the L2 flushed before each by a 256 MB memset, the
median of ``--iters`` launches), at K = 5 and K = 1000 classes, with dlogits: softmax_ce_head, softmax_ce_soft_head
(label smoothing 0.1) and softmax_kd_head (alpha 0.1, T 3), each unweighted and with a class-weight table.
Step times, ms: ResNet-50 (fine_tune_at=17) and MobileNetV2 (fine_tune_at=19), SGD with momentum, the whole step one
CUDA graph, without and with class_weight, in ``--pairs`` alternating rounds; each arm is the mean over ``--steps``
graph replays after 3 warm-up steps.  The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import ops, optim
from b200ddl.models.mobilenet_engine import MobileNetV2Engine
from b200ddl.models.resnet_engine import EngineTrainStep, ResNet50Engine

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402
from distill_times import _batch, _replays  # noqa: E402

ENGINES = (("ResNet-50 fine_tune_at=17", lambda N, S: ResNet50Engine(batch=N, num_classes=5, image_size=S,
                                                                     fine_tune_at=17)),
           ("MobileNetV2 fine_tune_at=19", lambda N, S: MobileNetV2Engine(batch=N, num_classes=5, image_size=S,
                                                                          fine_tune_at=19)))


def step_time(make, weighted, N, S, steps):
    eng = make(N, S)
    if weighted:
        eng.set_weighting("class")
        eng.set_class_weight(torch.tensor([1.0, 2.5, 0.5, 1.0, 4.0]))
    step = EngineTrainStep(eng, optim.SGD(0.01, momentum=0.9), use_graph=True)
    step.load(*_batch(N, S))
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
        table = torch.rand(K, device="cuda", generator=g) * 3
        logits32, dl16 = torch.empty(N, K, device="cuda"), torch.empty(N, ld, device="cuda", dtype=torch.bfloat16)
        loss_rows, stats = torch.empty(N, device="cuda"), torch.zeros(4, device="cuda")
        out = (logits32, dl16, loss_rows, stats, 1.0 / N)
        heads = {"softmax_ce_head": lambda **w: e.softmax_ce_head(lg16, bias, labels, *out, **w),
                 "softmax_ce_soft_head": lambda **w: e.softmax_ce_soft_head(lg16, bias, labels, None, 0.1, *out, **w),
                 "softmax_kd_head": lambda **w: e.softmax_kd_head(lg16, bias, tg16, tbias, labels, None, 0.1, 0.1, 3.0,
                                                                  *out, **w)}
        for name, run in heads.items():
            rows += [(f"{name} K={K}", time_launch(run, flush, iters)),
                     (f"{name} K={K} weighted", time_launch(lambda: run(class_weight=table), flush, iters))]
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    N, S = args.batch, args.size
    print("card:", card())
    out = {"card": card(), "batch": N, "size": S, "kernels": {}, "steps": {}}
    print(f"\nheads alone, batch {N}, median of {args.iters} launches each, L2 flushed before each")
    for name, us in kernel_rows(N, args.iters):
        print(f"{name:40s} {us:9.1f} us")
        out["kernels"][name] = us
    torch.cuda.empty_cache()
    print(f"\nms per step (mean of {args.steps} graph replays per arm), {args.pairs} alternating rounds, batch {N} at "
          f"{S}x{S}")
    arms = [(f"{name}{' class_weight' if w else ''}", make, w) for name, make in ENGINES for w in (False, True)]
    for _ in range(args.pairs):
        for arm, make, w in arms:
            out["steps"].setdefault(arm, []).append(step_time(make, w, N, S, args.steps))
            torch.cuda.empty_cache()
    for arm, _, _ in arms:
        print(f"{arm:42s} " + " ".join(f"{v:8.3f}" for v in out["steps"][arm]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
