"""ResNet-50 fine-tuning on the native engine: training-step time and peak memory per `fine_tune_at` and BatchNorm mode.

    python benchmarks/resnet_finetune_times.py [--batch 256] [--size 224] [--steps 20] [--rounds 2] [--json OUT.json]

Arms: the fully trainable `arch="resnet50"` step, its evaluation step, and `ResNet50Engine(fine_tune_at=k, batchnorm=m)`
for k in 17, 14, 8, 4, 0 and m in "inference", "training" (k = 17 has no trainable BatchNorm: one arm).  SGD with
momentum; every step is one CUDA graph.  The arms take turns over ``--rounds`` rounds: in every round each arm is built,
warmed up with 3 steps and replays ``--steps`` steps between two CUDA events, then is freed.  The table gives the mean
ms/step of the best round, the spread (max - min over rounds), and the `torch.cuda.max_memory_allocated` of building
and stepping that arm alone (reset before each build).  The card's name, power limit and maximum
SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import optim
from b200ddl.models.resnet_engine import EngineEvalStep, EngineTrainStep, ResNet50Engine

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card  # noqa: E402

ARMS = [("resnet50", None, None), ("resnet50 eval", None, "eval")] + \
    [(f"resnet50_head k={k} {m}", k, m) for k in (17, 14, 8, 4, 0) for m in ("inference", "training")
     if not (k == 17 and m == "training")]


def make(arm, N, S):
    _, k, m = arm
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 256, (N, S, S, 3), device="cuda", dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (N,), device="cuda", generator=g)
    if m == "eval":
        eng = ResNet50Engine(batch=N, num_classes=5, image_size=S)
        EngineTrainStep(eng, optim.SGD(0.01, momentum=0.9), use_graph=True)   # evaluate on the training build, as fit does
        step = EngineEvalStep(eng, use_graph=True)
        eng.set_input(x, y)
    else:
        kw = {} if k is None else dict(fine_tune_at=k, batchnorm=m)
        eng = ResNet50Engine(batch=N, num_classes=5, image_size=S, **kw)
        step = EngineTrainStep(eng, optim.SGD(0.01, momentum=0.9), use_graph=True)
        step.load(x, y)
    for _ in range(3):
        step.run()
    torch.cuda.synchronize()
    return eng, step


def window(step, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        step.run()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    info = card()
    print(f"card: {info}")
    # the arms take turns: each is built, warmed up, timed and freed in every round (all of them at batch 256 do not
    # fit in memory at once); its peak memory is that of its own build and steps
    times = {arm[0]: [] for arm in ARMS}
    peak = {}
    for _ in range(a.rounds):
        for arm in ARMS:
            gc.collect()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            eng, step = make(arm, a.batch, a.size)
            times[arm[0]].append(window(step, a.steps))
            peak[arm[0]] = torch.cuda.max_memory_allocated() / 2 ** 30
            del eng, step
    rows = []
    print(f"batch {a.batch}, {a.size}x{a.size}, SGD + momentum, one CUDA graph per step, best of {a.rounds} rounds "
          f"of {a.steps} steps")
    print(f"{'arm':34s} {'ms/step':>8s} {'spread':>7s} {'peak GiB':>9s}")
    for name, ts in times.items():
        rows.append({"arm": name, "ms": min(ts), "spread": max(ts) - min(ts), "peak_gib": peak[name]})
        print(f"{name:34s} {min(ts):8.2f} {max(ts) - min(ts):7.2f} {peak[name]:9.2f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": info, "batch": a.batch, "size": a.size, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
