"""Gradient accumulation and weight EMA: their kernels at ResNet-50's flat-buffer size, and what they cost in a step.

    python benchmarks/accum_ema_times.py [--batch 256] [--steps 20] [--pairs 3] [--iters 25] [--json OUT.json]

Kernel times: `grad_accumulate` (accumulate: accum += g; combine: g = (accum + g) / n, accum = 0) and `ema_update`
(without and with the overwrite of p and the bf16 copy), timed alone on the ResNet-50 engine's flat buffers - CUDA
events around one call, the L2 flushed before each (256 MB memset), the median of ``--iters`` calls - against the least
time their bytes need at 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth at 700 W).  Bytes per parameter: accumulate
reads g and reads + writes accum (12), combine reads and writes both (16), the EMA reads p and reads + writes ema (12),
and an overwrite also writes p and the bf16 copy (+6).  Step times: the ResNet-50 engine at ``--batch`` x 224^2, each
step variant one CUDA graph, in ``--pairs`` alternating rounds: SGD(momentum 0.9); the same with
gradient_accumulation_steps=4, its accumulation graph and its update graph timed separately; and with use_ema=True.
Each arm is the mean over ``--steps`` replays of its graph after 3 warm-up replays.  The card's name, power limit and
maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import ops, optim
from b200ddl.models.resnet_engine import EngineTrainStep, ResNet50Engine

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402

PEAK_BYTES = 3.35e12
BYTES = {"accumulate": 12, "combine": 16, "ema": 12, "ema + overwrite": 18}


def step_time(make, variant, N, steps):
    """Mean ms of one replay of the step graph `variant` ('update' or 'accumulate')."""
    eng = ResNet50Engine(batch=N, num_classes=1000, image_size=224)
    step = EngineTrainStep(eng, make(), use_graph=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 256, (N, 224, 224, 3), device="cuda", dtype=torch.uint8, generator=g)
    y = torch.randint(0, 1000, (N,), device="cuda", generator=g)
    step.load(x, y)
    step.capture()
    graph = step.graph if variant == "update" else step.accum_graph
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        graph.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    print("card:", card())
    out = {"card": card(), "batch": args.batch, "kernels": {}, "steps": {}}
    eng = ResNet50Engine(batch=1, num_classes=1000, image_size=224)
    n = eng.flat_numel
    del eng
    e = ops.ext("_b200_ops")
    p = torch.randn(n, device="cuda") * 0.05
    ema = p.clone()
    g = torch.randn(n, device="cuda") * 1e-3
    acc = torch.zeros(n, device="cuda")
    w16 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    hyper = {}
    for over in (False, True):
        h = torch.zeros(16, device="cuda")
        h[10], h[11], h[12] = 0.99, 0.01, float(over)
        hyper[over] = h
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = [("accumulate", time_launch(lambda: e.grad_accumulate(g, acc, 4, 0), flush, args.iters)),
            ("combine", time_launch(lambda: e.grad_accumulate(g, acc, 4, 1), flush, args.iters)),
            ("ema", time_launch(lambda: e.ema_update(p, ema, w16, hyper[False]), flush, args.iters)),
            ("ema + overwrite", time_launch(lambda: e.ema_update(p, ema, w16, hyper[True]), flush, args.iters))]
    print(f"\nalone, {n / 1e6:.2f} M parameters, median of {args.iters} calls, L2 flushed before each")
    print(f"{'kernel':18s} {'us':>9s} {'B/param':>8s} {'bound us':>9s} {'of bound':>9s}")
    for name, us in rows:
        nb = BYTES[name] * n
        floor = nb / PEAK_BYTES * 1e6
        print(f"{name:18s} {us:9.1f} {BYTES[name]:8d} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"][name] = {"us": us, "bytes": nb, "bound_us": floor}
    del p, ema, g, acc, w16, flush
    torch.cuda.empty_cache()
    arms = {"SGD": (lambda: optim.SGD(0.01, momentum=0.9), "update"),
            "n=4 accumulate step": (lambda: optim.SGD(0.01, momentum=0.9, gradient_accumulation_steps=4), "accumulate"),
            "n=4 update step": (lambda: optim.SGD(0.01, momentum=0.9, gradient_accumulation_steps=4), "update"),
            "use_ema=True": (lambda: optim.SGD(0.01, momentum=0.9, use_ema=True), "update")}
    res = {k: [] for k in arms}
    for _ in range(args.pairs):
        for k, (make, variant) in arms.items():
            res[k].append(step_time(make, variant, args.batch, args.steps))
            torch.cuda.empty_cache()
    print(f"\nResNet-50 training step at batch {args.batch}, ms (mean of {args.steps} graph replays per arm), "
          f"alternating rounds")
    for k, v in res.items():
        added = [(a - b) / b for a, b in zip(v, res["SGD"])]
        print(f"{k:22s} {' '.join(f'{t:7.3f}' for t in v)} | vs SGD {' '.join(f'{a:+.2%}' for a in added)}")
    out["steps"] = res
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
