"""Optimizer update and gradient-clip kernels at ResNet-50's flat-buffer size, and what they cost in a training step.

    python benchmarks/optimizer_times.py [--batch 256] [--steps 20] [--pairs 3] [--iters 25] [--json OUT.json]

Kernel times: each optimizer's update (`_step_cuda`: one launch, three for Lamb) and each clip mode's passes
(`_clip_cuda`), timed alone on the ResNet-50 engine's flat buffers and tensor segments - CUDA events around one call,
the L2 flushed before each (256 MB memset), the median of ``--iters`` calls - against the least time their bytes need
at 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth at 700 W).  Bytes per element come from BYTES below (fp32 reads
and writes of parameters, gradient and state, plus the 2-byte bf16 copy).  Step times: the ResNet-50 engine at
``--batch`` x 224^2, the whole step one CUDA graph, with SGD(momentum 0.9), SGD(momentum 0.9, global_clipnorm=1.0) and
Lamb, in ``--pairs`` alternating rounds; each arm is the mean over ``--steps`` graph replays after 3 warm-up steps.  The
card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import optim
from b200ddl.models.resnet_engine import EngineTrainStep, ResNet50Engine, _align

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402

PEAK_BYTES = 3.35e12
# bytes per flat-buffer element: p read + write (8), g read (4), each state read + write (8), bf16 copy (2)
BYTES = {"SGD": 22, "Adam": 30, "Adadelta": 30, "RMSprop": 22, "RMSprop(momentum, centered)": 38, "Adagrad": 22,
         "Adamax": 30, "AdamW": 30, "Lamb": 42,
         # pass 1 reads p, g, m, v and writes m, v (24); pass 3 reads p, m, v, writes p and the bf16 copy (18)
         "global_clipnorm": 4, "clipnorm": 12, "clipvalue": 8}   # sum of squares reads g; the apply pass reads + writes g
OPTS = {"SGD": lambda **k: optim.SGD(0.01, momentum=0.9, **k), "Adam": lambda **k: optim.Adam(**k),
        "Adadelta": lambda **k: optim.Adadelta(**k), "RMSprop": lambda **k: optim.RMSprop(**k),
        "RMSprop(momentum, centered)": lambda **k: optim.RMSprop(momentum=0.9, centered=True, **k),
        "Adagrad": lambda **k: optim.Adagrad(**k), "Adamax": lambda **k: optim.Adamax(**k),
        "AdamW": lambda **k: optim.AdamW(**k), "Lamb": lambda **k: optim.Lamb(**k)}
CLIPS = {"global_clipnorm": 1.0, "clipnorm": 1.0, "clipvalue": 0.01}


def step_time(make, N, steps):
    eng = ResNet50Engine(batch=N, num_classes=1000, image_size=224)
    step = EngineTrainStep(eng, make(), use_graph=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 256, (N, 224, 224, 3), device="cuda", dtype=torch.uint8, generator=g)
    y = torch.randint(0, 1000, (N,), device="cuda", generator=g)
    step.load(x, y)
    for _ in range(3):
        step.run()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        step.run()
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
    segs = [(s.offset, s.offset + _align(s.numel)) for s in eng.param_specs]
    del eng
    p = torch.randn(n, device="cuda") * 0.05
    g = torch.randn(n, device="cuda") * 1e-3
    w16 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = []
    for name, make in OPTS.items():
        o = make().attach(p, g, w16, segments=segs)
        o.begin_step()
        rows.append((name, time_launch(o._step_cuda, flush, args.iters), BYTES[name] * n))
    for clip, c in CLIPS.items():
        o = optim.SGD(0.01, **{clip: c}).attach(p, g, w16, segments=segs)
        o.begin_step()
        rows.append((clip, time_launch(o._clip_cuda, flush, args.iters), BYTES[clip] * n))
    print(f"\nalone, {n / 1e6:.2f} M elements in {len(segs)} tensors, median of {args.iters} calls, L2 flushed before each")
    print(f"{'launches':28s} {'us':>9s} {'B/elem':>7s} {'bound us':>9s} {'of bound':>9s}")
    for name, us, nb in rows:
        floor = nb / PEAK_BYTES * 1e6
        print(f"{name:28s} {us:9.1f} {nb / n:7.0f} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"][name] = {"us": us, "bytes": nb, "bound_us": floor}
    del p, g, w16, flush
    torch.cuda.empty_cache()
    arms = {"SGD": lambda: optim.SGD(0.01, momentum=0.9),
            "SGD(global_clipnorm=1.0)": lambda: optim.SGD(0.01, momentum=0.9, global_clipnorm=1.0),
            "Lamb": lambda: optim.Lamb(1e-3)}
    res = {k: [] for k in arms}
    for _ in range(args.pairs):
        for k, make in arms.items():
            res[k].append(step_time(make, args.batch, args.steps))
            torch.cuda.empty_cache()
    print(f"\nResNet-50 training step at batch {args.batch}, ms (mean of {args.steps} graph replays per arm), "
          f"alternating rounds")
    for k, v in res.items():
        added = [(a - b) / b for a, b in zip(v, res["SGD"])]
        print(f"{k:26s} {' '.join(f'{t:7.3f}' for t in v)} | vs SGD {' '.join(f'{a:+.2%}' for a in added)}")
    out["steps"] = res
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
