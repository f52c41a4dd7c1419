"""Random augmentation in the training step: the two kernels alone, and what they add to a training step.

    python benchmarks/augment_times.py [--batch 256] [--size 224] [--steps 20] [--pairs 3] [--iters 25] [--json OUT.json]

Kernel times: `augment_params` and `augment_warp` (csrc/augment.cu) at batch x size^2, each timed alone - CUDA events
around one launch, the L2 flushed before each (256 MB memset), the median of ``--iters`` launches - against the least
time their bytes need at 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth at 700 W; the warp reads the batch once and
writes it once).  Step times: the ResNet-50 engine and the MobileNetV2 engine with fine_tune_at=19 (head only), SGD
with momentum, the whole step one CUDA graph, without and with augmentation in ``--pairs`` alternating pairs; each arm
is the mean over ``--steps`` graph replays after 3 warm-up steps.  The card's name, power limit and maximum SM clock are
read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import optim
from b200ddl.models.augment import Augmentation, DeviceAugmenter
from b200ddl.models.mobilenet_engine import MobileNetV2Engine
from b200ddl.models.resnet_engine import EngineTrainStep, ResNet50Engine

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402

PEAK_BYTES = 3.35e12
AUG = Augmentation("horizontal", rotation=0.2, zoom=0.2, translation=0.1)


def step_time(arch, aug, N, S, steps):
    if arch == "resnet50":
        eng = ResNet50Engine(batch=N, num_classes=5, image_size=S, augmentation=aug)
    else:
        eng = MobileNetV2Engine(batch=N, num_classes=5, image_size=S, fine_tune_at=19, augmentation=aug)
    step = EngineTrainStep(eng, optim.SGD(0.01, momentum=0.9), use_graph=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 256, (N, S, S, 3), device="cuda", dtype=torch.uint8, generator=g)
    y = torch.randint(0, 5, (N,), device="cuda", generator=g)
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
    out = {"card": card(), "batch": N, "size": S, "augmentation": AUG.to_dict(), "kernels": {}, "steps": {}}
    x = torch.randint(0, 256, (N, S, S, 3), device="cuda", dtype=torch.uint8)
    a = DeviceAugmenter(AUG, x, seed=0)
    a.set_step(1)
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = [("augment_params", time_launch(a.run_params, flush, args.iters), a.params.numel() * 4 + a.rot_table.numel() * 4),
            ("augment_warp", time_launch(a.run_warp, flush, args.iters), 2 * x.numel())]
    print(f"\nkernels alone, batch {N} at {S}x{S}, median of {args.iters} launches each, L2 flushed before each")
    print(f"{'launch':16s} {'us':>9s} {'MB':>8s} {'bound us':>9s} {'of bound':>9s}")
    for name, us, nb in rows:
        floor = nb / PEAK_BYTES * 1e6
        print(f"{name:16s} {us:9.1f} {nb / 1e6:8.2f} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"][name] = {"us": us, "bytes": nb, "bound_us": floor}
    del a, x, flush
    torch.cuda.empty_cache()
    print(f"\ntraining step, ms (mean of {args.steps} graph replays per arm), alternating pairs")
    for arch in ("resnet50", "mobilenetv2_k19"):
        res = {"off": [], "on": []}
        for _ in range(args.pairs):
            for arm, aug in (("off", None), ("on", AUG)):
                res[arm].append(step_time(arch.split("_")[0], aug, N, S, args.steps))
                torch.cuda.empty_cache()
        added = [(on - off) / off for on, off in zip(res["on"], res["off"])]
        print(f"{arch:16s} off {' '.join(f'{v:7.3f}' for v in res['off'])} | on {' '.join(f'{v:7.3f}' for v in res['on'])}"
              f" | added {' '.join(f'{v:+.2%}' for v in added)}")
        out["steps"][arch] = {**res, "added": added}
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
