"""Color augmentation: the augment_color kernel alone, and what it adds to a training step.

    python benchmarks/color_times.py [--batch 256] [--small 32] [--size 224] [--steps 20] [--pairs 2] [--iters 25] [--json OUT.json]

Kernel times at batch x size^2, in place on the warp's output as the engines run it: before every launch, outside the
timed events, ``out`` is restored from a saved copy of the warp output of a random batch (so each launch colors a
freshly warped batch, never the output of an earlier launch) and the L2 is flushed by a 256 MB memset; CUDA events
around one launch, the median of ``--iters`` launches.  They are set against the least time their bytes need at
3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth at 700 W).  The bytes are one read and one write of the
batch for both variants: with contrast the kernel reads each image twice, the second time meant to come from L2.
- every color field on (contrast: a per-image reduction, a cluster barrier, then the chain) at the cluster size the
  launch picks, and at every forced cluster size;
- every color field but contrast (one pass, no barrier);
- augment_warp on the same batch, for scale;
- every color field on at batch ``--small``, at the cluster size the launch picks and at every forced one.
Step times: ResNet-50 and MobileNetV2 with fine_tune_at=19 and 14, SGD with momentum, the whole step one CUDA graph,
in ``--pairs`` alternating rounds over the arms: geometric augmentation only, geometric + every color field, and
every color field alone.  Each arm is the mean over ``--steps`` graph replays after 3 warm-up steps.  The card's name,
power limit and maximum SM clock are read in the same run.
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
GEO = dict(flip="horizontal", rotation=0.2, zoom=0.2, translation=0.1)
COLOR = dict(brightness=0.2, contrast=0.3, saturation=0.3, hue=0.1, grayscale=0.2)
NO_CONTRAST = {k: v for k, v in COLOR.items() if k != "contrast"}
ARMS = {"geometric": Augmentation(**GEO), "geometric+color": Augmentation(**GEO, **COLOR),
        "color": Augmentation(**COLOR)}
ARCHS = {"resnet50": None, "mobilenetv2_k19": 19, "mobilenetv2_k14": 14}


def step_time(arch, aug, N, S, steps):
    if arch == "resnet50":
        eng = ResNet50Engine(batch=N, num_classes=5, image_size=S, augmentation=aug)
    else:
        eng = MobileNetV2Engine(batch=N, num_classes=5, image_size=S, fine_tune_at=ARCHS[arch], augmentation=aug)
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


def time_color(aug, warped, flush, iters, cluster=0, warmup=5) -> float:
    """Median microseconds of augment_color in place on ``aug.out`` holding ``warped``, restored (and the L2 flushed)
    before every launch, outside the timed events."""
    ts = []
    for i in range(warmup + iters):
        aug.out.copy_(warped)
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        aug.run_color(cluster)
        e.record()
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append(s.elapsed_time(e) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def kernel_rows(N, S, iters, one_pass_rows=True):
    x = torch.randint(0, 256, (N, S, S, 3), device="cuda", dtype=torch.uint8)
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    full = DeviceAugmenter(Augmentation(**GEO, **COLOR), x, seed=0)
    one_pass = DeviceAugmenter(Augmentation(**GEO, **NO_CONTRAST), x, seed=0)
    for a in (full, one_pass):
        a.set_step(1)
        a.run_params()
        a.run_warp()
    torch.cuda.synchronize()
    warped = full.out.clone()   # the geometric parameters do not depend on the color fields: one warp serves both
    assert torch.equal(warped, one_pass.out)
    nb = 2 * x.numel()
    time_color(full, warped, flush, iters)   # discarded: the first timed series of a process runs slow
    G = full.run_color()
    rows = [(f"augment_color all fields, G={G} (picked)", time_color(full, warped, flush, iters), nb)]
    for g in (1, 2, 4, 8):
        rows.append((f"augment_color all fields, G={g}", time_color(full, warped, flush, iters, g), nb))
    if not one_pass_rows:
        return rows
    G1 = one_pass.run_color()
    rows += [(f"augment_color no contrast, G={G1} (picked)", time_color(one_pass, warped, flush, iters), nb),
             ("augment_warp", time_launch(full.run_warp, flush, iters), nb)]
    # what the timed launches colored: a fresh warp output, with most pixels still chromatic
    full.out.copy_(warped)
    full.run_color()
    torch.cuda.synchronize()
    chroma = lambda t: float((t.amax(-1) > t.amin(-1)).float().mean())   # noqa: E731
    print(f"pixels with max > min: warp output {chroma(warped):.0%}, after one color launch {chroma(full.out):.0%}")
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--small", type=int, default=32)
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
    out = {"card": card(), "batch": N, "size": S, "kernels": {}, "steps": {},
           "arms": {k: a.to_dict() for k, a in ARMS.items()}}
    print(f"\nkernels alone, batch {N} at {S}x{S}, median of {args.iters} launches each, L2 flushed before each")
    rows = kernel_rows(N, S, args.iters)
    print(f"{'launch':40s} {'us':>9s} {'MB':>8s} {'bound us':>9s} {'of bound':>9s}")
    for name, us, nb in rows:
        floor = nb / PEAK_BYTES * 1e6
        print(f"{name:40s} {us:9.1f} {nb / 1e6:8.2f} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"][name] = {"us": us, "bytes": nb, "bound_us": floor}
    print(f"\nsmall batch: augment_color all fields, batch {args.small} at {S}x{S}, same method")
    for name, us, nb in kernel_rows(args.small, S, args.iters, one_pass_rows=False):
        floor = nb / PEAK_BYTES * 1e6
        print(f"{name:40s} {us:9.1f} {nb / 1e6:8.2f} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"][f"batch {args.small}: {name}"] = {"us": us, "bytes": nb, "bound_us": floor}
    torch.cuda.empty_cache()
    print(f"\ntraining step, ms (mean of {args.steps} graph replays per arm), {args.pairs} alternating rounds")
    for arch in ARCHS:
        res = {arm: [] for arm in ARMS}
        for _ in range(args.pairs):
            for arm, aug in ARMS.items():
                res[arm].append(step_time(arch, aug, N, S, args.steps))
                torch.cuda.empty_cache()
        print(f"{arch:16s} " + " | ".join(f"{arm} {' '.join(f'{v:7.3f}' for v in ts)}" for arm, ts in res.items()))
        out["steps"][arch] = res
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
