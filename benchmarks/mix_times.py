"""MixUp, CutMix and label smoothing: the new kernels against the ones they replace, and what each option adds to a step.

    python benchmarks/mix_times.py [--batch 256] [--size 224] [--classes 1000] [--steps 20] [--pairs 2] [--iters 25]
                                   [--json OUT.json]

Kernel times at batch x size^2 (CUDA events around one launch, the L2 flushed before each by a 256 MB memset, the
median of ``--iters`` launches), against the least time their bytes need at 3.35 TB/s (the H100 SXM data-sheet HBM3
bandwidth at 700 W):
- augment_params against augment_mix_params (the same launch writing the mix rows too);
- augment_warp against the MixUp warp (reads the taps of two images: the batch twice) and the CutMix warp (once);
- softmax_ce_head against softmax_ce_soft_head, both on bf16 logits [batch, ``--classes``] with dlogits.
Step times: ResNet-50 and MobileNetV2 with fine_tune_at=19 and 14, SGD with momentum, the whole step one CUDA graph,
in ``--pairs`` alternating rounds over the arms: plain, geometric augmentation only, + mixup=0.2, + cutmix=1.0, and
label_smoothing=0.1 alone.  Each arm is the mean over ``--steps`` graph replays after 3 warm-up steps.  The card's name,
power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import ops, optim
from b200ddl.models.augment import Augmentation, DeviceAugmenter
from b200ddl.models.mobilenet_engine import MobileNetV2Engine
from b200ddl.models.resnet_engine import EngineTrainStep, ResNet50Engine

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402

PEAK_BYTES = 3.35e12
GEO = dict(flip="horizontal", rotation=0.2, zoom=0.2, translation=0.1)
ARMS = {"plain": (None, 0.0), "geometric": (Augmentation(**GEO), 0.0),
        "+mixup": (Augmentation(**GEO, mixup=0.2), 0.0), "+cutmix": (Augmentation(**GEO, cutmix=1.0), 0.0),
        "smoothing": (None, 0.1)}
ARCHS = {"resnet50": None, "mobilenetv2_k19": 19, "mobilenetv2_k14": 14}


def step_time(arch, aug, eps, N, S, steps):
    if arch == "resnet50":
        eng = ResNet50Engine(batch=N, num_classes=5, image_size=S, augmentation=aug)
    else:
        eng = MobileNetV2Engine(batch=N, num_classes=5, image_size=S, fine_tune_at=ARCHS[arch], augmentation=aug)
    eng.label_smoothing = eps
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


def kernel_rows(N, S, K, iters):
    x = torch.randint(0, 256, (N, S, S, 3), device="cuda", dtype=torch.uint8)
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    geo = DeviceAugmenter(Augmentation(**GEO), x, seed=0)
    mixup = DeviceAugmenter(ARMS["+mixup"][0], x, seed=0)
    cutmix = DeviceAugmenter(ARMS["+cutmix"][0], x, seed=0)
    for a in (geo, mixup, cutmix):
        a.set_step(1)
        a.run_params()
    table = 4 * geo.rot_table.numel()
    rows = [("augment_params", time_launch(geo.run_params, flush, iters), 32 * N + table),
            ("augment_mix_params", time_launch(mixup.run_params, flush, iters), 64 * N + 2 * table),
            ("augment_warp", time_launch(geo.run_warp, flush, iters), 2 * x.numel()),
            ("augment_mix_warp mixup", time_launch(mixup.run_warp, flush, iters), 3 * x.numel()),
            ("augment_mix_warp cutmix", time_launch(cutmix.run_warp, flush, iters), 2 * x.numel())]
    e = ops.ext("_b200_ops")
    ld = (K + 127) // 128 * 128
    g = torch.Generator(device="cuda").manual_seed(1)
    lg16 = (torch.randn(N, ld, device="cuda", generator=g) * 4).to(torch.bfloat16)
    bias = torch.randn(K, device="cuda", generator=g)
    labels = torch.randint(0, K, (N,), device="cuda", generator=g)
    logits32, dl16 = torch.empty(N, K, device="cuda"), torch.empty(N, ld, device="cuda", dtype=torch.bfloat16)
    loss_rows, stats = torch.empty(N, device="cuda"), torch.zeros(2, device="cuda")
    head_bytes = N * ld * 2 + K * 4 + N * 8 + N * K * 4 + N * ld * 2 + N * 4
    rows += [("softmax_ce_head", time_launch(lambda: e.softmax_ce_head(lg16, bias, labels, logits32, dl16, loss_rows,
                                                                       stats, 1.0 / N), flush, iters), head_bytes),
             ("softmax_ce_soft_head", time_launch(lambda: e.softmax_ce_soft_head(lg16, bias, labels, cutmix.mix, 0.1,
                                                                                 logits32, dl16, loss_rows, stats,
                                                                                 1.0 / N), flush, iters),
              head_bytes + 32 * N + 8 * N)]
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=2)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    N, S = args.batch, args.size
    print("card:", card())
    out = {"card": card(), "batch": N, "size": S, "classes": args.classes, "kernels": {}, "steps": {},
           "arms": {k: (a.to_dict() if a else None, eps) for k, (a, eps) in ARMS.items()}}
    print(f"\nkernels alone, batch {N} at {S}x{S} ({args.classes} classes for the heads), median of {args.iters} "
          f"launches each, L2 flushed before each")
    print(f"{'launch':24s} {'us':>9s} {'MB':>8s} {'bound us':>9s} {'of bound':>9s}")
    for name, us, nb in kernel_rows(N, S, args.classes, args.iters):
        floor = nb / PEAK_BYTES * 1e6
        print(f"{name:24s} {us:9.1f} {nb / 1e6:8.2f} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"][name] = {"us": us, "bytes": nb, "bound_us": floor}
    torch.cuda.empty_cache()
    print(f"\ntraining step, ms (mean of {args.steps} graph replays per arm), {args.pairs} alternating rounds")
    for arch in ARCHS:
        res = {arm: [] for arm in ARMS}
        for _ in range(args.pairs):
            for arm, (aug, eps) in ARMS.items():
                res[arm].append(step_time(arch, aug, eps, N, S, args.steps))
                torch.cuda.empty_cache()
        print(f"{arch:16s} " + " | ".join(f"{arm} {' '.join(f'{v:7.3f}' for v in ts)}" for arm, ts in res.items()))
        out["steps"][arch] = res
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
