"""MobileNetV2 fine-tuning with training-mode BatchNorm: step times against the alternatives, and the new kernels alone.

    python benchmarks/mobilenet_bn_train_times.py [--batch 256] [--size 224] [--steps 20] [--reps 2] [--iters 25]
                                                  [--json OUT.json]

For k in 14, 8, 0 and ``--reps`` alternating rounds, in this order each round: `MobileNetV2Engine(fine_tune_at=k,
batchnorm="training")`, the same with inference-mode BatchNorm, and the torch module
`FrozenBaseClassifier(fine_tune_at=k, batchnorm="training")` on cuDNN (bf16 autocast, channels_last, torch.optim.SGD).
SGD with momentum; the engines run each step as one CUDA graph, the module eagerly.  Step time = the mean over
``--steps`` steps after 3 warm-up steps, CUDA events around the window.  Each model is built, timed and freed in turn.

Kernel times: on the k = 0 engine, every launch of the new kernels (bn_apply ReLU6, the depthwise / stem statistics
convolutions, relu6_mask_reduce with sum(dz*c)) timed alone with the L2 flushed (conv_layer_times.time_launch), against
the least time its bytes need at 3.35 TB/s (H100 SXM data-sheet HBM3 bandwidth at 700 W; each operand read once, each
output written once).  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch
import torch.nn.functional as F

from b200ddl import optim
from b200ddl.models.mobilenet_engine import MobileNetV2Engine
from b200ddl.models.resnet_engine import EngineTrainStep

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402

PEAK_BYTES = 3.35e12


def _data(N, S):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 256, (N, S, S, 3), device="cuda", dtype=torch.uint8, generator=g)
    return x, torch.randint(0, 5, (N,), device="cuda", generator=g)


def _timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def engine_step(k, batchnorm, N, S, steps, keep=False):
    eng = MobileNetV2Engine(batch=N, num_classes=5, image_size=S, fine_tune_at=k, batchnorm=batchnorm)
    step = EngineTrainStep(eng, optim.SGD(0.01, momentum=0.9), use_graph=True)
    step.load(*_data(N, S))
    ms = _timed(step.run, steps)
    return (ms, eng) if keep else (ms, None)


def module_step(k, N, S, steps):
    from b200ddl.models.mobilenet import FrozenBaseClassifier, MobileNetV2Base

    base = MobileNetV2Base()
    mod = FrozenBaseClassifier(base, base.out_channels, 5, 0.5, True, k, batchnorm="training")
    mod = mod.cuda().to(memory_format=torch.channels_last).train()
    opt = torch.optim.SGD([p for p in mod.parameters() if p.requires_grad], lr=0.01, momentum=0.9)
    x8, y = _data(N, S)
    x = (x8.permute(0, 3, 1, 2).float() / 127.5 - 1.0).contiguous(memory_format=torch.channels_last)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(mod(x).float(), y)
        loss.backward()
        opt.step()

    return _timed(step, steps)


def kernel_rows(eng, flush, iters):
    """(name, microseconds, bytes) of every launch of the new kernels in one training step of `eng`."""
    e, rows = eng._e, []
    for i, lay in enumerate(eng._plan):
        if not lay["train"]:
            continue
        tag = f"{i:02d} {lay['kind']} {lay['conv'][5:]}"
        c, y, x = lay["c"], lay["y"], lay["x"]
        if lay["kind"] == "dw":
            rows.append((f"{tag} dwconv3x3_stats s{lay['stride']}", time_launch(
                lambda: e.dwconv3x3_stats(x, lay["w"], c, lay["ssum"], lay["ssq"], lay["stride"]), flush, iters),
                (x.numel() + c.numel()) * 2))
        elif lay["kind"] == "stem":
            rows.append((f"{tag} mbv2_stem_stats", time_launch(
                lambda: e.mbv2_stem_stats(x, lay["w"], c, lay["ssum"][:32], lay["ssq"][:32], 1.0 / 127.5, -1.0),
                flush, iters), x.numel() + c.numel() // c.shape[-1] * 32 * 2))
        if lay["act"] == "relu6":
            rows.append((f"{tag} bn_apply relu6", time_launch(
                lambda: e.bn_apply(c, lay["bscale"], lay["bshift"], None, None, None, y, True, None, True), flush,
                iters), 2 * c.numel() * 2))
        g, g2 = lay["g"], lay["g2"]
        nb = g.numel() * 2 * (3 + (g2 is not None) + (lay["act"] == "relu6"))   # g1 [+ g2] [+ y] + c in, dz out
        rows.append((f"{tag} mask_reduce+dzc", time_launch(
            lambda: e.relu6_mask_reduce(g, g2, y, g, lay["sum"], lay["act"] == "relu6", c, lay["sumc"]), flush,
            iters), nb))
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    N, S = args.batch, args.size
    print("card:", card())
    out = {"card": card(), "batch": N, "size": S, "steps": []}
    for k in (14, 8, 0):
        for rep in range(args.reps):
            row = {"k": k, "rep": rep}
            for name, fn in (("bn_training", lambda: engine_step(k, "training", N, S, args.steps)[0]),
                             ("bn_inference", lambda: engine_step(k, "inference", N, S, args.steps)[0]),
                             ("torch_module", lambda: module_step(k, N, S, args.steps))):
                row[name] = fn()
                gc.collect()
                torch.cuda.empty_cache()
            print(f"k={k:2d} round {rep}: training BN {row['bn_training']:8.2f} ms  inference BN "
                  f"{row['bn_inference']:8.2f} ms  torch module {row['torch_module']:8.2f} ms  -> "
                  f"{row['torch_module'] / row['bn_training']:.2f}x over the module, "
                  f"{row['bn_training'] / row['bn_inference'] - 1:+.1%} over inference BN")
            out["steps"].append(row)
    _, eng = engine_step(0, "training", N, S, 2, keep=True)
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = kernel_rows(eng, flush, args.iters)
    print(f"\nnew kernels, batch {N} at {S}x{S}, median of {args.iters} launches each, L2 flushed before each")
    print(f"{'launch':50s} {'us':>9s} {'MB':>8s} {'bound us':>9s} {'of bound':>9s}")
    out["kernels"] = []
    for name, us, nb in rows:
        floor = nb / PEAK_BYTES * 1e6
        print(f"{name:50s} {us:9.1f} {nb / 1e6:8.2f} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"].append({"launch": name, "us": us, "bytes": nb, "bound_us": floor})
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
