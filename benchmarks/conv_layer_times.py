"""Per-launch times of every implicit-GEMM convolution plan of one ResNet-50 training step, against the roofline.

    python benchmarks/conv_layer_times.py [--batch 256] [--iters 25] [--json OUT.json]

Builds ``ResNet50Engine(batch)`` for training, runs two eager steps (so every buffer holds step-like data), then times
each forward plan, each data-gradient plan (every part of a strided dgrad) and the FC head's two plans ALONE: CUDA
events around one launch, the L2 flushed before each launch (256 MB memset, as ``gpu_check.time_fn``), the median of
``--iters`` launches after 5 warm-up launches.  FLOPs and bytes come from the layer shapes (each operand read once,
the output written once); the roofline floor is max(FLOP / 989e12, bytes / 3.35e12) - the H100 SXM data-sheet dense
BF16 rate and HBM3 bandwidth at 700 W - and the column says which of the two bounds it.  The card name, power limit and
maximum SM clock are read with nvidia-smi in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import optim
from b200ddl.models.resnet_engine import EngineTrainStep, ResNet50Engine, resnet50_blocks
from b200ddl.ops.conv import ConvDgrad

PEAK_FLOPS = 989e12
PEAK_BYTES = 3.35e12


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the table is still useful; say what is missing
        return f"nvidia-smi unavailable ({e})"


def time_launch(fn, flush: torch.Tensor, iters: int, warmup: int = 5) -> float:
    """Median microseconds of one launch, L2 flushed before each."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def conv_shapes(N: int):
    """name -> (R, stride, H_in, H_out, C_in, C_out) of every convolution of the residual blocks."""
    out = {}
    for b in resnet50_blocks():
        n, mid = b.name, b.mid
        out[n + ".conv1"] = (1, 1, b.h_in, b.h_in, b.cin, mid)
        out[n + ".conv2"] = (3, b.stride, b.h_in, b.h_out, mid, mid)
        out[n + ".conv3"] = (1, 1, b.h_out, b.h_out, mid, 4 * mid)
        if b.downsample:
            out[n + ".downsample.0"] = (1, b.stride, b.h_in, b.h_out, b.cin, 4 * mid)
    return out


def dgrad_part_pixels(dg: ConvDgrad, N: int):
    """Output pixels of each part of a dgrad (stride 2: one output-parity class of dx each)."""
    _, H, W, _ = dg.dx.shape
    if dg.stride == 1:
        return [N * H * W]
    px = []
    for ph in range(2):
        for pw in range(2):
            if any((r - dg.pad) % 2 == ph and (s - dg.pad) % 2 == pw for r in range(dg.R) for s in range(dg.S)):
                px.append(N * len(range(ph, H, 2)) * len(range(pw, W, 2)))
    return px


def trained_engine(N: int) -> ResNet50Engine:
    """A training ``ResNet50Engine(batch=N)`` after two eager steps, so every buffer holds step-like data."""
    eng = ResNet50Engine(batch=N, num_classes=1000, seed=0)
    step = EngineTrainStep(eng, optim.SGD(0.1, momentum=0.9), use_graph=False)
    g = torch.Generator(device="cuda").manual_seed(0)
    step.load(torch.randint(0, 256, (N, 224, 224, 3), device="cuda", dtype=torch.uint8, generator=g),
              torch.randint(0, 1000, (N,), device="cuda", generator=g))
    for _ in range(2):
        step.run()
    torch.cuda.synchronize()
    return eng


def dgrad_jobs(eng: ResNet50Engine, N: int):
    """(layer, kind, plan, flops, bytes, k-blocks per tile) of every data-gradient launch of the residual blocks."""
    shapes = conv_shapes(N)
    blocks = {b.name: b for b in resnet50_blocks()}
    jobs = []
    for name, dg in eng._dg.items():
        R, s, hi, ho, ci, co = shapes[name]
        dy_elems = N * ho * ho * co
        for (plan, _, idx), px in zip(dg.parts, dgrad_part_pixels(dg, N)):
            flops = 2.0 * px * ci * co * len(idx)
            nbytes = 2.0 * (dy_elems + len(idx) * ci * co + px * ci)
            if plan.stats_mode == 2:
                nbytes += 2.0 * px * ci                      # pre-BN tile y
            elif plan.stats_mode == 3:
                b = blocks[name.rsplit(".", 1)[0]]
                skip_px = px // 4 if b.stride == 2 else px   # compact skip gradient of a strided projection
                nbytes += 2.0 * skip_px * ci + px * ci / 8 + 2.0 * px * ci  # skip gradient, ReLU bit mask, y3
            kind = "dgrad" if len(dg.parts) == 1 else f"dgrad[{len(idx)}taps]"
            jobs.append((name, kind, plan, flops, nbytes, len(idx) * (-(-co // 64))))
    return jobs


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this path")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "conv_layer_times.py needs a GPU"
    N = args.batch
    eng = trained_engine(N)
    shapes = conv_shapes(N)
    jobs = []  # (layer, kind, plan, flops, bytes, k-blocks per tile)
    for name, op in eng._fwd.items():
        R, s, hi, ho, ci, co = shapes[name]
        a_px = N * ho * ho if (R == 1 and s > 1) else N * hi * hi  # a strided 1x1 conv reads only its sampled pixels
        flops = 2.0 * N * ho * ho * co * ci * R * R
        nbytes = 2.0 * (a_px * ci + R * R * co * ci + N * ho * ho * co)
        jobs.append((name, "fwd", op.plan, flops, nbytes, R * R * (-(-ci // 64))))
    jobs += dgrad_jobs(eng, N)
    ncp = eng.classes_padded
    jobs.append(("fc", "fwd", eng._fc_fwd.plan, 2.0 * N * 2048 * ncp, 2.0 * (N * 2048 + ncp * 2048 + N * ncp), 2048 // 64))
    for plan, _, _ in eng._fc_dg.parts:
        jobs.append(("fc", "dgrad", plan, 2.0 * N * 2048 * ncp, 2.0 * (N * ncp + ncp * 2048 + N * 2048), -(-ncp // 64)))

    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = []
    for layer, kind, plan, flops, nbytes, kb in jobs:
        us = time_launch(plan.run, flush, args.iters)
        t_f, t_b = flops / PEAK_FLOPS * 1e6, nbytes / PEAK_BYTES * 1e6
        rows.append(dict(layer=layer, kind=kind, block_n=plan.block_n, stats_mode=plan.stats_mode,
                         resident_filter=bool(plan.resident_filter), halo=bool(plan.halo), tiles=plan.tiles,
                         grid=plan.grid, kblocks_per_tile=kb, us=us, tflops=flops / us / 1e6, gbps=nbytes / us / 1e3,
                         floor_us=max(t_f, t_b), bound="compute" if t_f >= t_b else "memory", flops=flops, bytes=nbytes))

    print(f"card: {card()}")
    print(f"batch {N}, {len(rows)} launches, median of {args.iters} launches each, L2 flushed before each")
    hdr = (f"{'layer':<22}{'kind':<14}{'bn':>4}{'st':>3}{'res':>4}{'halo':>5}{'tiles':>7}{'grid':>5}{'kb/t':>5}"
           f"{'us':>9}{'TFLOP/s':>9}{'GB/s':>7}{'floor':>8}{'bound':>8}{'x floor':>8}")
    print(hdr)
    for r in rows:
        print(f"{r['layer']:<22}{r['kind']:<14}{r['block_n']:>4}{r['stats_mode']:>3}{int(r['resident_filter']):>4}"
              f"{int(r['halo']):>5}{r['tiles']:>7}{r['grid']:>5}{r['kblocks_per_tile']:>5}{r['us']:>9.1f}"
              f"{r['tflops']:>9.1f}{r['gbps']:>7.0f}{r['floor_us']:>8.1f}{r['bound']:>8}{r['us'] / r['floor_us']:>8.2f}")
    tot, floor = sum(r["us"] for r in rows), sum(r["floor_us"] for r in rows)
    short = [r for r in rows if r["kblocks_per_tile"] <= 8]
    print(f"sum over all {len(rows)} launches: {tot / 1e3:.3f} ms (roofline floor {floor / 1e3:.3f} ms); "
          f"{len(short)} launches with <= 8 k-blocks per tile: {sum(r['us'] for r in short) / 1e3:.3f} ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), batch=N, rows=rows, total_us=tot), f, indent=1)


if __name__ == "__main__":
    main()
