"""Per-launch times of the data-gradient convolutions with a fused BatchNorm-backward epilogue, against HBM bandwidth.

    python benchmarks/dgrad_epilogue_times.py [--batch 256] [--iters 25] [--json OUT.json]

These are the ``ConvDgrad`` parts of one ResNet-50 training step whose plan has ``stats_mode`` 2 (conv2 / conv3 data
gradient: the pre-BN tile y is loaded and the bn1 / bn2 backward sums are reduced) or 3 (conv1 data gradient of every
block after the first: the block-gradient merge reads the skip gradient, the ReLU bit mask and the previous block's
y3).  They read several activation-sized operands per output and run few k-blocks per tile, so they are bound by
DRAM bytes, not by the tensor cores.  Each launch is timed alone, as in ``conv_layer_times.py``: the L2 flushed before
each launch, the median of ``--iters`` launches after 5 warm-up launches.  Bytes are the algorithmic bytes from the
layer shapes (``conv_layer_times.dgrad_jobs``), and the bound is those bytes at 3.35 TB/s, the H100 SXM data-sheet
HBM3 bandwidth at 700 W.  The card name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch

from conv_layer_times import PEAK_BYTES, card, dgrad_jobs, time_launch, trained_engine


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dgrad_epilogue_times.py needs a GPU")
    N = args.batch
    eng = trained_engine(N)
    jobs = [j for j in dgrad_jobs(eng, N) if j[2].stats_mode in (2, 3)]

    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = []
    for layer, _, plan, _, nbytes, kb in jobs:
        us = time_launch(plan.run, flush, args.iters)
        floor_us = nbytes / PEAK_BYTES * 1e6
        rows.append(dict(layer=layer, stats_mode=plan.stats_mode, block_n=plan.block_n, kblocks_per_tile=kb,
                         tiles=plan.tiles, grid=plan.grid, us=us, bytes=nbytes, gbps=nbytes / us / 1e3,
                         of_peak=floor_us / us, floor_us=floor_us))

    name = card()
    print(f"card: {name}")
    print(f"batch {N}, {len(rows)} launches with stats_mode 2 or 3, median of {args.iters} launches each, "
          f"L2 flushed before each")
    print(f"{'layer':<22}{'st':>3}{'bn':>5}{'kb/t':>5}{'tiles':>7}{'grid':>5}{'us':>9}{'MB':>8}{'GB/s':>7}{'of 3.35':>8}")
    for r in rows:
        print(f"{r['layer']:<22}{r['stats_mode']:>3}{r['block_n']:>5}{r['kblocks_per_tile']:>5}{r['tiles']:>7}"
              f"{r['grid']:>5}{r['us']:>9.1f}{r['bytes'] / 1e6:>8.1f}{r['gbps']:>7.0f}{r['of_peak']:>8.2f}")
    for mode in (2, 3):
        sel = [r for r in rows if r["stats_mode"] == mode]
        t, f = sum(r["us"] for r in sel), sum(r["floor_us"] for r in sel)
        print(f"stats_mode {mode}: {len(sel)} launches, {t / 1e3:.3f} ms (bytes bound {f / 1e3:.3f} ms, "
              f"{f / t:.2f} of it)")
    tot, floor = sum(r["us"] for r in rows), sum(r["floor_us"] for r in rows)
    print(f"sum over {len(rows)} launches: {tot / 1e3:.3f} ms (bytes bound {floor / 1e3:.3f} ms, {floor / tot:.2f} of it)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=name, batch=N, rows=rows, total_us=tot, floor_us=floor), f, indent=1)


if __name__ == "__main__":
    main()
