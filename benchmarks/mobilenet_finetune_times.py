"""MobileNetV2 fine-tuning on the native engine: training-step time per `fine_tune_at`, and the new backward kernels alone.

    python benchmarks/mobilenet_finetune_times.py [--batch 256] [--size 224] [--steps 20] [--iters 25] [--json OUT.json]

Step time: `MobileNetV2Engine(batch, fine_tune_at=k)` for k in 19 (head only), 14, 8, 0 (whole base), SGD with momentum,
the whole step as one CUDA graph; the mean over ``--steps`` graph replays after 3 warm-up steps, CUDA events around the
window.  Kernel times: on the k = 0 engine after its steps, every launch of the new kernels (csrc/mobilenet_bwd.cu) is
timed alone - CUDA events around one launch, the L2 flushed before each (256 MB memset), the median of ``--iters``
launches - against the least time its bytes need at 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth at 700 W; each
operand read once, each output written once).  The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from b200ddl import optim
from b200ddl.models.mobilenet_engine import MobileNetV2Engine
from b200ddl.models.resnet_engine import EngineTrainStep

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_layer_times import card, time_launch  # noqa: E402

PEAK_BYTES = 3.35e12


def step_time(k, N, S, steps):
    eng = MobileNetV2Engine(batch=N, num_classes=5, image_size=S, fine_tune_at=k)
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
    loss = step.result()[0]
    return eng, s.elapsed_time(e) / steps, loss


def kernel_rows(eng, flush, iters):
    """(name, microseconds, bytes) of every new-kernel launch of one backward of `eng` (fine_tune_at = 0)."""
    e, rows = eng._e, []
    lo = eng._ft_lowest
    for i in range(len(eng._plan) - 1, lo - 1, -1):
        lay = eng._plan[i]
        g, y, x, kind = lay["g"], lay["y"], lay["x"], lay["kind"]
        tag = f"{i:02d} {kind} {lay['conv'][5:]}"
        g2 = lay["g2"]
        nb = g.numel() * 2 * (2 + (g2 is not None) + (lay["act"] == "relu6"))   # g1 [+ g2] [+ y] in, dz out
        rows.append((f"{tag} mask_reduce", time_launch(
            lambda: e.relu6_mask_reduce(g, g2, y, g, lay["sum"], lay["act"] == "relu6"), flush, iters), nb))
        G = eng.g(lay["conv"] + ".weight")
        if kind == "dw":
            rows.append((f"{tag} dw_wgrad s{lay['stride']}", time_launch(
                lambda: e.dw_wgrad(g, x, G, lay["stride"]), flush, iters), (g.numel() + x.numel()) * 2))
            if i > lo:
                dx = eng._plan[i - 1]["g"]
                rows.append((f"{tag} dw_dgrad s{lay['stride']}", time_launch(
                    lambda: e.dw_dgrad(g, lay["w"], lay["scale"], dx, lay["stride"]), flush, iters),
                    (g.numel() + dx.numel()) * 2))
        elif kind == "stem":
            rows.append((f"{tag} stem_wgrad", time_launch(
                lambda: e.mbv2_stem_wgrad(x, g, G, 1.0 / 127.5, -1.0), flush, iters), x.numel() + g.numel()))
    wbytes = sum(eng.spec[s.name].numel * 4 for s in eng.param_specs)
    rows.append(("finalize (all layers)", time_launch(
        lambda: e.mbv2_ft_finalize(eng.params, eng.w16, eng.grads, eng._ft_finalize_table), flush, iters), 3 * wbytes))
    rows.append(("refresh (all layers)", time_launch(
        lambda: e.mbv2_ft_refresh(eng.params, eng._ft_refresh_table), flush, iters), wbytes + wbytes // 2))
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    N, S = args.batch, args.size
    print("card:", card())
    out = {"card": card(), "batch": N, "size": S, "steps": {}, "kernels": []}
    eng = None
    for k in (19, 14, 8, 0):
        del eng
        torch.cuda.empty_cache()
        eng, ms, loss = step_time(k, N, S, args.steps)
        print(f"fine_tune_at={k:2d}: {ms:8.2f} ms/step  ({N / ms * 1e3:8.0f} images/s)  trainable "
              f"{eng.trainable_parameters():,}  loss {loss:.4f}")
        out["steps"][k] = ms
    flush = torch.empty(256 * 1024 * 1024, device="cuda", dtype=torch.uint8)
    rows = kernel_rows(eng, flush, args.iters)
    print(f"\nnew backward kernels, batch {N} at {S}x{S}, median of {args.iters} launches each, L2 flushed before each")
    print(f"{'launch':44s} {'us':>9s} {'MB':>8s} {'bound us':>9s} {'of bound':>9s}")
    total = 0.0
    for name, us, nb in rows:
        floor = nb / PEAK_BYTES * 1e6
        total += us
        print(f"{name:44s} {us:9.1f} {nb / 1e6:8.2f} {floor:9.1f} {floor / us:8.0%}")
        out["kernels"].append({"launch": name, "us": us, "bytes": nb, "bound_us": floor})
    print(f"sum of new-kernel launches: {total / 1e3:.2f} ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
