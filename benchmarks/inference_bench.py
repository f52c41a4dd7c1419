"""Batch-inference throughput (BASELINE.json config 4): the trained ResNet-50's forward (BN folded to running
statistics, same wgmma conv kernels, CUDA graph) over synthetic images sharded across GPUs.

    python benchmarks/inference_bench.py --images 100000                       # one GPU
    torchrun --nproc-per-node 8 ... benchmarks/inference_bench.py --images 1000000

Every batch is copied from pinned host memory (ring loader) and its predictions (argmax) are read back to the host,
so the number is end to end.  Rank r scores shard r; the reported images/s is the aggregate, max time over ranks.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import b200ddl.parallel as hvd
from b200ddl.loader import SyntheticDataset
from b200ddl.models.resnet_engine import EngineEvalStep, ResNet50Engine


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=100000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--classes", type=int, default=5)
    args = ap.parse_args()
    hvd.init()
    rank, world = hvd.rank(), hvd.size()
    dev = hvd.device()
    eng = ResNet50Engine(batch=args.batch, num_classes=args.classes, device=dev)
    eng.build(training=False)
    ev = EngineEvalStep(eng, use_graph=True)
    steps = max(1, args.images // (args.batch * world))
    preds = torch.zeros(args.batch, dtype=torch.int64).pin_memory()
    with SyntheticDataset(args.batch, num_classes=args.classes, device=dev, cur_shard=rank, shard_count=world,
                          threads=6, pool_images=4096) as ds:
        for _ in range(5):
            x, y = next(ds)
            eng.set_input(x, y)
            ev.run()
        torch.cuda.synchronize()
        hvd.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            x, y = next(ds)
            eng.set_input(x, y)
            ev.run()
            preds.copy_(eng.logits.argmax(1), non_blocking=True)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    t = torch.tensor([dt], device=dev)
    if world > 1:
        import torch.distributed as dist

        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        n = steps * args.batch * world
        print(json.dumps({"metric": "resnet50_batch_inference_images_per_sec", "value": n / float(t.item()),
                          "images": n, "n_gpus": world, "batch": args.batch, "seconds": float(t.item()),
                          "h2d_bytes_per_step": args.batch * (224 * 224 * 3 + 8), "d2h_bytes_per_step": args.batch * 8}))
    hvd.shutdown()


if __name__ == "__main__":
    main()
