"""Numerics of the fused all-reduce + SGD-momentum + weight-multicast kernel (csrc/allreduce.cu: allreduce_sgd_nvls)
against the unfused sequence it replaces: NCCL all-reduce / N, then a plain PyTorch fp32 SGD-momentum update.

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/fused_update_check.py

Several steps with rank-dependent gradients over a flat buffer that spans several buckets.  Checked after every step:
  * fp32 master weights == reference (relative 2e-6: the kernel sums the N gradients in a different order than NCCL);
  * the bf16 working copy is exactly the round-to-nearest cast of the fp32 master;
  * master and bf16 copy are bit-identical on all ranks (they are written through the multicast mapping);
  * the momentum of the slice THIS rank owns (the optimizer state is sharded 1/N per bucket) == reference.
Exit code 0 = all passed, 1 = a check failed, 0 with "UNAVAILABLE" printed = no multicast mapping on this box.
"""
from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch
import torch.distributed as dist

import b200ddl.parallel as hvd
from b200ddl import optim
from b200ddl.utils import checksum_across_ranks


def main() -> int:
    hvd.init()
    rank, world = hvd.rank(), hvd.size()
    assert world >= 2, "run under torchrun with >= 2 ranks"
    dev = hvd.device()
    lr, mu, wd = 0.05, 0.9, 1e-4
    # "parameters" of uneven sizes (multiples of 1024 elements), ~9.4 M elements -> several 4 MB buckets
    sizes = [1024 * k for k in (3, 640, 1, 2048, 17, 4096, 5, 1300, 999, 64)]
    ranges, lo = [], 0
    for s in sizes:
        ranges.append((lo, lo + s))
        lo += s
    numel = lo
    g0 = torch.Generator(device=dev).manual_seed(7)
    p0 = torch.randn(numel, device=dev, generator=g0)
    dist.broadcast(p0, 0)

    opt = hvd.DistributedOptimizer(optim.SGD(lr, momentum=mu, weight_decay=wd), bucket_mb=4.0, fused_update=True)
    grads = opt.allocate_grads(numel, dev)
    p, w16 = opt.allocate_weights(p0.clone(), p0.to(torch.bfloat16))
    opt.attach(p, ranges, w16)
    if not opt.fused_update:
        if rank == 0:
            print("FUSED UPDATE CHECK UNAVAILABLE: no multicast mapping / unsupported optimizer on this box", flush=True)
        hvd.shutdown()
        return 0
    if rank == 0:
        print(f"world={world} numel={numel} buckets={[(b.lo, b.hi) for b in opt.buckets]}", flush=True)

    p_ref = p0.clone()
    m_ref = torch.zeros_like(p_ref)
    ok_all = True
    gl = torch.Generator(device=dev).manual_seed(1000 + rank)
    for step in range(4):
        g_local = torch.randn(numel, device=dev, generator=gl) * (1.0 + 0.25 * rank)
        # ---- reference: library all-reduce, average, plain fp32 update (same formula as SgdRule in csrc/optim_rules.cuh)
        g_avg = g_local.clone()
        dist.all_reduce(g_avg)
        g_avg /= world
        d = wd * p_ref + g_avg
        m_ref = mu * m_ref + d
        p_ref = p_ref - lr * m_ref
        # ---- fused path: gradients land in the symmetric buffer, buckets fire as their ranges complete
        opt.begin_step()
        opt.start_backward()
        grads.copy_(g_local)
        torch.cuda.synchronize()
        dist.barrier()  # every rank's gradients are in place before any peer reads them
        for a, b in reversed(ranges):  # readiness order of a backward pass: last parameter first
            opt.on_grads_ready(a, b)
        opt.step()
        torch.cuda.synchronize()
        dist.barrier()
        scale = float(p_ref.abs().max())
        err_p = float((p - p_ref).abs().max()) / scale
        cast_exact = bool(torch.equal(w16, p.to(torch.bfloat16)))
        same_p = checksum_across_ranks(p)
        same_w = checksum_across_ranks(w16)
        # momentum: only the slice of each bucket this rank owns is maintained
        mom = opt.opt.state["momentum"]
        err_m = 0.0
        for bk in opt.buckets:
            n = bk.hi - bk.lo
            per = -(-n // world)
            per = (per + 3) // 4 * 4
            a = bk.lo + min(n, rank * per)
            b = bk.lo + min(n, (rank + 1) * per)
            if b > a:
                err_m = max(err_m, float((mom[a:b] - m_ref[a:b]).abs().max()) / float(m_ref.abs().max()))
        good = err_p <= 2e-6 and cast_exact and same_p and same_w and err_m <= 2e-6
        flags = torch.tensor([1.0 if good else 0.0, err_p, err_m], device=dev)
        worst = flags.clone()
        dist.all_reduce(flags, op=dist.ReduceOp.MIN)
        dist.all_reduce(worst, op=dist.ReduceOp.MAX)
        ok_all &= bool(flags[0].item() == 1.0)
        if rank == 0:
            print(f"CHECK fused_update/step{step} err_params={worst[1].item():.3e} err_momentum(own slice)={worst[2].item():.3e} "
                  f"bf16_is_exact_cast={cast_exact} params_identical={same_p} bf16_identical={same_w} "
                  f"{'PASS' if flags[0].item() == 1.0 else 'FAIL'}", flush=True)
    if rank == 0:
        print("FUSED UPDATE CHECK " + ("PASS" if ok_all else "FAIL"), flush=True)
    hvd.shutdown()
    return 0 if ok_all else 1


if __name__ == "__main__":
    sys.exit(main())
