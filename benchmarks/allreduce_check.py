"""Fused all-reduce kernels: correctness vs NCCL and the 1 KB - 1 GB bandwidth sweep (BASELINE.json config 5).

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/allreduce_check.py [--quick] [--max-mb 1024]

For every size / dtype / algorithm (one-shot P2P, two-shot P2P, two-shot NVLS multimem):
  * numerics: result == (sum over ranks) / N computed by NCCL (fp32 tolerance 1e-5 rel, bf16 2e-2), and bit-identical
    on all ranks;
  * timing: CUDA events on the launching stream, warm-up, max over ranks; the NCCL baseline is
    `dist.all_reduce` + a separate `div_` kernel (what Horovod's DistributedOptimizer does).
Reported: algorithm bandwidth S/t, bus bandwidth S/t * 2(N-1)/N, and the fraction of the NVLink roofline
(450 GB/s per direction nominal on H100 NVLink 4).
"""
from __future__ import annotations

import tempfile

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch
import torch.distributed as dist

import b200ddl.parallel as hvd
from b200ddl.parallel import symm
from b200ddl.utils import checksum_across_ranks


def time_op(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item()) * 1e-3  # seconds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--medium", action="store_true", help="1 KB, 64 KB, 1 MB, 16 MB, 128 MB, 1 GB")
    ap.add_argument("--max-mb", type=float, default=1024.0)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "allreduce_check"))
    ap.add_argument("--f32-only", action="store_true", help="sweep the fp32 payload only (the gradient dtype)")
    ap.add_argument("--skip-extras", action="store_true", help="no broadcast / CTA sweep / DistributedOptimizer sections")
    args = ap.parse_args()
    hvd.init()
    rank, world = hvd.rank(), hvd.size()
    assert world >= 2, "run under torchrun with >= 2 ranks"
    dev = hvd.device()
    max_bytes = int(args.max_mb * 2 ** 20)
    buf = symm.SymmetricBuffer(max_bytes // 4, torch.float32, dev)
    comm = symm.make_comm(buf)
    if rank == 0:
        print(f"world={world} multicast={'yes' if buf.has_multicast else 'no'} buffer={max_bytes / 2**20:.0f} MiB", flush=True)
    if args.quick:
        sizes = [4096, 1 << 20, 32 << 20]
    elif args.medium:
        sizes = [s for s in (1 << 10, 1 << 16, 1 << 20, 1 << 24, 1 << 27, 1 << 30) if s <= max_bytes]
    else:
        sizes = [1 << k for k in range(10, 31, 2) if (1 << k) <= max_bytes]  # 1 KB .. 1 GB, x4
    ok_all = True
    rows = []
    g = torch.Generator(device=dev).manual_seed(1000 + rank)
    for dtype, name, esz in (((torch.float32, "f32", 4),) if args.f32_only else ((torch.float32, "f32", 4), (torch.bfloat16, "bf16", 2))):
        view = buf.tensor.view(dtype)
        for nbytes in sizes:
            n = nbytes // esz
            src = (torch.randn(n, device=dev, generator=g) * (rank + 1)).to(dtype)
            ref = src.clone().float()
            dist.all_reduce(ref)
            ref /= world
            algos = []
            if nbytes <= (4 << 20):
                algos.append("oneshot")
            algos.append("p2p")
            if buf.has_multicast:
                algos.append("nvls")
            blocks = 4 if nbytes <= (256 << 10) else (16 if nbytes <= (4 << 20) else (32 if nbytes <= (32 << 20) else 64))
            tol = 1e-5 if dtype == torch.float32 else 2.5e-2
            res = {"dtype": name, "bytes": nbytes, "world": world}
            for algo in algos:
                out = torch.empty(n, device=dev, dtype=dtype) if algo == "oneshot" else None

                def run():
                    if algo == "oneshot":
                        comm.oneshot(0, n, name, out, 1.0 / world, blocks)
                    elif algo == "p2p":
                        comm.twoshot_p2p(0, n, name, 1.0 / world, blocks)
                    else:
                        comm.twoshot_nvls(0, n, name, 1.0 / world, blocks)

                view[:n].copy_(src)
                torch.cuda.synchronize()
                dist.barrier()
                run()
                torch.cuda.synchronize()
                dist.barrier()
                got = (out if algo == "oneshot" else view[:n]).float()
                err = float((got - ref).abs().max() / (ref.abs().max() + 1e-12))
                same = checksum_across_ranks(out if algo == "oneshot" else view[:n])
                good = err <= tol and same
                ok_all &= good
                iters = 50 if nbytes <= (1 << 20) else (20 if nbytes <= (64 << 20) else 8)
                t = time_op(run, iters)
                res[algo] = {"err": err, "identical": same, "us": t * 1e6, "algbw_GBs": nbytes / t / 1e9,
                             "busbw_GBs": nbytes / t / 1e9 * 2 * (world - 1) / world}
                if rank == 0 and not good:
                    print(f"FAIL {name} {nbytes}B {algo}: err={err:.3e} identical={same}", flush=True)
            # NCCL baseline path: library all-reduce + separate scale kernel
            t_nccl = torch.empty(n, device=dev, dtype=dtype).copy_(src)

            def run_nccl():
                dist.all_reduce(t_nccl)
                t_nccl.div_(world)

            iters = 50 if nbytes <= (1 << 20) else (20 if nbytes <= (64 << 20) else 8)
            t = time_op(run_nccl, iters)
            res["nccl+div"] = {"us": t * 1e6, "algbw_GBs": nbytes / t / 1e9,
                               "busbw_GBs": nbytes / t / 1e9 * 2 * (world - 1) / world}
            # roofline: bytes that must cross NVLink per direction per GPU / link bandwidth
            two_shot = 2.0 * nbytes * (world - 1) / world
            nvls = nbytes * (1.0 + 1.0 / world)
            best = min((v["us"] for k, v in res.items() if isinstance(v, dict) and k != "nccl+div"), default=None)
            res["roofline_us_450"] = {"two_shot": two_shot / 450e9 * 1e6, "nvls": nvls / 450e9 * 1e6}
            if best:
                res["best_fraction_of_roofline_450"] = min(two_shot, nvls) / 450e9 * 1e6 / best
                res["speedup_vs_nccl"] = res["nccl+div"]["us"] / best
            rows.append(res)
            if rank == 0:
                parts = " ".join(f"{k}={v['us']:.1f}us/{v['busbw_GBs']:.0f}GB/s" for k, v in res.items()
                                 if isinstance(v, dict) and "us" in v)
                print(f"{name} {nbytes:>11d} B  {parts}  best/roofline450={res.get('best_fraction_of_roofline_450', 0):.2f} "
                      f"vs_nccl={res.get('speedup_vs_nccl', 0):.2f}x", flush=True)
    # ---- broadcast kernel (K2): hvd.broadcast on CUDA tensors runs csrc/allreduce.cu broadcast_kernel through a symmetric
    # staging buffer; compare with the value the root holds, for every root, several dtypes / sizes (incl. > 1 staging chunk)
    bc_sizes = [(torch.float32, 300_000), (torch.bfloat16, 1_000_001), (torch.int64, 4097)]
    if not args.quick:
        bc_sizes.append((torch.float32, 20_000_000))  # 80 MB > the 64 MB staging buffer
    for root in range(min(world, 3)):
        for dt, n in bc_sizes:
            gen = torch.Generator(device=dev).manual_seed(7 + rank * 31 + n)
            mine = (torch.randn(n, device=dev, generator=gen) * 100).to(dt)
            want = mine.clone()
            dist.broadcast(want, root)          # library result
            got = mine.clone()
            hvd.broadcast(got, root)            # our kernel
            torch.cuda.synchronize()
            same = bool(torch.equal(got, want))
            ok_all &= same
            if rank == 0:
                print(f"broadcast root={root} {str(dt).split('.')[-1]} n={n}: {'ok' if same else 'FAIL'}", flush=True)
    big = torch.randn(64 << 20, device=dev) if not args.quick else torch.randn(4 << 20, device=dev)
    t_k = time_op(lambda: hvd.broadcast(big, 0), 5, warmup=2)
    t_n = time_op(lambda: dist.broadcast(big, 0), 5, warmup=2)
    if rank == 0:
        print(f"broadcast {big.numel() * 4 / 2**20:.0f} MiB: kernel (staged) {t_k * 1e3:.2f} ms  NCCL {t_n * 1e3:.2f} ms", flush=True)
    # ---- CTA-count sweep at the gradient-bucket size (what DistributedOptimizer.comm_blocks should be)
    nb = min(16 << 20, max_bytes)
    view32 = buf.tensor.view(torch.float32)
    blk = {}
    for blocks in (8, 16, 32, 64):
        for algo in (("p2p", "nvls") if buf.has_multicast else ("p2p",)):
            fn = (lambda: comm.twoshot_p2p(0, nb // 4, "f32", 1.0 / world, blocks)) if algo == "p2p" else \
                 (lambda: comm.twoshot_nvls(0, nb // 4, "f32", 1.0 / world, blocks))
            blk[f"{algo}_{blocks}"] = time_op(fn, 20) * 1e6
    if rank == 0:
        print("bucket-size (16 MB f32) CTA sweep, us: " + " ".join(f"{k}={v:.1f}" for k, v in blk.items()), flush=True)
    rows.append({"cta_sweep_16MB_f32_us": blk, "world": world})
    # ---- DistributedOptimizer end to end on every algorithm (incl. one-shot writing back into the symmetric buffer)
    from b200ddl import optim
    for algo in ("auto", "p2p", "oneshot") + (("nvls",) if buf.has_multicast else ()):
        nparam = 3_000_000
        params = torch.zeros(nparam, device=dev)
        opt = hvd.DistributedOptimizer(optim.SGD(0.1), bucket_mb=4.0, algo=algo)
        grads = opt.allocate_grads(nparam, dev)
        ranges = [(i, min(i + 250_000, nparam)) for i in range(0, nparam, 250_000)]
        opt.attach(params, ranges, None, grads)
        gen = torch.Generator(device=dev).manual_seed(99 + rank)
        local = torch.randn(nparam, device=dev, generator=gen) * (rank + 1)
        ref = local.clone()
        dist.all_reduce(ref)
        ref /= world
        grads.copy_(local)
        torch.cuda.synchronize()
        dist.barrier()
        opt.start_backward()
        for a, b in ranges:
            opt.on_grads_ready(a, b)
        opt.finish_backward()
        torch.cuda.synchronize()
        err = float((grads - ref).abs().max() / ref.abs().max())
        same = checksum_across_ranks(grads)
        good = err <= 1e-5 and same
        ok_all &= good
        if rank == 0:
            print(f"DistributedOptimizer algo={algo} ({opt.algo}) buckets={len(opt.buckets)} tail={opt.buckets[-1].total}: "
                  f"err={err:.2e} identical={same} {'ok' if good else 'FAIL'}", flush=True)
    if rank == 0:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"allreduce_sweep_w{world}.json"), "w") as f:
            json.dump(rows, f, indent=1)
        print("ALLREDUCE CHECK " + ("PASS" if ok_all else "FAIL"), flush=True)
    hvd.shutdown()
    sys.exit(0 if ok_all else 1)


if __name__ == "__main__":
    main()
