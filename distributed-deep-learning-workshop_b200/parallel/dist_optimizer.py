"""DistributedOptimizer: synchronous data parallelism with the gradient all-reduce fused and overlapped.

Reference: `hvd.DistributedOptimizer(optimizer)` (P1/03:302, P2/02:189) - Horovod enqueues every gradient, fuses
ready tensors into a fusion buffer (memcpy in), calls ncclAllReduce, scales by 1/N (separate kernel) and copies
out (SURVEY.md §3.3).  Here the gradients are *born* inside one flat symmetric buffer (the wgrad kernels write
there), so there is no copy in/out; when a bucket of that buffer is complete the hook launches ONE kernel on a
high-priority communication stream that reduces the bucket across GPUs over NVLink (NVLS multimem or P2P), applies
1/N (x loss-scale^-1) and writes the result back to every rank, while backward continues on the compute stream.

Modes (``algo``):  'auto' | 'nvls' | 'p2p' | 'oneshot'  - our kernels;   'nccl' - the baseline path
(`dist.all_reduce` + separate divide), kept selectable for A/B measurements;  'gloo' is implied on CPU.
"""
from __future__ import annotations

import contextlib
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

from . import core
from ..optim.fused import FlatOptimizer


class _Bucket:
    __slots__ = ("lo", "hi", "pending", "total")

    def __init__(self, lo: int, hi: int):
        self.lo, self.hi = lo, hi
        self.total = hi - lo
        self.pending = self.total


class DistributedOptimizer:
    """Wraps a fused flat optimizer; averages gradients over all ranks before every update."""

    def __init__(self, optimizer: FlatOptimizer, bucket_mb: float = 16.0, overlap: bool = True, algo: str = "auto",
                 comm_blocks: int = 32, average: bool = True, fused_update: bool = False, tail_mb: float = 1.0,
                 nvls_min_mb: Optional[float] = None, nvls_blocks: Optional[int] = None):
        self.opt = optimizer
        self.bucket_bytes = int(bucket_mb * 2 ** 20)
        # The LAST bucket to complete is the only all-reduce nothing can hide (backward has ended): keep it small.  The
        # final `tail_mb` of the gradient buffer (the layers that finish last: stem + first stage) become their own bucket.
        self.tail_bytes = int(tail_mb * 2 ** 20)
        # 'auto' picks the kernel PER BUCKET: with 2 ranks the P2P two-shot always, with more ranks the in-switch NVLS
        # reduction from 1 MB up (it needs few CTAs, so NVLS buckets use `nvls_blocks`).  `benchmarks/allreduce_check.py`
        # sweeps both against NCCL to check the crossover on a given box.
        if nvls_min_mb is None:
            nvls_min_mb = 1e9 if core.size() <= 2 else 1.0
        self.nvls_min_bytes = int(nvls_min_mb * 2 ** 20)
        # each rank only reduces 1/world of the bucket, so the more ranks the fewer CTAs saturate the switch's reduction path
        self.nvls_blocks = nvls_blocks if nvls_blocks is not None else 16
        self.overlap = overlap
        self.algo = algo
        # CTAs of a comm kernel (512 threads each); they occupy SM slots only while a bucket is in flight
        self.comm_blocks = comm_blocks
        self.average = average
        # fused_update: reduce-scatter + SGD-momentum update of my 1/N slice + multicast of the new fp32/bf16 weights
        # in ONE kernel per bucket (csrc/allreduce.cu: allreduce_sgd_nvls); optimizer state is sharded over ranks.
        self.fused_update = fused_update
        self._wsym = None
        self._w16sym = None
        self._wcomm = None
        self.world = core.size()
        self.rank = core.rank()
        self.buckets: List[_Bucket] = []
        self.grads: Optional[torch.Tensor] = None
        self._comm = None
        self._sym = None
        self._comm_stream = None
        self._oneshot_tmp = None
        self._launched = 0
        self.allreduce_launches = 0
        self.timeline = None  # utils.Timeline: per-bucket all-reduce spans on the comm stream
        self.extra_wait_streams = []  # streams that also produce gradients (e.g. the engine's wgrad side stream)

    # -- forwarded optimizer surface -------------------------------------------------------------------------
    @property
    def learning_rate(self) -> float:
        return self.opt.learning_rate

    @learning_rate.setter
    def learning_rate(self, v: float) -> None:
        self.opt.learning_rate = v

    lr = learning_rate

    def __getattr__(self, item):
        if item in ("opt",):
            raise AttributeError(item)
        return getattr(self.opt, item)

    # -- setup ----------------------------------------------------------------------------------------------
    def allocate_grads(self, numel: int, device: torch.device) -> torch.Tensor:
        """Flat fp32 gradient buffer: symmetric (peer-mapped, multicast) memory when running on >1 GPU."""
        use_sym = (self.world > 1 and device.type == "cuda" and self.algo not in ("nccl", "gloo"))
        if use_sym:
            from . import symm

            self._sym = symm.SymmetricBuffer(numel, torch.float32, device)
            self._comm = symm.make_comm(self._sym)
            self.grads = self._sym.tensor
            if self.algo == "auto":
                self.algo = "auto-sym" if self._sym.has_multicast else "p2p"
            if self.algo == "nvls" and not self._sym.has_multicast:
                raise RuntimeError("algo='nvls' requested but the symmetric buffer has no multicast mapping")
        else:
            self.grads = torch.zeros(numel, device=device, dtype=torch.float32)
            if self.world > 1 and self.algo == "auto":
                self.algo = "nccl" if device.type == "cuda" else "gloo"
        if device.type == "cuda" and self.world > 1:
            self._comm_stream = torch.cuda.Stream(device=device, priority=-1)
        return self.grads

    def allocate_weights(self, params: torch.Tensor, w16: Optional[torch.Tensor]):
        """fused_update only: move the fp32 master (and bf16 copy) into symmetric + multicast memory.  Returns the
        (params, w16) tensors the model must use from now on, or the inputs unchanged when fusion is unavailable."""
        # the per-bucket kernel sees one bucket at a time, so it cannot apply a clip that needs the whole gradient; it
        # updates every step and has no accumulation or EMA pass
        ok = (self.fused_update and self.world > 1 and params.is_cuda and self._sym is not None
              and self._sym.has_multicast and getattr(self.opt, "name", "") == "SGD" and not self.opt.nesterov
              and getattr(self.opt, "clip_mode", None) is None
              and getattr(self.opt, "gradient_accumulation_steps", None) is None
              and not getattr(self.opt, "use_ema", False))
        if not ok:
            self.fused_update = False
            return params, w16
        from . import symm

        self._wsym = symm.SymmetricBuffer(params.numel(), torch.float32, params.device)
        self._wsym.tensor.copy_(params)
        self._wcomm = symm.make_comm(self._wsym)
        new_w16 = w16
        if w16 is not None:
            self._w16sym = symm.SymmetricBuffer(w16.numel(), torch.bfloat16, w16.device)
            self._w16sym.tensor.copy_(w16)
            new_w16 = self._w16sym.tensor
        return self._wsym.tensor, new_w16

    def attach(self, params: torch.Tensor, spec_ranges: List[Tuple[int, int]], w16: Optional[torch.Tensor] = None,
               grads: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Bind flat params; build buckets from the per-parameter [lo, hi) ranges (in readiness order)."""
        if grads is None:
            grads = self.grads if self.grads is not None else self.allocate_grads(params.numel(), params.device)
        self.grads = grads
        self.opt.attach(params, grads, w16, segments=spec_ranges)
        self.buckets = []
        elem_budget = max(1, self.bucket_bytes // 4)
        lo = None
        hi = 0
        for a, b in spec_ranges:
            if lo is None:
                lo = a
            hi = b
            if hi - lo >= elem_budget:
                self.buckets.append(_Bucket(lo, hi))
                lo = None
        if lo is not None:
            self.buckets.append(_Bucket(lo, hi))
        # split a small tail off the last bucket (ranges are in readiness order, so the tail completes last)
        tail_elems = self.tail_bytes // 4
        if tail_elems > 0 and self.buckets and spec_ranges:
            last = self.buckets[-1]
            cut = last.hi
            for a, b in reversed(spec_ranges):
                if a < last.lo or last.hi - a > tail_elems:
                    break
                cut = a
            if last.lo < cut < last.hi:
                self.buckets[-1] = _Bucket(last.lo, cut)
                self.buckets.append(_Bucket(cut, last.hi))
        return grads

    # -- hot path ------------------------------------------------------------------------------------------
    def begin_step(self) -> None:
        self.opt.begin_step()
        if self.fused_update:
            self._state_complete = False   # called once per step even when the step itself is a CUDA-graph replay

    def start_backward(self) -> None:
        for b in self.buckets:
            b.pending = b.total
        self._launched = 0

    def on_grads_ready(self, lo: int, hi: int) -> None:
        """Engine / autograd hook: gradient elements [lo, hi) of the flat buffer are final."""
        if self.world == 1:
            return
        for i, b in enumerate(self.buckets):
            if hi <= b.lo or lo >= b.hi:
                continue
            b.pending -= min(hi, b.hi) - max(lo, b.lo)
            if b.pending <= 0 and self.overlap:
                self._reduce_bucket(b)

    def _reduce_bucket(self, b: _Bucket) -> None:
        n = b.hi - b.lo
        if self._comm_stream is not None:
            for st in self.extra_wait_streams:
                self._comm_stream.wait_stream(st)
        scale = (1.0 / self.world) if self.average else 1.0
        if self.fused_update:
            cs = self._comm_stream
            cs.wait_stream(torch.cuda.current_stream())
            span = (self.timeline.device_span(f"allreduce+sgd[{b.lo}:{b.hi}]", "comm", stream=cs)
                    if self.timeline is not None else contextlib.nullcontext())
            with torch.cuda.stream(cs), span:
                self._comm.allreduce_sgd(self._wcomm, b.lo, n, self.opt.state["momentum"],
                                         self._w16sym.mc_ptr if self._w16sym is not None else 0, scale,
                                         self.opt._hyper, self.comm_blocks)
        elif self.algo in ("nvls", "p2p", "oneshot", "auto-sym"):
            cs = self._comm_stream
            cs.wait_stream(torch.cuda.current_stream())
            algo = self.algo
            if algo == "auto-sym":
                algo = "nvls" if n * 4 >= self.nvls_min_bytes else "p2p"
            span = (self.timeline.device_span(f"allreduce[{b.lo}:{b.hi}] {algo}", "comm", stream=cs)
                    if self.timeline is not None else contextlib.nullcontext())
            with torch.cuda.stream(cs), span:
                if algo == "nvls":
                    self._comm.twoshot_nvls(b.lo, n, "f32", scale, self.nvls_blocks if self.algo == "auto-sym" else self.comm_blocks)
                elif algo == "p2p":
                    self._comm.twoshot_p2p(b.lo, n, "f32", scale, self.comm_blocks)
                else:
                    # one-shot reads every peer's slice and has no barrier between its load and store phases, so it
                    # must NOT write into the symmetric source buffer: reduce into a private tensor, copy back after
                    # the kernel's end barrier (same stream)
                    if self._oneshot_tmp is None or self._oneshot_tmp.numel() < n:
                        self._oneshot_tmp = torch.empty(max(n, max(bb.total for bb in self.buckets)),
                                                        device=self.grads.device, dtype=torch.float32)
                    tmp = self._oneshot_tmp[:n]
                    self._comm.oneshot(b.lo, n, "f32", tmp, scale, self.comm_blocks)
                    self.grads[b.lo:b.hi].copy_(tmp)
        elif self.algo == "nccl":
            # baseline: library collective + separate elementwise kernel (what Horovod does)
            cs = self._comm_stream
            cs.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(cs):
                view = self.grads[b.lo:b.hi]
                dist.all_reduce(view)
                if self.average:
                    view.div_(self.world)
        else:  # gloo / CPU
            view = self.grads[b.lo:b.hi]
            dist.all_reduce(view)
            if self.average:
                view.div_(self.world)
        self.allreduce_launches += 1
        self._launched += 1

    def finish_backward(self) -> None:
        """Reduce whatever has not been launched yet and make the compute stream wait for the comm stream."""
        if self.world == 1:
            return
        if not self.overlap or self._launched < len(self.buckets):
            for b in self.buckets:
                if b.pending > 0 or not self.overlap:
                    self._reduce_bucket(b)
                    b.pending = 0
        if self._comm_stream is not None:
            torch.cuda.current_stream().wait_stream(self._comm_stream)

    @property
    def is_update_step(self) -> bool:
        return self.opt.is_update_step

    def step(self, update: Optional[bool] = None) -> None:
        """Every micro-batch is all-reduced (the sum is linear, so accumulating reduced gradients is exact); ``update``
        as in `FlatOptimizer.step`."""
        self.finish_backward()
        if not self.fused_update:
            self.opt.step(update)  # fused_update: the per-bucket kernels already updated and broadcast the weights
        else:
            self._state_complete = False   # momentum now differs per rank outside the owned slices

    @property
    def state_is_sharded(self) -> bool:
        """True when this rank's optimizer state is only valid on its own slices (fused_update after a step and before
        `consolidate_state()`): `Trainer.save` refuses to write such a state."""
        return bool(self.fused_update and self.world > 1 and not getattr(self, "_state_complete", True))

    # -- utilities -----------------------------------------------------------------------------------------
    @staticmethod
    def owned_range(lo: int, hi: int, rank: int, world: int):
        """Elements [a, b) of bucket [lo, hi) whose optimizer state rank `rank` owns under fused_update - the slicing of
        csrc/allreduce.cu allreduce_sgd_nvls_kernel (float4 vectors split evenly, the last rank takes the short end)."""
        nvec = (hi - lo) // 4
        per = -(-nvec // world)
        v0 = min(per * rank, nvec)
        v1 = min(v0 + per, nvec)
        return lo + 4 * v0, lo + 4 * v1

    def consolidate_state(self) -> None:
        """COLLECTIVE (every rank must call it).  With fused_update each rank holds the momentum of only its 1/N slice of
        every bucket; this makes every rank's state tensors complete (sum of the owners' slices), so that a checkpoint
        written by rank 0 can be resumed on any world size and `broadcast_parameters` does not overwrite live slices
        with rank 0's stale ones.  No-op without fused_update."""
        if not self.state_is_sharded or not self.buckets:
            # no fused step has run since the state was last complete (fresh optimizer, just-loaded checkpoint, ...)
            self._state_complete = True
            return
        for name, v in self.opt.state.items():
            if not torch.is_tensor(v) or v.numel() != self.grads.numel():
                continue   # scalars (step counters) are replicated already
            full = torch.zeros_like(v)
            for b in self.buckets:
                a, e = self.owned_range(b.lo, b.hi, self.rank, self.world)
                if e > a:
                    full[a:e] = v[a:e]
            v.copy_(core.allreduce(full, average=False))
        self._state_complete = True

    def broadcast_parameters(self, params: torch.Tensor, root: int = 0) -> None:
        self.consolidate_state()
        core.broadcast(params, root)
        for v in self.opt.state.values():
            core.broadcast(v, root)
