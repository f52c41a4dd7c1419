"""Sharded image loader (SURVEY.md L2/C12): the Petastorm `make_spark_converter` surface on a pinned ring buffer.

Reference usage (P1/03:137-144, 204-219, 332-348, 425-426)::

    converter = make_spark_converter(df)                      ->  conv = make_converter(table, cache_dir)
    len(converter)                                            ->  len(conv)
    with converter.make_tf_dataset(batch_size, cur_shard=rank, shard_count=size) as ds:
                                                              ->  with conv.make_dataset(batch_size, cur_shard, shard_count) as ds:
    converter.delete()                                        ->  conv.delete()

`make_dataset` yields ``(images uint8 [B,H,W,3], labels int64 [B])`` forever (`num_epochs=None`, the reference's
dead-lock avoidance for unequal shards, P1/03:199).  On a GPU the yielded tensors are views of a small device-side
staging ring (two buffers for the pinned-ring datasets, three for `decode='gpu'`): a batch is valid until the next-but-one
`next()`; `Trainer.fit / evaluate` consume it immediately, anything that keeps batches around must `.clone()` them.  Rows are read from the parquet cache by `workers_count` decode
threads (PIL releases the GIL), written straight into pinned host slots of the native `RingLoader`
(csrc/ring_loader.cpp) and moved to the GPU with cudaMemcpyAsync on a side stream, double-buffered on the device.
`SyntheticDataset` feeds the same ring from native gather threads (JPEG-shaped uint8 tensors; no network here).
"""
from __future__ import annotations

import os
import shutil
import threading
import uuid
from typing import Iterator, Optional, Tuple

import numpy as np
import torch

from ..models.preprocess import IMG_HEIGHT, IMG_WIDTH, decode_image
from ..utils.cpus import usable_cpus


def _device_index(device) -> int:
    if device is None:
        return torch.cuda.current_device() if torch.cuda.is_available() else -1
    d = torch.device(device)
    if d.type != "cuda":
        return -1
    return d.index if d.index is not None else torch.cuda.current_device()


class RingDataset:
    """Iterable over a native RingLoader; context-manager like Petastorm's dataset."""

    def __init__(self, batch_size: int, image_size: Tuple[int, int], device=None, num_slots: int = 6):
        from .. import ops

        self.batch_size = batch_size
        self.h, self.w = image_size
        self.dev_index = _device_index(device)
        ext = ops.ext("_b200_loader")
        self.ring = ext.RingLoader(num_slots, batch_size, self.h * self.w * 3, self.dev_index, 2)
        self._closed = False

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        return self

    def __next__(self):
        img, lab = self.ring.next()
        return img.view(self.batch_size, self.h, self.w, 3), lab

    def close(self) -> None:
        if not self._closed:
            self._closed = True
            self.ring.close()

    @property
    def h2d_bytes_per_batch(self) -> int:
        return self.batch_size * (self.h * self.w * 3 + 8)


class SyntheticDataset(RingDataset):
    """JPEG-shaped synthetic images assembled by native gather threads from a pool of pre-generated images."""

    def __init__(self, batch_size: int, num_classes: int = 1000, image_size=(IMG_HEIGHT, IMG_WIDTH), device=None,
                 cur_shard: int = 0, shard_count: int = 1, threads: int = 4, pool_images: int = 2048, seed: int = 0,
                 num_slots: int = 6):
        super().__init__(batch_size, image_size, device, num_slots)
        self.ring.start_synthetic(threads, pool_images, num_classes, seed, cur_shard, shard_count)


class _TableDataset(RingDataset):
    """Rows of one shard of the parquet cache -> decoded uint8 batches in the pinned ring.

    Sharding: shard s owns the contiguous global row range [n*s/k, n*(s+1)/k) and opens ONLY the row groups that
    intersect it (no read amplification: k ranks together read the cache once, not k times).  `shuffle=True` permutes
    the shard's row groups and the rows inside every group with `seed + epoch` (Petastorm shuffles row groups too).
    Row groups stay Arrow arrays (no `to_pylist`); the short critical section only hands out (array, index) pairs, the
    decode (PIL releases the GIL) runs outside it in `workers_count` threads."""

    def __init__(self, files, total_rows, batch_size, image_size, device, cur_shard, shard_count, num_epochs,
                 workers_count, shuffle, seed, decode_processes: int = 0):
        nproc = int(decode_processes or 0)
        self._chunk = 16 if batch_size >= 64 else max(1, batch_size // 4)   # images per decode request
        chunks_per_batch = -(-batch_size // self._chunk)
        # process mode: enough slots that every decode process can hold a chunk of SOME slot while others are being consumed
        slots = max(4, workers_count + 2) if nproc <= 0 else max(6, -(-nproc // chunks_per_batch) + 4)
        super().__init__(batch_size, image_size, device, num_slots=slots)
        self.files = files
        self.total_rows = int(total_rows)
        self.cur_shard, self.shard_count = cur_shard, shard_count
        self.num_epochs = num_epochs
        self.shuffle, self.seed = shuffle, seed
        n, k = self.total_rows, shard_count
        self.row_lo, self.row_hi = (n * cur_shard) // k, (n * (cur_shard + 1)) // k
        self.row_groups_read = 0   # statistics: how many row groups this shard has opened
        self._stop = threading.Event()
        self._lock = threading.Lock()
        self._row_iter = self._rows()
        self._active_workers = max(1, workers_count)
        self._error: Optional[BaseException] = None
        # decode PROCESSES (loader/_decode_worker.py).  `workers_count` PLANNER threads cut batches into chunks of
        # `self._chunk` rows and queue them; ONE light driver thread per process takes a chunk, ships the compressed bytes and
        # receives the decoded pixels straight into the chunk's rows of the pinned slot (`recv_bytes_into`; the socket reads
        # release the GIL).  A slot is committed by whichever driver finishes its last chunk.
        self._pools = None
        if nproc > 0:
            import queue

            from ..utils.procpool import start_script_workers

            script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_decode_worker.py")
            self._pools = start_script_workers(script, nproc, env={"OMP_NUM_THREADS": "1"})
            self._work = queue.Queue(maxsize=4 * nproc)
            self._plan_lock = threading.Lock()
            self._pending = {}               # slot -> chunks still being decoded
            self._seq_next = 0               # batches are numbered in the order they are cut from the row stream ...
            self._seq_commit = 0             # ... and committed in that order (reorder buffer): the batch sequence is
            self._seq_done = {}              # deterministic for a given seed, however the decode processes race
            self._slot_seq = {}
            self._planners_left = min(max(1, workers_count), 4)
            self._drivers_left = nproc
            self._threads = [threading.Thread(target=self._planner, daemon=True) for _ in range(self._planners_left)]
            self._threads += [threading.Thread(target=self._driver, args=(k,), daemon=True) for k in range(nproc)]
        else:
            self._threads = [threading.Thread(target=self._worker, daemon=True) for _ in range(max(1, workers_count))]
        self.decode_processes = nproc
        for t in self._threads:
            t.start()

    def __len__(self) -> int:
        """Full batches per epoch of THIS shard, so that `fit(ds)` / `steps_per_epoch=len(ds)` work like they do for a
        Keras dataset."""
        return (self.row_hi - self.row_lo) // self.batch_size

    def _plan(self):
        """[(file index, row group, first row inside the group, row count)] of this shard, in file order."""
        import pyarrow.parquet as pq

        plan = []
        for fi, (path, base) in enumerate(self.files):
            md = pq.ParquetFile(path).metadata
            g0 = base
            for rg in range(md.num_row_groups):
                nr = md.row_group(rg).num_rows
                lo, hi = max(self.row_lo, g0), min(self.row_hi, g0 + nr)
                if hi > lo:
                    plan.append((fi, rg, lo - g0, hi - lo))
                g0 += nr
        return plan

    def _rows(self):
        """Infinite (or `num_epochs`) stream of (content array, label array, row index) of THIS shard."""
        import pyarrow.parquet as pq

        plan = self._plan()
        handles = {}
        epoch = 0
        while (self.num_epochs is None or epoch < self.num_epochs) and plan:
            order = list(range(len(plan)))
            rng = np.random.default_rng(self.seed + epoch) if self.shuffle else None
            if rng is not None:
                rng.shuffle(order)
            for pi in order:
                fi, rg, skip, count = plan[pi]
                if fi not in handles:
                    handles[fi] = pq.ParquetFile(self.files[fi][0])
                t = handles[fi].read_row_group(rg, columns=["content", "label_idx"])
                self.row_groups_read += 1
                contents = t.column("content").combine_chunks()
                labels = t.column("label_idx").to_numpy()
                idx = np.arange(skip, skip + count)
                if rng is not None:
                    rng.shuffle(idx)
                for j in idx:
                    yield contents, labels, int(j)
            epoch += 1

    def _fail(self, ex: BaseException) -> None:
        """A dead decode process, a corrupt row ...: end the stream; `__next__` re-raises once the committed batches are drained."""
        if not self._stop.is_set():
            self._error = ex
            self._stop.set()
            self.ring.finish()

    def _worker(self):
        try:
            self._produce()
        except BaseException as ex:
            self._fail(ex)
        finally:
            # the LAST worker to run out of rows ends the stream: the consumer drains what is committed and then gets
            # StopIteration (without this a `for batch in ds:` over a finite dataset blocked forever)
            with self._lock:
                self._active_workers -= 1
                last = self._active_workers == 0
            if last and not self._stop.is_set():
                self.ring.finish()

    def _produce(self):
        while not self._stop.is_set():
            batch = self._take_batch()
            if len(batch) < self.batch_size:
                return  # finite epochs exhausted (drop the tail batch, like steps_per_epoch = n // batch)
            slot = self.ring.acquire_fill()
            if slot < 0:
                return
            img, lab = self.ring.slot_tensors(slot)
            img = img.numpy().reshape(self.batch_size, self.h, self.w, 3)
            lab = lab.numpy()
            for i, (contents, labels, j) in enumerate(batch):
                img[i] = decode_image(contents[j].as_py(), (self.h, self.w))
                lab[i] = labels[j]
            self.ring.commit(slot)

    def _take_batch(self):
        with self._lock:
            batch = []
            try:
                for _ in range(self.batch_size):
                    batch.append(next(self._row_iter))
            except StopIteration:
                pass
        return batch

    def _planner(self):
        """Process mode: batch -> slot -> chunks on the work queue."""
        import queue

        try:
            while not self._stop.is_set():
                # slot first, then the batch and its sequence number in one critical section: slots are acquired in
                # sequence order too, so the oldest uncommitted batch always owns a slot (no reorder-buffer deadlock)
                slot = self.ring.acquire_fill()
                if slot < 0:
                    break
                with self._plan_lock:
                    batch = self._take_batch()
                    seq = self._seq_next
                    if len(batch) == self.batch_size:
                        self._seq_next += 1
                if len(batch) < self.batch_size:
                    break
                img, lab = self.ring.slot_tensors(slot)
                dst = memoryview(img.numpy().reshape(-1))
                lab = lab.numpy()
                for i, (_, labels, j) in enumerate(batch):
                    lab[i] = labels[j]
                chunks = [(slot, dst, first, batch[first:first + self._chunk]) for first in range(0, self.batch_size, self._chunk)]
                with self._lock:
                    self._pending[slot] = len(chunks)
                    self._slot_seq[slot] = seq
                for item in chunks:
                    while not self._stop.is_set():
                        try:
                            self._work.put(item, timeout=0.5)
                            break
                        except queue.Full:
                            continue
        except BaseException as ex:
            self._fail(ex)
        finally:
            with self._lock:
                self._planners_left -= 1
                last = self._planners_left == 0
            if last:   # every chunk is queued: one sentinel per driver, behind the last real item
                for _ in range(self.decode_processes):
                    while True:
                        try:
                            self._work.put(None, timeout=0.5)
                            break
                        except queue.Full:
                            if self._stop.is_set():
                                break

    def _driver(self, k: int):
        """Process mode: the thread that talks to decode process k."""
        import queue

        conn = self._pools[k][1]
        row = self.h * self.w * 3
        try:
            while not self._stop.is_set():
                try:
                    item = self._work.get(timeout=0.5)
                except queue.Empty:
                    continue
                if item is None:
                    break
                slot, dst, first, rows = item
                payloads = [contents[j].as_buffer() for contents, _, j in rows]
                head = np.array([self.h, self.w, len(rows)] + [len(b) for b in payloads], dtype=np.int32).tobytes()
                conn.send_bytes(b"".join([head] + [memoryview(b) for b in payloads]))
                got = conn.recv_bytes_into(dst[first * row:(first + len(rows)) * row])   # pixels land in the pinned slot
                if got != len(rows) * row:
                    raise RuntimeError(f"decode worker {k} returned {got} bytes for {len(rows)} images")
                with self._lock:
                    self._pending[slot] -= 1
                    if self._pending[slot] == 0:
                        del self._pending[slot]
                        self._seq_done[self._slot_seq.pop(slot)] = slot
                        while self._seq_commit in self._seq_done:      # commit in sequence order
                            self.ring.commit(self._seq_done.pop(self._seq_commit))
                            self._seq_commit += 1
        except BaseException as ex:
            self._fail(ex)
        finally:
            with self._lock:
                self._drivers_left -= 1
                last = self._drivers_left == 0
            if last and not self._stop.is_set():
                self.ring.finish()   # finite epochs: everything decoded has been committed

    def __next__(self):
        try:
            return super().__next__()
        except StopIteration:
            if self._error is not None:
                raise RuntimeError(f"the loader's decode pipeline failed: {self._error!r}") from self._error
            raise

    def close(self) -> None:
        self._stop.set()
        super().close()
        if self._pools:
            # the driver threads own the connections: let them finish the chunk in flight before the exit frames are sent
            # (two writers on one socket would interleave their frames)
            for t in self._threads:
                if t is not threading.current_thread():
                    t.join(timeout=20)
            for proc, conn in self._pools:
                try:
                    conn.send_bytes(b"")
                    conn.close()
                except Exception:
                    pass
            for proc, _ in self._pools:
                try:
                    proc.wait(timeout=5)
                except Exception:
                    proc.kill()
            self._pools = None


class _GpuDecodeDataset:
    """`make_dataset(decode='gpu')`: only the COMPRESSED bytes cross PCIe; the JPEG payloads are decoded on the GPU and resized
    by our kernel straight into the uint8 device batch (the reference's tf.io.decode_jpeg + resize, P1/03:182-189).

    Native path (`csrc/jpeg_decode.cpp`, extension `_b200_jpeg`): nvJPEG (library) batched decode - HARDWARE backend (the
    NVJPG engines: no SM time, no CPU Huffman decode) when the GPU has it, else GPU-hybrid - into one scratch buffer, then ONE
    launch of our batched anti-aliased resize kernel (`csrc/jpeg_resize.cu`, PIL's BILINEAR filter).  Batch k+1 is decoded on a
    side stream while the model trains on batch k (three device buffers, event-chained both ways; no host synchronisation).
    Fallbacks: `torchvision.io.decode_jpeg(device=cuda)` + `resize_bilinear_u8` when the native decoder cannot be created
    (`B200DDL_JPEG_BACKEND=torchvision` forces it; `=hardware|gpu_hybrid|hybrid` pins a backend); rows that are not JPEG
    (PNG, raw tensors) take the CPU decoder.  Same sharding / shuffle / epoch semantics as the pinned-ring dataset (it reuses
    its row planner); yields (images uint8 [B,H,W,3], labels int64 [B]).  The yielded tensors are views of a 3-deep device
    ring: a batch stays valid until the SECOND `next()` after it (consume it - `fit` copies it into the engine's input right
    away - or `.clone()` it)."""

    _BUFFERS = 3

    def __init__(self, files, total_rows, batch_size, image_size, device, cur_shard, shard_count, num_epochs, shuffle, seed):
        import types

        from .. import ops

        self.batch_size = batch_size
        self.h, self.w = image_size
        self.device = torch.device("cuda", _device_index(device))
        self._e = ops.ext("_b200_ops")
        # borrow the row planner of the ring dataset without starting its decode threads
        self._src = types.SimpleNamespace(files=files, total_rows=int(total_rows), cur_shard=cur_shard, shard_count=shard_count,
                                          num_epochs=num_epochs, shuffle=shuffle, seed=seed, row_groups_read=0,
                                          batch_size=batch_size)
        n, k = int(total_rows), shard_count
        self._src.row_lo, self._src.row_hi = (n * cur_shard) // k, (n * (cur_shard + 1)) // k
        self._src._plan = lambda: _TableDataset._plan(self._src)
        self._rows = _TableDataset._rows(self._src)
        R = self._BUFFERS
        self._out = [torch.empty(batch_size, self.h, self.w, 3, device=self.device, dtype=torch.uint8) for _ in range(R)]
        self._lab = [torch.empty(batch_size, device=self.device, dtype=torch.int64) for _ in range(R)]
        self._lab_host = [torch.empty(batch_size, dtype=torch.int64).pin_memory() for _ in range(R)]
        self._done = [None] * R          # event on the decode stream: buffer r holds a finished batch
        self._keep = [None] * R          # the Arrow buffers whose addresses nvJPEG was given (alive until the buffer is reused)
        self._stream = torch.cuda.Stream(device=self.device)
        self._entry_events = []          # events recorded on the consumer's stream at the entry of __next__ (oldest first)
        self._k = 0                      # batches handed out
        self._issued = 0                 # batches whose decode has been enqueued
        self._exhausted = False
        self.compressed_bytes = 0
        self.gpu_decoded = 0
        self.cpu_decoded = 0
        self.backend = "torchvision"
        self.backend_errors = []
        self._dec = None
        want = os.environ.get("B200DDL_JPEG_BACKEND", "")
        if want != "torchvision":
            try:
                jpeg = ops.ext("_b200_jpeg")
                for name in ([want] if want else ["hardware", "gpu_hybrid"]):
                    try:
                        self._dec = jpeg.JpegDecoder(batch_size, name, 4, self.device.index)
                        self.backend = "nvjpeg:" + name
                        break
                    except Exception as ex:   # ARCH_MISMATCH: no hardware engine on this GPU, ...
                        self.backend_errors.append(f"{name}: {str(ex).splitlines()[0][:160]}")
            except Exception as ex:
                self.backend_errors.append(f"_b200_jpeg: {str(ex).splitlines()[0][:160]}")

    def __len__(self) -> int:
        return (self._src.row_hi - self._src.row_lo) // self.batch_size

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def close(self) -> None:
        self._rows = iter(())
        self._exhausted = True
        torch.cuda.synchronize(self.device)   # nothing may still read the bitstreams / write the buffers we drop
        self._keep = [None] * self._BUFFERS

    def __iter__(self):
        return self

    def _take(self):
        batch = []
        try:
            for _ in range(self.batch_size):
                batch.append(next(self._rows))
        except StopIteration:
            pass
        return batch if len(batch) == self.batch_size else None

    def _issue(self, wait_event) -> bool:
        """Enqueue the decode of the next batch into buffer `issued % R` on the decode stream.  `wait_event`: consumer-stream
        event after which that buffer is no longer read."""
        import warnings

        batch = self._take()
        if batch is None:
            self._exhausted = True
            return False
        r = self._issued % self._BUFFERS
        out, lab, lab_host = self._out[r], self._lab[r], self._lab_host[r]
        ptrs, lens, keep, jpeg_idx, other = [], [], [], [], []
        for i, (contents, lbls, j) in enumerate(batch):
            buf = contents[j].as_buffer()
            lab_host[i] = int(lbls[j])
            if buf.size >= 3 and bytes(buf[:3]) == b"\xff\xd8\xff":
                ptrs.append(buf.address)
                lens.append(buf.size)
                keep.append(buf)
                jpeg_idx.append(i)
                self.compressed_bytes += buf.size
            else:
                other.append((i, contents[j].as_py()))
        st = self._stream
        if wait_event is not None:
            st.wait_event(wait_event)
        with torch.cuda.stream(st):
            if jpeg_idx:
                contiguous = jpeg_idx == list(range(len(jpeg_idx)))
                if self._dec is not None:
                    try:
                        if contiguous and len(jpeg_idx) == self.batch_size:
                            self._dec.decode_resize(ptrs, lens, out)
                        else:   # mixed batch: decode the JPEG rows into a temporary and scatter them
                            tmp = torch.empty(len(jpeg_idx), self.h, self.w, 3, device=self.device, dtype=torch.uint8)
                            self._dec.decode_resize(ptrs, lens, tmp)
                            out[torch.tensor(jpeg_idx, device=self.device)] = tmp
                    except RuntimeError as ex:
                        # e.g. a progressive JPEG the hardware engine does not take: this and all later batches go the library way
                        self.backend_errors.append(f"{self.backend}: {str(ex).splitlines()[0][:160]}")
                        self._dec, self.backend = None, "torchvision"
                if self._dec is None:
                    import torchvision

                    with warnings.catch_warnings():
                        warnings.simplefilter("ignore")  # read-only buffers: decode_jpeg does not write to them
                        data = [torch.from_numpy(np.frombuffer(b, dtype=np.uint8)) for b in keep]
                    imgs = torchvision.io.decode_jpeg(data, device=self.device, mode=torchvision.io.ImageReadMode.RGB)
                    for i, img in zip(jpeg_idx, imgs):
                        self._e.resize_bilinear_u8(img.unsqueeze(0), out[i:i + 1], True)  # [1,3,h,w] planar -> [1,H,W,3]
                self.gpu_decoded += len(jpeg_idx)
            for i, payload in other:
                out[i].copy_(torch.from_numpy(np.ascontiguousarray(decode_image(payload, (self.h, self.w)))))
                self.cpu_decoded += 1
            lab.copy_(lab_host, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(st)
        self._done[r] = ev
        self._keep[r] = keep
        self._issued += 1
        return True

    def __next__(self):
        cur = torch.cuda.current_stream(self.device)
        entry = torch.cuda.Event()
        entry.record(cur)            # everything the consumer enqueued so far (incl. its reads of the batch handed out last)
        self._entry_events.append(entry)
        if len(self._entry_events) > 2:
            self._entry_events.pop(0)
        if self._issued == self._k and not self._exhausted:
            self._issue(None)        # first call: nothing has been prefetched yet
        if self._issued == self._k:
            raise StopIteration
        # prefetch the batch after this one: it overwrites the buffer handed out two calls ago, whose reads the consumer
        # enqueued before the PREVIOUS call's entry event
        if not self._exhausted and self._issued - self._k < 2:
            self._issue(self._entry_events[0] if len(self._entry_events) == 2 else None)
        r = self._k % self._BUFFERS
        cur.wait_event(self._done[r])
        self._k += 1
        return self._out[r], self._lab[r]


class Converter:
    """Materialised, shardable copy of a table (Petastorm `SparkDatasetConverter`)."""

    def __init__(self, table, cache_dir: str, rows_per_group: int = 256):
        import pyarrow.parquet as pq

        self.cache_dir = os.path.join(cache_dir, "converter_" + uuid.uuid4().hex[:12])
        os.makedirs(self.cache_dir, exist_ok=True)
        cols = [c for c in ("content", "label_idx") if c in table.columns]
        if cols != ["content", "label_idx"]:
            raise ValueError("converter needs columns ['content', 'label_idx'] (reference P1/03:102-103)")
        arrow = table.select(cols).to_arrow()
        self._n = arrow.num_rows
        path = os.path.join(self.cache_dir, "part-00000.parquet")
        pq.write_table(arrow, path, compression="none", row_group_size=rows_per_group)
        self.files = [(path, 0)]

    def __len__(self) -> int:
        return self._n

    def make_dataset(self, batch_size: int = 32, cur_shard: Optional[int] = None, shard_count: Optional[int] = None,
                     num_epochs: Optional[int] = None, workers_count: int = 4, image_size=(IMG_HEIGHT, IMG_WIDTH),
                     device=None, shuffle: bool = False, seed: int = 0, decode: str = "cpu", decode_processes=None):
        """``decode='cpu'``: PIL decode + resize into the pinned ring - in `workers_count` threads (default), or, with
        ``decode_processes=N`` (or ``'auto'``: 1.5 x the USABLE cpus - cgroup quota - divided by the ranks of this node; the default
        on a GPU for datasets of >= 4096 rows; 0 = threads only), in N decode PROCESSES driven by those threads (threads of one process stop scaling at ~4.6 k images/s, see _decode_worker.py);
        ``decode='gpu'``: nvJPEG decode + our resize kernel on the device (`_GpuDecodeDataset`)."""
        if (cur_shard is None) != (shard_count is None):
            raise ValueError("cur_shard and shard_count must be given together")
        cs, sc = (0, 1) if cur_shard is None else (int(cur_shard), int(shard_count))
        if not (0 <= cs < sc):
            raise ValueError("need 0 <= cur_shard < shard_count")
        if decode == "gpu":
            return _GpuDecodeDataset(self.files, self._n, batch_size, image_size, device, cs, sc, num_epochs, shuffle, seed)
        if decode != "cpu":
            raise ValueError("decode must be 'cpu' or 'gpu'")
        if decode_processes is None:
            # default: processes when a GPU consumes a dataset big enough to amortise starting them
            on_gpu = _device_index(device) >= 0
            decode_processes = "auto" if (on_gpu and self._n >= 4096) else 0
        if decode_processes == "auto":
            # 1.5 processes per USABLE cpu (cgroup quota, not cpu_count) shared by the ranks of this node: the pool is never
            # 100 % busy (chunks arrive in bursts), mild oversubscription measured best (16-CPU quota: 8 procs 3.6 k, 48: 6.2 k
            # images/s, 32 bare processes 6.5 k, 120: 4.2 k)
            lws = max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1")))
            decode_processes = min(96, int(1.5 * usable_cpus() / lws + 0.5))
            if decode_processes < 3:
                decode_processes = 0   # not worth the processes: decode threads
        return _TableDataset(self.files, self._n, batch_size, image_size, device, cs, sc, num_epochs, workers_count,
                             shuffle, seed, decode_processes=int(decode_processes or 0))

    # reference spelling
    make_tf_dataset = make_dataset
    make_torch_dataset = make_dataset

    def delete(self) -> None:
        shutil.rmtree(self.cache_dir, ignore_errors=True)


class InMemoryDataset:
    """`toPandas()` + `from_tensor_slices((content, label_idx)).map(preprocess).batch(B)` (reference P1/02:97-139,
    P2/01:137-151): the whole table is decoded once into driver memory; finite, re-iterable, `len()` = batches.
    ``weight_column``: batches are ``(images, labels, sample_weight float32 [B])`` with the weights read from that column
    (Keras's ``(x, y, sample_weight)`` datasets)."""

    def __init__(self, table_or_pdf, batch_size: int, image_size=(IMG_HEIGHT, IMG_WIDTH), drop_last: bool = True,
                 weight_column: Optional[str] = None):
        pdf = table_or_pdf.to_pandas() if hasattr(table_or_pdf, "to_pandas") else table_or_pdf
        self.images = torch.from_numpy(np.stack([decode_image(c, image_size) for c in pdf["content"]]))
        self.labels = torch.from_numpy(pdf["label_idx"].to_numpy(dtype=np.int64))
        self.weights = None
        if weight_column is not None:
            if weight_column not in pdf.columns:
                raise ValueError(f"weight_column {weight_column!r} is not a column of the table")
            self.weights = torch.from_numpy(pdf[weight_column].to_numpy(dtype=np.float32))
        self.batch_size = max(1, min(batch_size, len(self.labels)))
        n = len(self.labels)
        self.n = n // self.batch_size * self.batch_size if drop_last else n

    def __len__(self) -> int:
        return max(1, -(-self.n // self.batch_size))

    def __iter__(self):
        for i in range(0, self.n, self.batch_size):
            if self.weights is None:
                yield self.images[i:i + self.batch_size], self.labels[i:i + self.batch_size]
            else:
                yield (self.images[i:i + self.batch_size], self.labels[i:i + self.batch_size],
                       self.weights[i:i + self.batch_size])


def make_converter(table, cache_dir: Optional[str] = None) -> Converter:
    """`make_spark_converter(df)` (reference P1/03:140-141)."""
    if cache_dir is None:
        cache_dir = os.path.join(os.environ.get("TMPDIR", "/tmp"), "b200ddl_converter_cache")
    return Converter(table, cache_dir)


make_spark_converter = make_converter

__all__ = ["make_converter", "make_spark_converter", "Converter", "SyntheticDataset", "RingDataset", "InMemoryDataset"]
