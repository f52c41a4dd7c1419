"""Host -> device writes of small per-step values that a replayed CUDA graph reads from device memory."""
from __future__ import annotations

from typing import Callable, List, Optional

import torch


class PinnedUpload:
    """Writes ``dst`` (a small device tensor) from a ring of pinned host rows with an async copy on the current stream.

    The host runs several steps ahead of the device, so the row an async copy reads from must not be refilled before
    that copy has executed: each row remembers an event recorded after its copy, and is reused only once that event
    has completed (``depth`` steps later, so in practice it never waits)."""

    def __init__(self, dst: torch.Tensor, depth: int = 64):
        self.dst = dst
        self.ring = torch.zeros(depth, dst.numel(), dtype=dst.dtype).pin_memory()
        self._events: List[Optional[torch.cuda.Event]] = [None] * depth
        self._slot = 0

    def push(self, fill: Callable[[torch.Tensor], None]) -> torch.Tensor:
        """``fill(row)`` writes the values into a free pinned row, which is then copied to ``dst``; returns the row."""
        i = self._slot
        self._slot = (i + 1) % self.ring.shape[0]
        ev = self._events[i]
        if ev is not None:
            ev.synchronize()
        row = self.ring[i]
        fill(row)
        self.dst.copy_(row.view(self.dst.shape), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._events[i] = ev
        return row
