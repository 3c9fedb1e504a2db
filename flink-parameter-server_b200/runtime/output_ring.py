"""E5: the per-update worker output stream of the device tier (``ps.output((user, userVector))`` after
every update, PSOnlineMatrixFactorizationWorker.scala:52), batched and flushed by a DEVICE-side
count / timer policy (K11; CountLogic.scala:5-29, TimerLogic.scala:6-51).

The fused kernel writes ``(id, vector)`` records into a device staging area; after each micro-batch
``native.output_step`` runs the policy kernel and, when it fires, the flush kernel that copies the staged
records into a ring in pinned host memory and publishes the new tail with a system-scope release store.
``poll()`` reads whatever has been published -- a plain host memory read, no stream synchronisation --
and hands back ``(ids, vectors)``; ``records()`` yields ``Left((id, vector))`` like the host tier.
``every=n`` samples one update in ``n`` (the full stream, one row per update at benchmark rates, is far
more than the host link carries)."""
from __future__ import annotations

from typing import Iterator, List, Optional, Tuple

import numpy as np
import torch

from ..api import Left
from ..ops import native


class OutputRing:
    def __init__(self, dim: int, device: torch.device, ring_capacity: int = 1 << 16,
                 staging_capacity: int = 1 << 16, every: int = 1, flush_count: int = 1,
                 flush_interval_ms: Optional[float] = None, require: str = "any"):
        self.dim, self.stride = int(dim), (int(dim) + 3) // 4 * 4
        self.device = torch.device(device)
        self.every = max(1, int(every))
        self.count_max = max(0, int(flush_count))
        self.interval_ns = 0 if flush_interval_ms is None else int(float(flush_interval_ms) * 1e6)
        self.require_all = require == "all"
        self.s_ids = torch.full((staging_capacity,), -1, dtype=torch.int64, device=self.device)
        self.s_vecs = torch.zeros((staging_capacity, self.stride), dtype=torch.float32, device=self.device)
        self.state = torch.zeros(native.OUT_STATE_WORDS, dtype=torch.int64, device=self.device)
        self.ring_ids = torch.zeros(ring_capacity, dtype=torch.int64).pin_memory()
        self.ring_vecs = torch.zeros((ring_capacity, self.stride), dtype=torch.float32).pin_memory()
        self.host_tail = torch.zeros(1, dtype=torch.int64).pin_memory()
        self.host_head = torch.zeros(1, dtype=torch.int64).pin_memory()
        self._tail_np = self.host_tail.numpy()          # volatile view: the device writes it
        self._head = 0

    # ---- producer side -------------------------------------------------------------------------------
    def kernel_args(self) -> Tuple:
        """``output=`` argument of ``native.mf_sgd_fused``."""
        return (self.s_ids, self.s_vecs, self.state[0:1], self.s_ids.numel(), self.every)

    def emitted(self, n_records: int) -> int:
        return -(-int(n_records) // self.every)

    def after_kernel(self, n_records: int, force: bool = False) -> None:
        """Run the device-side policy (+ flush) for the records the kernel just staged."""
        native.output_step(self.state, self.s_ids, self.s_vecs, self.ring_ids, self.ring_vecs, self.host_tail,
                           self.host_head, n_new=self.emitted(n_records), count_max=self.count_max,
                           interval_ns=self.interval_ns, require_all=self.require_all, force=force)

    def flush(self) -> None:
        self.after_kernel(0, force=True)

    # ---- consumer side (host, no CUDA calls) ---------------------------------------------------------------
    def poll(self) -> Tuple[np.ndarray, np.ndarray]:
        tail = int(self._tail_np[0])
        n = tail - self._head
        if n <= 0:
            return np.empty(0, dtype=np.int64), np.empty((0, self.dim), dtype=np.float32)
        cap = self.ring_ids.numel()
        idx = (self._head + np.arange(n)) % cap
        ids = self.ring_ids.numpy()[idx].copy()
        vecs = self.ring_vecs.numpy()[idx, : self.dim].copy()
        keep = ids >= 0                                  # holes left by voided records
        if not keep.all():
            ids, vecs = ids[keep], vecs[keep]
        self._head = tail
        self.host_head[0] = tail                        # frees the slots for the device
        return ids, vecs

    def records(self) -> Iterator[Left]:
        ids, vecs = self.poll()
        for i, v in zip(ids.tolist(), vecs):
            yield Left((i, v.astype(np.float64)))

    def counters(self) -> dict:
        st = self.state.cpu().tolist()
        return {"staged": st[0], "published": st[1], "flushes": st[5], "dropped": st[6]}
