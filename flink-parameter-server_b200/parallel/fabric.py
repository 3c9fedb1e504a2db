"""Symmetric-heap fabric over NVLink/NVSwitch.

Each PS rank owns one device allocation; all ranks map all allocations, so a kernel running on
any GPU can address any shard by pointer.  This is the GPU-native replacement of the
reference's ``partitionCustom`` + Flink network stack (FPS:416-420, 455-463) and of its
iteration feedback edge (FPS:477-480): a pull is a peer load, a push is a peer reduction.

Bootstrap uses ``torch.distributed`` (NCCL or gloo) only to exchange 64-byte CUDA IPC handles.
A fallback to ``torch.distributed._symmetric_memory`` (CUDA VMM + fd passing) is used when
legacy CUDA IPC is refused by the container.
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch
import torch.distributed as dist

from ..ops import native


def _dist_ready() -> bool:
    return dist.is_available() and dist.is_initialized()


class SymmetricHeap:
    """A same-size device allocation on every rank of ``group`` with all peers mapped."""

    def __init__(self, nbytes: int, group=None, device: Optional[int] = None,
                 mode: Optional[str] = None):
        self.nbytes = int((nbytes + 255) // 256 * 256)
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.group = group
        self.world = dist.get_world_size(group) if _dist_ready() else 1
        self.rank = dist.get_rank(group) if _dist_ready() else 0
        self.mode = mode or os.environ.get("FPS_FABRIC", "ipc")
        self._opened: List[int] = []
        self._symm_keepalive = None
        self._owned = False
        self.peer_ptrs: List[int] = []
        with torch.cuda.device(self.device):
            if self.world == 1:
                self.local_ptr = native.heap_alloc(self.nbytes)
                self._owned = True
                self.peer_ptrs = [self.local_ptr]
            elif self.mode == "symm":
                self._init_symm()
            else:
                try:
                    self._init_ipc()
                except RuntimeError as e:  # container refuses legacy IPC -> VMM path
                    if os.environ.get("FPS_FABRIC") == "ipc":
                        raise
                    self._cleanup_ipc()
                    self.mode = "symm"
                    self._init_symm()

    # -- CUDA IPC -------------------------------------------------------------------------
    def _init_ipc(self) -> None:
        self.local_ptr = native.heap_alloc(self.nbytes)
        self._owned = True
        handle = native.ipc_get_handle(self.local_ptr)
        handles: List[Optional[bytes]] = [None] * self.world
        dist.all_gather_object(handles, handle, group=self.group)
        ok = 1
        ptrs = []
        err = None
        for r, h in enumerate(handles):
            if r == self.rank:
                ptrs.append(self.local_ptr)
                continue
            try:
                p = native.ipc_open_handle(h)
                self._opened.append(p)
                ptrs.append(p)
            except RuntimeError as e:
                ok = 0
                err = e
                break
        flags = [None] * self.world
        dist.all_gather_object(flags, ok, group=self.group)
        if not all(flags):
            raise RuntimeError(f"CUDA IPC mapping failed on some rank: {err}")
        self.peer_ptrs = ptrs

    def _cleanup_ipc(self) -> None:
        for p in self._opened:
            try:
                native.ipc_close(p)
            except RuntimeError:
                pass
        self._opened = []
        if self._owned:
            try:
                native.heap_free(self.local_ptr)
            except RuntimeError:
                pass
            self._owned = False

    # -- torch symmetric memory (CUDA VMM) ------------------------------------------------
    def _init_symm(self) -> None:
        import torch.distributed._symmetric_memory as symm

        grp = self.group if self.group is not None else dist.group.WORLD
        t = symm.empty(self.nbytes, dtype=torch.uint8, device=torch.device("cuda", self.device))
        hdl = symm.rendezvous(t, grp)
        t.zero_()
        self._symm_keepalive = (t, hdl)
        self.peer_ptrs = [int(p) for p in hdl.buffer_ptrs]
        self.local_ptr = self.peer_ptrs[self.rank]
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)

    # -- views ----------------------------------------------------------------------------
    def local_tensor(self, shape, dtype: torch.dtype = torch.float32, offset: int = 0) -> torch.Tensor:
        return native.tensor_from_ptr(self.local_ptr + offset, shape, dtype, self.device)

    def peer_tensor(self, rank: int, shape, dtype: torch.dtype = torch.float32,
                    offset: int = 0) -> torch.Tensor:
        """Zero-copy view of a *peer's* allocation (loads/stores go over NVLink)."""
        return native.tensor_from_ptr(self.peer_ptrs[rank] + offset, shape, dtype, self.device)

    def barrier(self) -> None:
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)

    def close(self) -> None:
        if self.world > 1:
            try:
                self.barrier()
            except Exception:
                pass
        self._cleanup_ipc()
        self._symm_keepalive = None

    def __del__(self):  # best effort
        try:
            self._cleanup_ipc()
        except Exception:
            pass


class P2PGather:
    """One-sided gather of small per-rank tensors (partial top-K lists, E9 of SURVEY §2.11;
    reference: the parallelism-1 merge sinks, CollectTopKFromEachWorker.scala:41-56) -- no NCCL.

    Every rank owns ``world`` receive slots (x 2, alternating by call) in a symmetric heap.  A sender
    stores its tensor straight into the destination's slot ``[rank]`` through the peer mapping (a copy
    kernel whose destination is NVLink peer memory) and then stores the call's sequence number into the
    destination's flag ``[rank]``; the destination polls its own flags, reads its slots and stores an
    acknowledgement back, which is what lets a sender reuse a slot two calls later.
    """

    def __init__(self, max_bytes: int, group=None, device: Optional[int] = None):
        self.slot = int((max_bytes + 255) // 256 * 256)
        self.group = group
        self.world = dist.get_world_size(group) if _dist_ready() else 1
        self.rank = dist.get_rank(group) if _dist_ready() else 0
        w = self.world
        self._flags_off = 2 * w * self.slot
        self._acks_off = self._flags_off + 256 * ((8 * w + 255) // 256)
        total = self._acks_off + 256 * ((8 * w + 255) // 256)
        self.heap = SymmetricHeap(total, group=group, device=device)
        self.device = self.heap.device
        self.seq = 0
        self._last_use = [[0, 0] for _ in range(w)]   # per destination and buffer: the call that used it last
        self.flags = self.heap.local_tensor((w,), torch.int64, self._flags_off)
        self.acks = self.heap.local_tensor((w,), torch.int64, self._acks_off)
        self.heap.barrier()

    def _wait(self, t: torch.Tensor, idx, value: int, what: str, timeout_s: float = 60.0) -> None:
        import time

        t0 = time.time()
        while True:
            cur = t if idx is None else t[idx]
            if int(cur.min().item()) >= value:
                return
            if time.time() - t0 > timeout_s:
                raise TimeoutError(f"P2PGather: {what} did not arrive (rank {self.rank}, seq {value})")
            time.sleep(0.0002)

    def gather(self, x: torch.Tensor, dst: Optional[int] = 0):
        """Collective.  ``dst=None``: every rank receives every tensor (all-gather); otherwise only
        ``dst`` does.  Returns the list of ``world`` tensors (same shape / dtype as ``x``) or ``None``."""
        x = x.contiguous()
        nbytes = x.numel() * x.element_size()
        if nbytes > self.slot:
            raise ValueError(f"tensor of {nbytes} bytes exceeds the gather slot ({self.slot})")
        if self.world == 1:
            return [x.clone()]
        self.seq += 1
        seq, buf = self.seq, self.seq & 1
        dsts = range(self.world) if dst is None else [int(dst)]
        raw = x.view(torch.uint8).reshape(-1)
        for d in dsts:
            prev = self._last_use[d][buf]
            if prev:      # slot reuse: the destination must have consumed the call that used it last
                self._wait(self.acks, d, prev, f"ack of rank {d}")
            self._last_use[d][buf] = seq
            off = (buf * self.world + self.rank) * self.slot
            self.heap.peer_tensor(d, (nbytes,), torch.uint8, off).copy_(raw)          # one-sided store
            self.heap.peer_tensor(d, (1,), torch.int64, self._flags_off + 8 * self.rank).fill_(seq)
        if dst is not None and self.rank != dst:
            return None
        self._wait(self.flags, None, seq, "a partial list")
        out = []
        for r in range(self.world):
            off = (buf * self.world + r) * self.slot
            out.append(self.heap.local_tensor((nbytes,), torch.uint8, off).clone().view(x.dtype).reshape(x.shape))
        torch.cuda.current_stream(self.device).synchronize()
        for r in range(self.world):   # acknowledge: the slots of this call may be overwritten
            self.heap.peer_tensor(r, (1,), torch.int64, self._acks_off + 8 * self.rank).fill_(seq)
        return out

    def close(self) -> None:
        self.heap.close()
