"""Device-resident sharded parameter table (the GPU-native "parameter server").

One dense fp32 block ``[rows_per_shard, stride]`` per PS rank lives in that GPU's HBM inside a
:class:`SymmetricHeap`; every rank maps every shard, and kernels address rows through the
``ShardTable`` pointer table.  Semantics reproduced from the reference stores:

* lazy ``paramInit`` on first pull (SimplePSLogic.scala:13-14) -- init is a pure function of the
  id (Philox keyed by ``(seed, id, column)``), so the shard is materialised eagerly and a
  *touched* bitmap records which ids were ever pulled/pushed (what ``close()`` would dump,
  SimplePSLogicWithClose.scala:27-31);
* additive ``paramUpdate`` on push (``vectorSum``, Vector.scala:72-84) -- fused into the push as
  ``red.global.add.v4.f32`` executed by the owner's memory system;
* hash (``abs(id) % n``, FPS:191-199) or range (RangePSLogicWithClose.scala:51-62) partitioning.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch
import torch.distributed as dist

from ..errors import FactorIsNotANumberException
from ..ops import native
from ..utils.metrics import GLOBAL as METRICS
from ..parallel.fabric import SymmetricHeap


_VALIDATE = os.environ.get("FPS_VALIDATE_IDS", "0") == "1"


class ShardedTable:
    def __init__(self, num_ids: int, dim: int, *, partition: str = "hash", group=None,
                 device: Optional[int] = None, init: str = "uniform", init_range=(-0.01, 0.01),
                 seed: int = 0, track_touched: bool = False, fabric_mode: Optional[str] = None,
                 num_shards: Optional[int] = None):
        """``num_shards`` = psParallelism (default: one shard per rank).  With fewer shards than ranks
        the shards live on ranks ``0 .. num_shards-1`` and the other ranks are pure workers
        (workerParallelism > psParallelism, FPS:340-481); every rank still maps every shard."""
        self.dim = int(dim)
        self.stride = (self.dim + 3) // 4 * 4
        self.num_ids = int(num_ids)
        self.partition = partition
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.group = group
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        self.n_shards = self.world if num_shards is None else int(num_shards)
        if not 1 <= self.n_shards <= self.world:
            raise ValueError("num_shards must be in [1, world size] (use MultiShardTable for several "
                             "shards per process)")
        if self.n_shards > native.FPS_MAX_SHARDS:
            raise ValueError(f"at most {native.FPS_MAX_SHARDS} shards are supported")
        self.owns_shard = self.rank < self.n_shards
        self.rows_per_shard = -(-self.num_ids // self.n_shards)
        self.div = self.rows_per_shard
        self.mode = native.PART_HASH if partition == "hash" else native.PART_RANGE
        self.seed = int(seed)
        self.track_touched = bool(track_touched)

        row_bytes = self.rows_per_shard * self.stride * 4
        self._bitmap_words = (self.rows_per_shard + 31) // 32
        self._bitmap_off = (row_bytes + 255) // 256 * 256
        total = self._bitmap_off + (self._bitmap_words * 4 if track_touched else 0)
        self.heap = SymmetricHeap(total, group=group, device=self.device, mode=fabric_mode)
        self.local = self.heap.local_tensor((self.rows_per_shard, self.stride), torch.float32)
        self.touched = (self.heap.local_tensor((self._bitmap_words,), torch.int32, self._bitmap_off)
                        if track_touched else None)

        self._check_agreement()
        tc = native.ShardTableC()
        for r in range(self.n_shards):
            tc.base[r] = self.heap.peer_ptrs[r]
            tc.touched[r] = (self.heap.peer_ptrs[r] + self._bitmap_off) if track_touched else None
        tc.rows_per_shard = self.rows_per_shard
        tc.div = self.div
        tc.num_shards = self.n_shards
        tc.dim = self.dim
        tc.stride = self.stride
        tc.mode = self.mode
        tc.shard_shift = native.log2_or_neg(self.n_shards)
        self.table_c = tc
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=self.cuda_device)

        if init == "uniform":
            self.init_uniform(*init_range)
        elif init == "zeros":
            pass  # heap is zero-filled
        else:
            raise ValueError(f"unknown init {init!r}")
        self.heap.barrier()

    # ------------------------------------------------------------------------------------
    @property
    def cuda_device(self) -> torch.device:
        return torch.device("cuda", self.device)

    def _check_agreement(self) -> None:
        """All ranks must describe the same table: a kernel computes peer row addresses from ITS view
        (slot = id / num_shards, stride), so a rank that passed a different ``num_ids`` / ``dim`` would
        read and reduce out of bounds in its peers' allocations."""
        if self.world == 1:
            return
        mine = (self.num_ids, self.dim, self.stride, self.n_shards, self.partition, self.rows_per_shard)
        views = [None] * self.world
        dist.all_gather_object(views, mine, group=self.group)
        if any(v != mine for v in views):
            raise ValueError(f"ranks disagree on the table geometry (num_ids, dim, stride, shards, "
                             f"partition, rows_per_shard): {views}")

    def validate_ids(self, ids: torch.Tensor) -> None:
        """Optional bounds check (one host sync): every id must address an allocated slot."""
        if ids.numel() == 0:
            return
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= self.rows_per_shard * self.n_shards:
            raise IndexError(f"parameter id out of range: [{lo}, {hi}] not within [0, {self.num_ids})")

    def init_uniform(self, lo: float, hi: float) -> None:
        """K4: slot <- init(id) for every slot of the local shard."""
        if not self.owns_shard:
            return
        with torch.cuda.device(self.device):
            native.init_rows(self.local, self.dim, self.rank, self.n_shards, self.mode, self.div,
                             self.seed, lo, hi)

    def local_ids(self) -> torch.Tensor:
        """Global ids of the local shard's slots, in slot order."""
        slots = torch.arange(self.rows_per_shard if self.owns_shard else 0, device=self.cuda_device,
                             dtype=torch.int64)
        if self.mode == native.PART_HASH:
            return slots * self.n_shards + self.rank
        return slots + self.rank * self.div

    # -- generic tensor tier: batched pull / push ---------------------------------------------
    def pull(self, ids: torch.Tensor, out: Optional[torch.Tensor] = None,
             pull_limit: int = 0) -> torch.Tensor:
        """values[i] = table[ids[i]] -- one-sided gather from the owning shards (K1).
        ``pull_limit`` > 0 bounds the row pulls in flight on the device (the pull limiter).
        Hash mode addresses ``abs(id)``; negative keys must be interned first (see ``_reject_negative``)."""
        self._reject_negative(ids)
        if out is None:
            out = torch.empty((ids.numel(), self.dim), dtype=torch.float32, device=ids.device)
        native.pull_gather(self._table_on(ids.device), ids, out, touch=self.track_touched,
                           max_inflight_rows=pull_limit,
                           credits=self._credits(pull_limit, ids.device) if pull_limit > 0 else None)
        METRICS.inc("ps_pull_rows", ids.numel())
        return out

    def _table_on(self, device) -> native.ShardTableC:
        """The pointer table valid on ``device`` (MultiShardTable keeps one LUT copy per GPU)."""
        tf = getattr(self, "table_for", None)
        return tf(device.index) if tf is not None and device.index is not None else self.table_c

    def _credits(self, pull_limit: int, device) -> torch.Tensor:
        """Device credit counter of the pull limiter: ``[credits, stalls]``, armed with ``pull_limit``."""
        key = (int(pull_limit), str(device))
        store = self.__dict__.setdefault("_credit_counters", {})
        if key not in store:
            store[key] = torch.tensor([int(pull_limit), 0], dtype=torch.int32, device=device)
        return store[key]

    def credit_stalls(self) -> int:
        return sum(int(c[1]) for c in self.__dict__.get("_credit_counters", {}).values())

    def _reject_negative(self, ids: torch.Tensor) -> None:
        """``FPS_VALIDATE_IDS=1``: range-check ids (one host sync per call).  The device tables address
        ``abs(id)``, so ``+x`` and ``-x`` would alias: negative / opaque keys go through an interner."""
        if _VALIDATE:
            self.validate_ids(ids)

    def push(self, ids: torch.Tensor, deltas: torch.Tensor, scale: float = 1.0) -> None:
        """table[ids[i]] += scale * deltas[i] -- push fused with the additive paramUpdate (K2)."""
        self._reject_negative(ids)
        native.push_add(self._table_on(ids.device), ids, deltas, scale=scale, touch=self.track_touched,
                        nan_flag=self.nan_flag if self.nan_flag.device == ids.device else None)
        METRICS.inc("ps_push_rows", ids.numel())

    def pull_dot(self, ids: torch.Tensor, local_vectors: torch.Tensor) -> torch.Tensor:
        score = torch.empty(ids.numel(), dtype=torch.float32, device=ids.device)
        native.pull_dot(self._table_on(ids.device), ids, local_vectors, score)
        return score

    def check_finite(self) -> None:
        """Raise like ``FactorIsNotANumberException`` (Vector.scala:78-80) if a NaN was pushed."""
        if int(self.nan_flag.item()) != 0:
            raise FactorIsNotANumberException("non-finite value pushed to the parameter server")

    # -- model export / import (PS output at close; transformWithModelLoad) -------------------
    def dump_local(self, only_touched: Optional[bool] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(ids, values) of the local shard -- the ``close()`` dump of the *WithClose logics."""
        torch.cuda.synchronize(self.device)
        if not self.owns_shard:
            return (torch.empty(0, dtype=torch.int64, device=self.cuda_device),
                    torch.empty((0, self.dim), dtype=torch.float32, device=self.cuda_device))
        ids = self.local_ids()
        valid = ids < self.num_ids
        if only_touched is None:
            only_touched = self.track_touched
        if only_touched and self.touched is not None:
            words = self.touched
            slots = torch.arange(self.rows_per_shard, device=self.cuda_device)
            bits = (words[slots >> 5] >> (slots & 31)) & 1
            valid = valid & (bits != 0)
        sel = valid.nonzero(as_tuple=True)[0]
        return ids[sel], self.local[sel, : self.dim].clone()

    def load(self, ids: torch.Tensor, values: torch.Tensor) -> None:
        """Model load: overwrite rows with given values (any rank may load any id)."""
        native.push_assign(self._table_on(ids.device), ids, values.to(torch.float32).contiguous(),
                           touch=self.track_touched)

    def barrier(self) -> None:
        self.heap.barrier()

    def close(self) -> None:
        self.heap.close()

    def row_accumulators(self, width: int = 1) -> "RowAccumulators":
        """Zeroed fp32 optimizer state partitioned exactly like this table: one per row (``width=1``, row-wise
        AdaGrad) or one per element (``width=stride``, element-wise AdaGrad)."""
        return RowAccumulators(self, width)


class RowAccumulators:
    """Optimizer state of a :class:`ShardedTable`: a ``[rows_per_shard]`` (``width=1``: one per row) or
    ``[rows_per_shard, stride]`` (``width=stride``: one per element, at its parameter's slot and column) fp32 block
    per shard in its own symmetric heap, so peers read and reduce it the way they reach the rows.  ``table_c``
    addresses it with the table's partitioning (stride 1, or the table's dim and stride); ``local`` is this rank's
    block."""

    def __init__(self, table: ShardedTable, width: int = 1):
        if int(width) not in (1, table.stride):
            raise ValueError(f"width must be 1 (per row) or the table's stride {table.stride} (per element), "
                             f"got {width}")
        self.table = table
        self.width = int(width)
        self.heap = SymmetricHeap(table.rows_per_shard * self.width * 4, group=table.group, device=table.device,
                                  mode=table.heap.mode)
        shape = (table.rows_per_shard,) if self.width == 1 else (table.rows_per_shard, self.width)
        self.local = self.heap.local_tensor(shape, torch.float32)
        src = table.table_c
        tc = native.ShardTableC()
        for r in range(table.n_shards):
            tc.base[r] = self.heap.peer_ptrs[r]
        tc.rows_per_shard, tc.div, tc.num_shards = src.rows_per_shard, src.div, src.num_shards
        tc.dim, tc.stride = (1, 1) if self.width == 1 else (src.dim, src.stride)
        tc.mode, tc.shard_shift, tc.lut = src.mode, src.shard_shift, src.lut
        self.table_c = tc
        self.heap.barrier()

    def dump_local(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(ids, accumulators) of the local shard's valid rows (``[n]``, or ``[n, stride]`` per element)."""
        torch.cuda.synchronize(self.table.device)
        ids = self.table.local_ids()
        sel = (ids < self.table.num_ids).nonzero(as_tuple=True)[0]
        return ids[sel], self.local[sel].clone()

    def load(self, ids: torch.Tensor, values: torch.Tensor) -> None:
        """Overwrite the local shard's accumulators of ``ids`` (ids this rank owns)."""
        t = self.table
        slots = ids // t.n_shards if t.mode == native.PART_HASH else ids - t.rank * t.div
        self.local[slots] = values.to(self.local.device, torch.float32)

    def close(self) -> None:
        self.heap.close()
