"""Device (H100) implementation of online / offline SGD matrix factorisation.

Capability parity with ``PSOnlineMatrixFactorization.psOnlineMF`` and
``PSOfflineMatrixFactorization.psOfflineMF`` (reference:
M/matrix/factorization/PSOnlineMatrixFactorization.scala:39-75,
M/matrix/factorization/workers/PSOnlineMatrixFactorizationWorker.scala:22-90):

* user vectors live on the *worker* that owns the user (``user % workerParallelism``),
* item vectors live on the parameter server, sharded ``item % psParallelism``,
* every rating triggers pull(item) -> SGD delta -> local user update -> push(item delta).

Device mechanism: one process per GPU is both worker ``rank`` and PS shard ``rank``; the whole
worker step for a micro-batch is ONE kernel (``fps_mf_sgd_fused``) that pulls item rows with
16-byte loads from the owner's HBM over NVSwitch, computes the update and pushes the delta back
with ``red.global.add.v4.f32`` -- no messages, no NCCL, no separate elementwise kernel.
"""
from __future__ import annotations

import math
import os
from typing import Iterable, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from ...errors import FactorIsNotANumberException
from ...ops import native
from ...utils.metrics import GLOBAL as METRICS
from ...runtime.device_stream import DevicePrefetcher
from ...store.replica_cache import ReplicaCache
from ...store.sharded_table import ShardedTable

ERR_SIGMOID = 0  # reference parity: e = sigmoid(r - u.v)   (SGDUpdater.scala:8)
ERR_PLAIN = 1    # textbook SGD:     e = r - u.v

DEFAULT_DEVICE_PULL_LIMIT = 0  # 0 = as many row slots in flight as the GPU can hold

L2_TABLE_BYTES = 48 << 20      # item tables above this do not stay in an H100's 50 MB L2 between launches
WINDOW_BUDGET = 256 << 20      # device memory of the step window: slot table + record staging
WINDOW_BYTES_PER_ROW = 8 + 12  # per item row and window slot: one slot-table entry + one int32-array record
WINDOW_MAX_STRIDE = 128        # floats per row the window kernel handles (k <= 128)


OPTIMIZERS = ("sgd", "adagrad")


def check_optimizer(optimizer: str, *, item_cache: bool, output_ring=None, kernel: Optional[str] = None) -> None:
    """Raise ``ValueError`` for an optimizer :class:`DeviceOnlineMF` cannot run with these settings.  Row-wise
    AdaGrad runs per launch on the register-staged kernel, reading its accumulators where the rows live, so it
    needs the direct mode (``item_cache=False``) and has no output ring or TMA kernel."""
    if optimizer not in OPTIMIZERS:
        raise ValueError(f"optimizer must be 'sgd' or 'adagrad', got {optimizer!r}")
    if optimizer == "sgd":
        return
    if item_cache:
        raise ValueError("optimizer='adagrad' is not supported in the replica (item_cache) mode, the multi-GPU "
                         "default: pass item_cache=False to read and update the item rows on their owners")
    if output_ring is not None:
        raise ValueError("optimizer='adagrad' does not support the per-update output ring (output_ring=None)")
    if kernel == "tma":
        raise ValueError("optimizer='adagrad' runs on the register-staged kernel: pass kernel=None or 'reg'")


NEGATIVE_SAMPLING = ("uniform", "seen")
STATS_SIZE = {"pointwise": 2, "bpr": 3, "warp": 4}


def check_warp(loss: str, margin: Optional[float], *, optimizer: str, negative_sampling: str) -> Optional[float]:
    """The margin :class:`DeviceOnlineMF` trains ``loss`` with (``None`` unless ``loss="warp"``, whose default is
    1.0); ``ValueError`` for a setting WARP cannot run.  WARP runs with SGD only, and its rank estimate needs one
    candidate domain for every record: ``negative_sampling="uniform"``."""
    if loss != "warp":
        if margin is not None:
            raise ValueError(f"margin is a parameter of loss='warp' (got loss={loss!r}): drop margin= or pass "
                             f"loss='warp'")
        return None
    margin = 1.0 if margin is None else float(margin)
    if not math.isfinite(margin):
        raise ValueError(f"margin must be a finite number, got {margin!r}")
    if optimizer != "sgd":
        raise ValueError(f"loss='warp' trains with SGD only: pass optimizer='sgd' (got {optimizer!r})")
    if negative_sampling != "uniform":
        raise ValueError("loss='warp' needs negative_sampling='uniform': its rank estimate assumes every record "
                         "draws from the same item range")
    return margin


def check_negative_sampling(negative_sampling: str, negative_sample_rate: int, negatives=None) -> None:
    """Raise ``ValueError`` for a negative-sampling setting :class:`DeviceOnlineMF` cannot run.  ``"seen"`` draws
    the negatives itself from the items the worker has seen, so it needs a positive ``negative_sample_rate`` and
    takes no ``step(negatives=...)``."""
    if negative_sampling not in NEGATIVE_SAMPLING:
        raise ValueError(f"negative_sampling must be 'uniform' or 'seen', got {negative_sampling!r}")
    if negative_sampling != "seen":
        return
    if int(negative_sample_rate) < 1:
        raise ValueError("negative_sampling='seen' needs negative_sample_rate >= 1 (or negative_sampling='uniform')")
    if negatives is not None:
        raise ValueError("negative_sampling='seen' draws the negatives itself: call step() without negatives=, or "
                         "use negative_sampling='uniform' to pass explicit negatives")


def step_window_size(step_window: Optional[int], *, world: int, item_cache: bool, loss: str, table_rows: int,
                     stride: int, env: Optional[str] = None, optimizer: str = "sgd") -> int:
    """Micro-batches per step window of :class:`DeviceOnlineMF` (0 = off).

    ``None`` = auto: on for one worker without an item cache whose item table exceeds the L2 (where every
    micro-batch re-reads it from HBM), unless ``FPS_STEP_WINDOW=0`` (``env``).  ``0`` / ``1`` = off, ``n >= 2`` =
    at most ``n`` (and at most ``native.WINDOW_MAX``).  The slot table and the staging area take
    ``W * table_rows * 20`` bytes, capped at ``WINDOW_BUDGET``: ``W`` is lowered to fit, and the window is off
    below 2.  Row-wise AdaGrad (``optimizer="adagrad"``) runs per launch: 0."""
    if world != 1 or item_cache or loss != "pointwise" or optimizer != "sgd" or stride > WINDOW_MAX_STRIDE \
            or table_rows < 1:
        return 0
    if step_window is None:
        if env == "0" or table_rows * stride * 4 <= L2_TABLE_BYTES:
            return 0
        w = native.WINDOW_MAX
    else:
        w = min(int(step_window), native.WINDOW_MAX)
    w = min(w, WINDOW_BUDGET // (table_rows * WINDOW_BYTES_PER_ROW))
    return w if w >= 2 else 0


def step_windowable(*, neg: int, output_ring, pull_limit: int, credits, kernel: Optional[str], kernel_env: str,
                    reg_variant_env: Optional[str], l2_hints: bool, packed: bool, dtypes: Tuple, n_records: int,
                    table_rows: int, on_gpu: bool, capturing: bool) -> bool:
    """Whether one pointwise ``step()`` can join the window: the per-launch path it replaces is the default
    register-staged kernel (no negatives, output ring, pull limiter, L2 hints or other variant) on int32 or
    packed64 records, no more of them than the table has rows, outside CUDA-graph capture."""
    if neg != 0 or output_ring is not None or pull_limit != 0 or credits is not None or l2_hints:
        return False
    if (kernel or kernel_env) != "reg" or reg_variant_env not in (None, "0") or capturing or not on_gpu:
        return False
    ok_dtypes = dtypes == (torch.int64,) if packed else dtypes == (torch.int32, torch.int32, torch.float32)
    return ok_dtypes and n_records <= table_rows


class DeviceOnlineMF:
    def __init__(self, num_users: int, num_items: int, num_factors: int = 10,
                 range_min: float = -0.01, range_max: float = 0.01, learning_rate: float = 0.01,
                 negative_sample_rate: int = 0, pull_limit: int = DEFAULT_DEVICE_PULL_LIMIT,
                 group=None, seed: int = 0, err_mode: int = ERR_SIGMOID,
                 device: Optional[int] = None, track_touched: bool = False,
                 kernel: Optional[str] = None, item_cache: Optional[bool] = None,
                 sync_every: int = 4, user_memory: int = 0,
                 sync_interval_ms: Optional[float] = None, item_blocking: Optional[bool] = None,
                 block_bytes: int = 16 << 20, flush_count: Optional[int] = None,
                 flush_require: str = "any", replica_own_inplace: Optional[bool] = None,
                 output_ring=None, loss: str = "pointwise", regularization: float = 0.0,
                 step_window: Optional[int] = None, optimizer: str = "sgd",
                 negative_sampling: str = "uniform", margin: Optional[float] = None):
        """``loss="bpr"``: pairwise (Bayesian Personalised Ranking) updates, each positive rating paired
        with ``negative_sample_rate`` negatives (sampled) or with the ``negatives=`` of :meth:`step`;
        ``regularization`` is its L2 weight.  The pointwise loss has no regulariser.

        ``step_window``: how many micro-batches :meth:`step` may defer and then apply in one item-major pass
        (see :meth:`step` and :func:`step_window_size`; ``None`` = auto, ``0`` = off).

        ``optimizer="adagrad"``: row-wise AdaGrad (DESIGN §2.10) instead of SGD with one global rate.  Each row
        keeps one fp32 accumulator ``G`` of its mean squared delta and steps by ``learning_rate / (sqrt(G) +
        1e-8)``; users' accumulators stay on their worker, items' on the item's shard.  It runs per launch (no
        step window) in the direct mode only: ``item_cache=False`` when there is more than one GPU.

        ``negative_sampling``: where negatives come from.  ``"uniform"`` draws them uniformly over ``[0,
        num_items)``.  ``"seen"`` draws them, as the reference and the host tiers do, from the items this worker
        has seen so far (DESIGN §2.11): a device registry keeps them in first-occurrence order (see
        :meth:`seen_items`), rating ``p`` of a micro-batch samples from the items seen before it, rejecting the
        user's last ``user_memory`` items and the positive, and gets ``min(negative_sample_rate, |domain| -
        |user's recent items|)`` negatives.  It needs ``negative_sample_rate >= 1``.

        ``loss="warp"``: WARP, the Weighted Approximate-Rank Pairwise loss (DESIGN §2.12).  Each positive rating
        examines up to ``negative_sample_rate`` candidates (sampled as BPR's negatives, or the ``negatives=`` of
        :meth:`step`) until one scores within ``margin`` (default 1.0) of the positive, and makes one hinge update
        scaled by ``ln((num_items - 1) // n)``, ``n`` the candidates it took.  ``regularization`` is its L2 weight.  It
        runs with SGD and ``negative_sampling="uniform"``, in the direct and the replica mode."""
        self._pending = []           # staged micro-batches of the step window: (records, format)
        self.step_window = 0
        check_negative_sampling(negative_sampling, negative_sample_rate)
        self.negative_sampling = negative_sampling
        if loss not in ("pointwise", "bpr", "warp"):
            raise ValueError(f"loss must be 'pointwise', 'bpr' or 'warp', got {loss!r}")
        self.loss, self.reg = loss, float(regularization)
        if loss == "pointwise" and self.reg != 0.0:
            raise ValueError("regularization is only supported with loss='bpr' or loss='warp'")
        self.margin = check_warp(loss, margin, optimizer=optimizer, negative_sampling=negative_sampling)
        if loss != "pointwise":
            if output_ring is not None:
                raise ValueError(f"the per-update output ring is not supported with loss={loss!r}")
            if kernel == "tma":
                raise ValueError(f"kernel='tma' is not supported with loss={loss!r}")
            if item_blocking:
                raise ValueError(f"item_blocking is not supported with loss={loss!r}")
            item_blocking = False
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.cuda_device = torch.device("cuda", self.device)
        self.group = group
        ready = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if ready else 1
        self.rank = dist.get_rank(group) if ready else 0
        if item_cache is None:
            item_cache = self.world > 1 and os.environ.get("FPS_ITEM_CACHE", "1") != "0"
        check_optimizer(optimizer, item_cache=bool(item_cache), output_ring=output_ring, kernel=kernel)
        self.optimizer = optimizer
        self.num_users, self.num_items, self.k = int(num_users), int(num_items), int(num_factors)
        self.lr = float(learning_rate)
        self.neg = int(negative_sample_rate)
        self.pull_limit = int(pull_limit)
        self.err_mode = int(err_mode)
        self.seed = int(seed)
        self.step_no = 0
        self.kernel = kernel
        # pull limiter (WL:196-250) = device credit counter [credits, stalls] consumed inside the fused kernel
        # (a warp takes its credits all at once, so limits below one warp's worth of pulls fall back to the
        # static form of the limiter: a capped grid)
        # (the BPR kernel has only the static form)
        self.credits = (torch.tensor([self.pull_limit, 0], dtype=torch.int32, device=self.cuda_device)
                        if self.pull_limit >= 32 and os.environ.get("FPS_STATIC_LIMITER", "0") != "1"
                        and loss == "pointwise" and optimizer == "sgd" else None)
        self.output_ring = output_ring     # E5: per-update (user, vector) output stream (runtime/output_ring.py)
        with torch.cuda.device(self.device):
            # parameter server: item vectors, sharded item % psParallelism
            self._items = ShardedTable(num_items, num_factors, partition="hash", group=group,
                                      device=self.device, init="uniform",
                                      init_range=(range_min, range_max), seed=seed * 2 + 1,
                                      track_touched=track_touched)
            # worker-local state: vectors of the users this worker owns (user % W == rank)
            n_local = -(-self.num_users // self.world)
            self._users = torch.empty((n_local, self._items.stride), dtype=torch.float32,
                                     device=self.cuda_device)
            native.init_rows(self._users, self.k, self.rank, self.world, native.PART_HASH, n_local,
                             seed * 2 + 2, range_min, range_max)
            # pointwise: [sum (r - u.v)^2, updates]; BPR: [sum softplus(-x), triples, triples with x > 0];
            # WARP: [sum L * (margin - x), positives updated, candidates examined, positives]
            self._stats = torch.zeros(STATS_SIZE[loss], dtype=torch.float32, device=self.cuda_device)
            # row-wise AdaGrad: one fp32 accumulator per user row (worker-local) and per item row (item shard)
            self._user_acc = self._item_acc = None
            if optimizer == "adagrad":
                self._user_acc = torch.zeros(n_local, dtype=torch.float32, device=self.cuda_device)
                self._item_acc = self._items.row_accumulators()
            self._nan_flag = torch.zeros(1, dtype=torch.int32, device=self.cuda_device)
            # K5: per-user memory of recently seen items (userMemory of the reference, default 128
            # there; 0 here = sample uniformly inside the fused kernel, rejecting only the positive)
            self.user_memory = int(user_memory) if self.neg > 0 else 0
            if self.user_memory > 0:
                self.seen = torch.full((n_local, self.user_memory), -1, dtype=torch.int32,
                                       device=self.cuda_device)
                self.seen_pos = torch.zeros(n_local, dtype=torch.int32, device=self.cuda_device)
            # negative_sampling="seen": the items this worker has seen, in first-occurrence order
            self._registry = (native.seen_registry(self.num_items, self.cuda_device)
                              if negative_sampling == "seen" else None)
        # ---- item-cache mode (sender-side combining) --------------------------------------------
        # The worker trains a local owner-major replica of the item table (pulls and pushes stay in local
        # HBM); its segments are the per-destination send buffers of the reference's batching senders.
        # After every micro-batch a device-side count / timer policy (fps_flush_policy) picks the
        # destinations to flush -- by default each destination once per `sync_every` micro-batches,
        # staggered -- and a few TMA-driven CTAs (fps_replica_exchange) push (replica - base) to those
        # master shards and fold the other workers' contributions (master - base) into the replica while
        # the training kernel keeps running.  Asynchronous (no barriers); staleness ~ `sync_every` steps.
        self.item_cache = bool(item_cache)
        self.sync_every = max(1, int(sync_every))
        self.sync_interval_ms = sync_interval_ms
        self.flush_count, self.flush_require = flush_count, flush_require
        self._own_inplace = replica_own_inplace
        self.replica = (ReplicaCache(self._items, self.sync_every, sync_interval_ms,
                                     require=flush_require, flush_count=flush_count,
                                     own_inplace=replica_own_inplace)
                        if self.item_cache else None)
        # ---- L2 blocking: deal each micro-batch into buckets of <= 16 MB of item rows (fps_bucket.cu) ----
        # only where the item rows are read from local HBM (single GPU, or the local replica)
        row_bytes = self._items.stride * 4
        if item_blocking is None:
            item_blocking = ((self.world == 1 or self.item_cache) and self.num_items * row_bytes > (48 << 20)
                             and (self.neg == 0 or self.user_memory > 0 or negative_sampling == "seen")
                             and os.environ.get("FPS_ITEM_BLOCKING", "1") != "0")
        self.item_blocking = bool(item_blocking)
        block_bytes = int(os.environ.get("FPS_BLOCK_BYTES", block_bytes))
        self.l2_hints = self.item_blocking and os.environ.get("FPS_L2_HINTS", "0") == "1"
        per_bucket = max(1, int(block_bytes) // row_bytes)
        self.block_shift = max(0, per_bucket.bit_length() - 1)
        # buckets are ranges of rows of the table the fused kernel reads: the item shard (N = 1) or the
        # owner-major replica (row = owner * rows_per_shard + slot)
        table_rows = self._items.rows_per_shard * self.world if self.item_cache else self.num_items
        self._table_rows = table_rows
        while -(-table_rows >> self.block_shift) > native.BUCKET_MAX:
            self.block_shift += 1
        self.block_buckets = max(1, -(-table_rows >> self.block_shift))
        if self.item_blocking:
            with torch.cuda.device(self.device):
                self._bucket_scratch = torch.zeros(2 * native.BUCKET_MAX, dtype=torch.int32,
                                                   device=self.cuda_device)
        # ---- step window (fps_mf_window.cu): buffers allocated by the first windowed step ----------------
        self.step_window = step_window_size(step_window, world=self.world, item_cache=self.item_cache,
                                            loss=self.loss, table_rows=self.num_items, stride=self._items.stride,
                                            env=os.environ.get("FPS_STEP_WINDOW"), optimizer=optimizer)
        self._win = None
        self._win_phase_ns = None   # optional int64 [4]: build / apply ns of every drain (mf_window_drain)
        self._graph_capture = False
        self._per_launch = False
        self._items.barrier()

    # -- model state: every read applies the pending step window first ------------------------------------
    @property
    def stats(self) -> torch.Tensor:
        self._drain()
        return self._stats

    @property
    def users(self) -> torch.Tensor:
        self._drain()
        return self._users

    @property
    def items(self) -> ShardedTable:
        self._drain()
        return self._items

    @property
    def nan_flag(self) -> torch.Tensor:
        self._drain()
        return self._nan_flag

    @property
    def accumulators(self) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
        """Row-wise AdaGrad state ``(user_acc [n_local], item_acc_local [rows_per_shard])``, slot-indexed like
        ``users`` and ``items.local``; ``None`` with ``optimizer="sgd"``."""
        self._drain()
        if self._item_acc is None:
            return None
        return self._user_acc, self._item_acc.local

    def _windowable(self, users, items, ratings) -> bool:
        if self.step_window < 2 or self._graph_capture or self._per_launch:
            return False
        packed = items is None
        return step_windowable(
            neg=self.neg, output_ring=self.output_ring, pull_limit=self.pull_limit, credits=self.credits,
            kernel=self.kernel, kernel_env=os.environ.get("FPS_MF_KERNEL", "reg"),
            reg_variant_env=os.environ.get("FPS_MF_REG_VARIANT"), l2_hints=self.l2_hints, packed=packed,
            dtypes=(users.dtype,) if packed else (users.dtype, items.dtype, ratings.dtype),
            n_records=users.numel(), table_rows=self.num_items, on_gpu=users.is_cuda,
            capturing=torch.cuda.is_current_stream_capturing())

    def _stage(self, users, items, ratings) -> None:
        """Copy one micro-batch into the next slot of the device staging area (stream-ordered; the caller may
        reuse its tensors at once).  No kernel runs."""
        if self._win is None:
            rows, w = self.num_items, self.step_window
            slot_bytes = -(-rows * 12 // 256) * 256
            with torch.cuda.device(self.device):
                dev = self.cuda_device
                self._win = {
                    "slot_bytes": slot_bytes,
                    "stage": torch.empty(w * slot_bytes, dtype=torch.uint8, device=dev),
                    "slots": torch.full((w, rows), -1, dtype=torch.int64, device=dev),   # item-major slot table
                    "user_bits": torch.zeros(-(-self._users.shape[0] // 32), dtype=torch.int32, device=dev),
                    "ctl": torch.zeros(2 * native.WINDOW_MAX, dtype=torch.int32, device=dev),
                    "slot_stats": torch.zeros((w, 2), dtype=torch.float32, device=dev),
                }
        j = len(self._pending)
        n = users.numel()
        sb = self._win["slot_bytes"]
        slot = self._win["stage"][j * sb:(j + 1) * sb]
        if items is None:
            slot[:8 * n].view(torch.int64).copy_(users.reshape(-1), non_blocking=True)
        else:
            ids = slot[:12 * n].view(torch.int32)
            ids[:n].copy_(users.reshape(-1), non_blocking=True)
            ids[n:2 * n].copy_(items.reshape(-1), non_blocking=True)
            ids[2 * n:].view(torch.float32).copy_(ratings.reshape(-1), non_blocking=True)
        self._pending.append((n, 1 if items is None else 0))
        self.step_no += 1
        METRICS.inc("mf_ratings", n)

    def _drain(self) -> int:
        """Apply the staged micro-batches in order (one launch); returns how many there were."""
        n = len(self._pending)
        if n == 0:
            return 0
        counts, fmts = zip(*self._pending)
        self._pending = []
        w = self._win
        native.mf_window_drain(w["stage"], w["slot_bytes"], counts, fmts, self._users, self._items.local, self.lr,
                               self.err_mode, w["slots"], w["user_bits"], w["ctl"], self._stats, w["slot_stats"],
                               self._nan_flag, phase_ns=self._win_phase_ns)
        return n

    # ------------------------------------------------------------------------------------
    def flush(self) -> None:
        """Apply the pending step window; item-cache mode: push every pending local delta to the master shards
        and wait for it."""
        self._drain()
        if self.replica is not None:
            self.replica.flush()

    def step(self, users: torch.Tensor, items: Optional[torch.Tensor] = None,
             ratings: Optional[torch.Tensor] = None, negatives: Optional[torch.Tensor] = None) -> None:
        """Process one micro-batch of ratings whose users belong to this worker (async SGD).
        ``step(packed)`` with a single int64 tensor takes packed64 records (``native.pack_ratings``).
        ``negatives`` (``loss="bpr"`` / ``"warp"`` only): ``[n, m]`` item ids paired with each rating, ``-1`` = none
        (WARP: the candidates, examined in column order).

        Lazy with a step window (``step_window``): an eligible micro-batch (:func:`step_windowable`) is only
        copied into a device staging slot -- the caller may reuse its tensors at once -- and the window is
        applied, in order and in one launch, before any observation of the model (``stats``, ``users``,
        ``items``, ``nan_flag``, :meth:`flush`, :meth:`predict`, :meth:`save`, :meth:`check_finite`, ...), before
        an ineligible step, and when it is full.  The tables then equal, bitwise, one fused launch per
        micro-batch whenever each micro-batch has distinct users and distinct items; a micro-batch with a user
        or an item twice is applied on its own, as racy as the per-launch path."""
        if self.loss == "pointwise" and negatives is None and self._windowable(users, items, ratings):
            self._stage(users, items, ratings)
            if len(self._pending) >= self.step_window:
                self._drain()
            return
        self._drain()
        check_negative_sampling(self.negative_sampling, self.neg, negatives)
        if self.loss != "pointwise":
            self._step_pairwise(users, items, ratings, negatives)
            return
        if negatives is not None:
            raise ValueError("negatives= needs loss='bpr' or loss='warp'")
        neg = self.neg
        if self.user_memory > 0 or self._registry is not None:
            # negatives drawn by a sampler kernel (the per-user seen ring, the seen-items registry); the fused kernel
            # then consumes the expanded batch as plain records
            users, items, ratings = self._sample_negatives(users, items, ratings)
            neg = 0
        n_records = users.numel()
        fed = False
        ring = self.output_ring
        out_args = ring.kernel_args() if ring is not None else None
        # The deal pays only when rows are revisited inside the launch: a local-table micro-batch with no more
        # records than the table has rows touches a row about once whatever the order (on one H100 the fused
        # kernel took the same time with and without it, profiles/h100_mf_step_breakdown.json).  The replica
        # mode always deals: the bucket histogram feeds its flush policy.
        revisits = self.item_cache or n_records * (1 + neg) > self._table_rows
        if self.item_blocking and self.block_buckets > 1 and revisits:
            hashed = self.item_cache and self._items.mode == native.PART_HASH
            fed = hashed
            users, items, ratings = native.bucket_by_item(
                users, items, ratings, self.block_shift, self.block_buckets, self._bucket_scratch,
                num_shards=self.world if hashed else 1, rows_per_shard=self._items.rows_per_shard,
                pending=self.replica.pending if hashed else None)
        if self.item_cache:
            # policy + exchange kernels of this micro-batch go first (side stream): their CTAs take the
            # slots the training grid leaves free
            self.replica.after_step(n_records * (1 + neg), fed=fed)
            native.mf_sgd_fused(users, items, ratings, self._users, self.world, self.replica.table_c,
                                self.lr, err_mode=self.err_mode, neg_rate=neg,
                                num_items=self.num_items, seed=self.seed, step=self.step_no,
                                stats=self._stats, nan_flag=self._nan_flag,
                                max_inflight_rows=self.pull_limit, kernel="reg", l2_hints=self.l2_hints,
                                reserve_total=self.replica.reserve_total(), output=out_args,
                                credits=self.credits)
        else:
            native.mf_sgd_fused(users, items, ratings, self._users, self.world, self._items.table_c,
                                self.lr, err_mode=self.err_mode, neg_rate=neg,
                                num_items=self.num_items, seed=self.seed, step=self.step_no,
                                stats=self._stats, nan_flag=self._nan_flag,
                                max_inflight_rows=self.pull_limit, kernel=self.kernel,
                                l2_hints=self.l2_hints, output=out_args, credits=self.credits,
                                item_acc=self._item_acc.table_c if self._item_acc is not None else None,
                                user_acc=self._user_acc)
        if ring is not None:               # device-side count / timer policy + flush to the pinned host ring
            ring.after_kernel(users.numel() * (1 + neg))
        self.step_no += 1
        METRICS.inc("mf_ratings", users.numel())

    def _step_pairwise(self, users, items, ratings, negatives) -> None:
        if negatives is not None:
            if self.item_cache:
                raise ValueError("negatives= is not supported in the replica (item_cache) mode")
            n = int(negatives.shape[1]) if negatives.dim() == 2 else 0
        elif self.neg < 1:
            raise ValueError(f"loss={self.loss!r} needs negative_sample_rate >= 1 or explicit negatives=")
        elif self.user_memory > 0 or self._registry is not None:
            # negatives that avoid the user's recent items: the sampler's expanded [n, 1 + m] records,
            # with the negatives it could not find voided
            per = 1 + self.neg
            ou, oi, orat = self._sample_negatives(users, items, ratings)
            ou, oi = ou.view(-1, per), oi.view(-1, per)
            negatives = torch.where(ou[:, 1:] >= 0, oi[:, 1:], torch.full_like(oi[:, 1:], -1)).contiguous()
            users, items, ratings = ou[:, 0].contiguous(), oi[:, 0].contiguous(), orat.view(-1, per)[:, 0].contiguous()
            n = self.neg
        else:
            n = self.neg                   # drawn inside the kernel
        if self.output_ring is not None:
            raise ValueError(f"the per-update output ring is not supported with loss={self.loss!r}")
        n_pos = users.numel()
        cand, reserve = self._items.table_c, 0
        if self.item_cache:
            # uniform per-destination counts feed the flush policy (pairwise batches are not dealt into buckets);
            # a WARP positive updates at most one candidate
            self.replica.after_step(n_pos * (n if self.loss == "bpr" else 1), fed=False)
            cand, reserve = self.replica.table_c, self.replica.reserve_total()
        if self.loss == "warp":
            native.mf_warp_fused(users, items, ratings, self._users, cand, self.lr, self.reg, margin=self.margin,
                                 rank_items=self.num_items, negatives=negatives, n_neg=n, num_items=self.num_items,
                                 seed=self.seed, step=self.step_no, anchor_div=self.world, stats=self._stats,
                                 nan_flag=self._nan_flag, max_inflight_rows=self.pull_limit, reserve_total=reserve)
            self.step_no += 1
            METRICS.inc("mf_ratings", n_pos)
            return
        native.mf_bpr_fused(users, items, ratings, self._users, cand, self.lr, self.reg, negatives=negatives,
                            n_neg=n, num_items=self.num_items, seed=self.seed, step=self.step_no,
                            anchor_div=self.world, stats=self._stats, nan_flag=self._nan_flag,
                            max_inflight_rows=self.pull_limit, reserve_total=reserve,
                            anchor_acc=self._user_acc,
                            cand_acc=self._item_acc.table_c if self._item_acc is not None else None)
        self.step_no += 1
        METRICS.inc("mf_ratings", n_pos)

    def _sample_negatives(self, users, items, ratings):
        """Expanded ``(users, items, ratings)`` records: each rating, then its ``negative_sample_rate`` negatives."""
        memory = self.user_memory > 0
        if self._registry is not None:
            return native.neg_sample_seen(users, items, ratings, self.neg, self._registry,
                                          self.seen if memory else None, self.seen_pos if memory else None,
                                          self.world, seed=self.seed, step=self.step_no)
        return native.neg_sample(users, items, ratings, self.neg, self.num_items, self.seen, self.seen_pos,
                                 self.world, seed=self.seed, step=self.step_no)

    def seen_items(self) -> torch.Tensor:
        """The item ids this worker has seen, in first-occurrence order (int64, on the device); the domain of
        ``negative_sampling="seen"``.  Raises ``ValueError`` with ``negative_sampling="uniform"``."""
        if self._registry is None:
            raise ValueError("seen_items() needs negative_sampling='seen'")
        order, count, _ = self._registry
        return order[:int(count.item())].to(torch.int64)

    def make_graph_step(self, batch_size: int, packed: bool = True):
        """CUDA-graph a fixed-size micro-batch step for launch-bound streaming (small batches).

        Returns ``(static_inputs, replay)``: copy the next batch into ``static_inputs`` (device
        tensors) and call ``replay()``; the captured graph contains the stats reset and the fused
        kernel, so one ``cudaGraphLaunch`` replaces the Python + ctypes launch path.  The graph holds the
        per-launch kernel: ``replay()`` applies a pending step window first."""
        self._drain()
        dev = self.cuda_device
        if packed:
            static = (torch.zeros(batch_size, dtype=torch.int64, device=dev),)
        else:
            static = (torch.zeros(batch_size, dtype=torch.int32, device=dev),
                      torch.zeros(batch_size, dtype=torch.int32, device=dev),
                      torch.zeros(batch_size, dtype=torch.float32, device=dev))
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        self._graph_capture = True       # warm-up and capture take the per-launch path
        try:
            with torch.cuda.stream(s):
                for _ in range(2):  # warm up outside capture
                    self._stats.zero_(); self.step(*static)
            torch.cuda.current_stream(dev).wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=s):
                self._stats.zero_()
                self.step(*static)
        finally:
            self._graph_capture = False

        def replay():
            self._drain()
            graph.replay()
        return static, replay

    def fit_stream(self, host_batches: Iterable[Sequence[torch.Tensor]],
                   loss_every: int = 1):
        """End-to-end training over pinned host micro-batches ``(users, items, ratings)``.

        Yields one host-side ``(sum_sq_err, n_updates)`` per micro-batch (device -> host read of
        the step's result), lagging the launch by one step so copies, kernels and reads overlap.
        With ``loss="bpr"`` the pair is ``(sum softplus(-x), n_triples)``, with ``loss="warp"`` ``(sum L * (margin -
        x), positives updated)``.
        It reads the loss after every micro-batch, so it takes the per-launch path (no step window).
        """
        self._drain()
        pf = DevicePrefetcher(host_batches, self.cuda_device, depth=2)
        self.prefetcher = pf
        pending = []
        ring = [torch.empty(self._stats.numel(), dtype=torch.float32).pin_memory() for _ in range(4)]
        i = 0
        for batch in pf:
            self._stats.zero_()
            self._per_launch = True
            try:
                self.step(*batch)
            finally:
                self._per_launch = False
            host = ring[i % len(ring)]
            host.copy_(self._stats, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            pending.append((host, ev))
            i += 1
            if len(pending) > 2:
                h, e = pending.pop(0)
                e.synchronize()
                yield float(h[0]), float(h[1])
        self.flush()
        for h, e in pending:
            e.synchronize()
            yield float(h[0]), float(h[1])

    # -- quality / export -------------------------------------------------------------------
    def predict(self, users: torch.Tensor, items: torch.Tensor) -> torch.Tensor:
        """u.v for (user, item) pairs whose users are local (pull fused with the dot)."""
        self.flush()
        slots = (users.to(torch.int64) // self.world)
        local = self._users[slots].contiguous()
        return self._items.pull_dot(items, local)

    def user_vectors(self) -> Tuple[torch.Tensor, torch.Tensor]:
        self._drain()
        n_local = self._users.shape[0]
        ids = torch.arange(n_local, device=self.cuda_device) * self.world + self.rank
        sel = ids < self.num_users
        return ids[sel], self._users[sel, : self.k].clone()

    def item_vectors(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """All item vectors of the local shard (the fused kernel does not maintain the touched bitmap:
        with Philox lazy-init every id has a well-defined value whether or not it was pulled)."""
        self.flush()
        return self._items.dump_local(only_touched=False)

    # -- checkpoint / resume (the reference only has export + transformWithModelLoad; SURVEY §5) ------
    def save(self, directory: str) -> str:
        """Every rank writes its user partition and its item shard to ``directory/rank<r>.npz``, with their
        AdaGrad accumulators when ``optimizer="adagrad"``."""
        import numpy as np

        os.makedirs(directory, exist_ok=True)
        self.barrier()
        uid, uvec = self.user_vectors()
        iid, ivec = self.item_vectors()
        path = os.path.join(directory, f"rank{self.rank}_of{self.world}.npz")
        extra = {}
        if self._item_acc is not None:
            aid, aval = self._item_acc.dump_local()
            extra = dict(user_acc=self._user_acc[uid // self.world].cpu().numpy(), item_acc_ids=aid.cpu().numpy(),
                         item_acc=aval.cpu().numpy())
        np.savez(path, user_ids=uid.cpu().numpy(), user_vecs=uvec.cpu().numpy(), item_ids=iid.cpu().numpy(),
                 item_vecs=ivec.cpu().numpy(), step_no=self.step_no, **extra)
        return path

    def load(self, directory: str) -> None:
        """Resume from :meth:`save` (same world size): users go back to their worker, items to their
        shard (one-sided assign), replicas are re-pulled.  AdaGrad accumulators are restored, or zeroed when
        the checkpoint has none."""
        import numpy as np

        self._drain()
        d = np.load(os.path.join(directory, f"rank{self.rank}_of{self.world}.npz"))
        uid = torch.from_numpy(d["user_ids"]).to(self.cuda_device)
        self._users[uid // self.world, : self.k] = torch.from_numpy(d["user_vecs"]).to(self.cuda_device)
        self._items.load(torch.from_numpy(d["item_ids"]).to(self.cuda_device),
                        torch.from_numpy(d["item_vecs"]).to(self.cuda_device))
        self.step_no = int(d["step_no"])
        if self._item_acc is not None:
            self._user_acc.zero_()
            self._item_acc.local.zero_()
            if "item_acc" in d.files:
                self._user_acc[uid // self.world] = torch.from_numpy(d["user_acc"]).to(self.cuda_device)
                self._item_acc.load(torch.from_numpy(d["item_acc_ids"]).to(self.cuda_device),
                                    torch.from_numpy(d["item_acc"]))
        self._items.barrier()
        if self.replica is not None:
            self.replica = ReplicaCache(self._items, self.sync_every, self.sync_interval_ms,
                                        require=self.flush_require, flush_count=self.flush_count,
                                        own_inplace=self._own_inplace)

    def check_finite(self) -> None:
        self._drain()
        if int(self._nan_flag.item()) != 0:
            raise FactorIsNotANumberException("non-finite SGD update")

    def barrier(self) -> None:
        self.flush()
        self._items.barrier()

    def refresh(self) -> None:
        """Collective quiesce: every delta is in the masters and every replica equals the master."""
        self._drain()
        if self.replica is not None:
            self.replica.refresh()
        else:
            self._items.barrier()

    def close(self) -> None:
        self._drain()
        if self._item_acc is not None:
            self._item_acc.close()
        self._items.close()
