"""``psOnlineMF(..., backend="device")`` / ``psOfflineMF(..., backend="device")``: reference-shaped
entry points over :class:`DeviceOnlineMF`.

``src`` is an iterable of ``Rating`` records (any size; micro-batched on the host, packed64, pinned)
or of ready ``(users, items, ratings)`` host tensors.  In a multi-rank job every rank passes its own
partition of the stream (users with ``user % world == rank``), like Flink's parallel sources behind
``partitionCustom(user % n)``.  The result stream holds ``Left((userId, vector))`` for the local
users touched and ``Right((itemId, vector))`` for the local shard's items (model dump at close).
"""
from __future__ import annotations

from typing import Iterator, List, Optional, Sequence

import torch

from ...api import Left, Right
from ...ops import native
from ...runtime.stream import ResultStream, as_stream
from .common import Rating
from .device import ERR_PLAIN, ERR_SIGMOID, STATS_SIZE, DeviceOnlineMF, check_warp


def _batches(src, batch_size: int) -> Iterator[Sequence[torch.Tensor]]:
    buf: List[Rating] = []
    for rec in (src.collect() if hasattr(src, "collect") else src):
        if isinstance(rec, (tuple, list)) and len(rec) in (1, 3) and torch.is_tensor(rec[0]):
            yield tuple(t if t.is_pinned() or not torch.cuda.is_available() else t.pin_memory() for t in rec)
            continue
        buf.append(rec)
        if len(buf) >= batch_size:
            yield _pack(buf)
            buf = []
    if buf:
        yield _pack(buf)


def _pack(buf: List[Rating]):
    u = torch.tensor([r.user for r in buf], dtype=torch.int32)
    i = torch.tensor([r.item for r in buf], dtype=torch.int32)
    r = torch.tensor([r.rating for r in buf], dtype=torch.float32)
    return (u.pin_memory(), i.pin_memory(), r.pin_memory())


def _result(model: DeviceOnlineMF, seen_users: Optional[set]) -> ResultStream:
    out = []
    uid, uvec = model.user_vectors()
    for i, v in zip(uid.cpu().tolist(), uvec.cpu().double().numpy()):
        if seen_users is None or i in seen_users:
            out.append(Left((i, v)))
    iid, ivec = model.item_vectors()
    for i, v in zip(iid.cpu().tolist(), ivec.cpu().double().numpy()):
        out.append(Right((i, v)))
    rs = ResultStream(out)
    rs.model = model
    return rs


def _agree_max(num_users: int, num_items: int, group):
    """Sizes derived from a rank's LOCAL partition differ between ranks; every rank must build the same
    table geometry (peer row addresses are computed from it), so take the maximum over the job."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return num_users, num_items
    sizes = [None] * dist.get_world_size(group)
    dist.all_gather_object(sizes, (int(num_users), int(num_items)), group=group)
    return max(s[0] for s in sizes), max(s[1] for s in sizes)


def ps_online_mf_device(src, numFactors=10, rangeMin=-0.01, rangeMax=0.01, learningRate=0.01,
                        negativeSampleRate=0, pullLimit=0, seed=0, plain_residual=False,
                        numUsers: Optional[int] = None, numItems: Optional[int] = None,
                        batch_size: int = 1 << 16, group=None, epochs: int = 1,
                        userMemory: int = 128, updateOutput: Optional[int] = None,
                        outputFlushCount: int = 1, outputFlushMs: Optional[float] = None,
                        loss: str = "pointwise", regularization: float = 0.0,
                        optimizer: str = "sgd", negativeSampling: Optional[str] = None,
                        margin: Optional[float] = None) -> ResultStream:
    """``updateOutput=n``: also emit ``Left((userId, userVector))`` for one update in ``n`` (``1`` = every
    update, the reference's worker output PSOnlineMatrixFactorizationWorker.scala:52) through the device
    output ring (count / timer flushed on the device); the final dump then holds only the item shard.
    ``loss="bpr"``: pairwise updates, every rating > 0 paired with ``negativeSampleRate`` sampled
    negatives, L2 weight ``regularization`` (see :class:`DeviceOnlineMF`); it has no per-update output,
    so ``updateOutput`` with ``loss="bpr"`` raises ``ValueError``.
    ``loss="warp"``: WARP, each rating > 0 examining up to ``negativeSampleRate`` sampled candidates until one is
    within ``margin`` (default 1.0) of it (see :class:`DeviceOnlineMF`); no per-update output either.
    ``optimizer="adagrad"``: row-wise AdaGrad (see :class:`DeviceOnlineMF`); a multi-rank job then reads and
    updates the item rows on their owners (no item cache).
    ``negativeSampling="seen"``: negatives from the items each rank has seen so far, the rule of the reference and
    the host tiers (see :class:`DeviceOnlineMF`); the registry of seen items carries over from epoch to epoch.
    ``None`` or ``"uniform"``: uniform over the whole item range."""
    if updateOutput and loss != "pointwise":
        raise ValueError(f"updateOutput (the per-update output ring) is not supported with loss={loss!r}")
    recs = None
    if numUsers is None or numItems is None:
        recs = list(src.collect() if hasattr(src, "collect") else src)
        numUsers = 1 + max((r.user for r in recs), default=0)
        numItems = 1 + max((r.item for r in recs), default=0)
        src = recs
        numUsers, numItems = _agree_max(numUsers, numItems, group)
    # pullLimit: None or 0 = as many row slots in flight as the GPU holds; any positive value bounds the
    # rows in flight on the device (the reference's 1600 default is a JVM-queue bound -- pass it
    # explicitly if that is what is wanted)
    model = DeviceOnlineMF(numUsers, numItems, numFactors, rangeMin, rangeMax, learningRate,
                           negativeSampleRate, pull_limit=int(pullLimit or 0),
                           group=group, seed=seed, err_mode=ERR_PLAIN if plain_residual else ERR_SIGMOID,
                           track_touched=True,
                           user_memory=min(int(userMemory), 256) if negativeSampleRate > 0 else 0,
                           loss=loss, regularization=regularization, optimizer=optimizer,
                           item_cache=False if optimizer == "adagrad" else None,
                           negative_sampling=negativeSampling or "uniform", margin=margin)
    ring, updates = None, []
    if updateOutput:
        from ...runtime.output_ring import OutputRing

        cap = max(1 << 16, 2 * batch_size * (1 + negativeSampleRate))
        ring = OutputRing(numFactors, model.cuda_device, ring_capacity=4 * cap, staging_capacity=cap,
                          every=int(updateOutput), flush_count=outputFlushCount, flush_interval_ms=outputFlushMs)
        model.output_ring = ring
    seen = set()
    data = list(_batches(src, batch_size))
    for b in data:
        if len(b) == 3:
            seen.update(b[0].tolist())
    for _ in range(max(1, epochs)):
        for _loss in model.fit_stream(iter(data)):
            if ring is not None:
                updates.extend(ring.records())
    model.check_finite()
    model.barrier()
    if ring is not None:
        ring.flush()
        torch.cuda.synchronize(model.cuda_device)
        updates.extend(ring.records())
        res = _result(model, set())               # item shard dump only; user vectors came as the update stream
        rs = ResultStream(updates + [r for r in res.collect() if r.is_right])
        rs.model, rs.output_ring = model, ring
        return rs
    return _result(model, seen if seen else None)


def ps_offline_mf_device(src, iterations=10, **kw) -> ResultStream:
    """Multi-epoch variant: the finite stream is buffered once and replayed ``iterations`` times
    (PSOfflineMatrixFactorizationWorker.scala:97-128)."""
    return ps_online_mf_device(src, epochs=iterations, **kw)


# ---------------------------------------------------------------------------------------------------
# psTopKGenerator(..., backend="device") / psOnlineLearnerAndGenerator(..., backend="device")
# ---------------------------------------------------------------------------------------------------
class _ListWithModel(list):
    """A plain result list (like the host tier returns) that also carries the trained model."""

    model = None


def _seen_filter(rows, K: int, memory: int):
    """The sequential part of ``CollectTopKFromEachWorker`` (utils/CollectTopKFromEachWorker.scala:41-56):
    drop items in the user's recent set (bounded by ``memory``; -1 = unbounded), keep ``K``, then remember
    the rated item.  ``rows``: iterable of ``(user, item, ts, [(score, itemId), ...])`` in stream order."""
    from collections import deque

    seen, order, out = {}, {}, []
    for user, item, ts, cand in rows:
        s = seen.setdefault(user, set())
        out.append((user, item, ts, [c for c in cand if c[1] not in s][:K]))
        s.add(item)
        q = order.setdefault(user, deque())
        q.append(item)
        if memory > -1 and len(q) > memory:
            s.discard(q.popleft())
    return out


class _SeenWindow:
    """The per-user recent-item state of :func:`_seen_filter`, kept across micro-batches so the device
    top-K can exclude the seen items exactly instead of over-fetching and filtering afterwards.  Same
    ``(set, deque)`` bookkeeping, including its quirk: an item rated twice inside the window leaves the
    set when its older copy leaves the window."""

    def __init__(self, memory: int):
        self.memory = int(memory)
        self.seen, self.order = {}, {}

    def exclusions(self, users, items):
        """For a micro-batch ``(users, items)`` in stream order: the items each rating's list must not
        contain (the user's set *before* that rating, so earlier ratings of the same batch count), as a
        CSR ``(offsets int64 [n + 1], item ids int64)`` of numpy arrays; then advance the state past the
        batch.  Each set is copied by numpy, O(|set|) per rating without a per-item Python loop."""
        import numpy as np
        from collections import deque

        lens = np.zeros(len(users) + 1, dtype=np.int64)
        parts = []
        for j, (user, item) in enumerate(zip(users, items)):
            s = self.seen.setdefault(user, set())
            if s:
                parts.append(np.fromiter(s, dtype=np.int64, count=len(s)))
                lens[j + 1] = len(s)
            s.add(item)
            q = self.order.setdefault(user, deque())
            q.append(item)
            if self.memory > -1 and len(q) > self.memory:
                s.discard(q.popleft())
        ids = np.concatenate(parts) if parts else np.zeros(0, dtype=np.int64)
        return np.cumsum(lens), ids

    def device_exclusions(self, users, items, dev):
        """:meth:`exclusions` as device tensors, or ``None`` when no rating of the batch excludes anything."""
        off, ids = self.exclusions(users, items)
        if ids.size == 0:
            return None
        return torch.from_numpy(off).to(dev), torch.from_numpy(ids).to(dev)


def ps_topk_generator_device(src, model, K: int = 100, workerK: int = 75, userMemory: int = 0,
                             batch_size: int = 4096, group=None, sort_by_length: bool = True):
    """Top-K serving over a pre-trained model on the device tier (capability of ``psTopKGenerator``,
    PSTopKGenerator.scala:47-107): the user vectors of ``model`` are loaded into a sharded PS table, the
    item vectors stay with this worker, every query is scored on the wgmma kernel (length-sorted item
    table = the LEMP LENGTH bound) and the per-worker lists are merged.  ``model`` has the reference's
    orientation: ``Left((itemId, (len, vec)))`` / ``Right((userId, (len, vec)))``.  In a multi-rank job
    every rank passes its own part of the model and the *same* query stream.  Unknown users get an empty
    list (the reference's ``invalidParam``).  Returns ``[(itemId, timestamp, [(score, itemId)])]``.
    Vectors of up to 511 factors: the user table carries one extra "loaded" column and the scoring
    kernel takes rows of at most 512 floats."""
    import numpy as np
    import torch.distributed as dist

    from ...store.sharded_table import ShardedTable
    from .device_topk import DistributedTopK

    dev = torch.device("cuda", torch.cuda.current_device())
    entries = list(model.collect() if hasattr(model, "collect") else model)
    items = [(e.value[0], np.asarray(e.value[1][1], dtype=np.float32)) for e in entries if e.is_left]
    users = [(e.value[0], np.asarray(e.value[1][1], dtype=np.float32)) for e in entries if not e.is_left]
    k = len(items[0][1]) if items else len(users[0][1])
    n_users = 1 + max([u for u, _ in users], default=0)
    ready = dist.is_available() and dist.is_initialized()
    if ready:
        t = torch.tensor([n_users, k], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
        n_users, k = int(t[0]), int(t[1])
    # one extra column flags "this user was loaded": item rows carry 0 there, so scores are unchanged
    table = ShardedTable(n_users, k + 1, group=group, init="zeros")
    if users:
        uid = torch.tensor([u for u, _ in users], dtype=torch.int64, device=dev)
        uvec = torch.zeros((len(users), k + 1), dtype=torch.float32, device=dev)
        uvec[:, :k] = torch.from_numpy(np.stack([v for _, v in users])).to(dev)
        uvec[:, k] = 1.0
        table.load(uid, uvec)
    table.barrier()
    local = torch.zeros((max(len(items), 1), table.stride), dtype=torch.float32, device=dev)
    if items:
        local[: len(items), :k] = torch.from_numpy(np.stack([v for _, v in items])).to(dev)
        item_ids = torch.tensor([i for i, _ in items], dtype=torch.int64, device=dev)
    else:
        item_ids = torch.full((1,), -1, dtype=torch.int64, device=dev)
    serving = DistributedTopK(table, local, item_ids, group=group)
    if sort_by_length and len(items) >= 2048:
        from .device_topk import DeviceTopK

        serving.local = DeviceTopK(local, sort_by_length=True)
    ratings = list(src.collect() if hasattr(src, "collect") else src)
    window = _SeenWindow(userMemory) if userMemory != 0 else None    # seen items are excluded on the device
    rows = []
    for a in range(0, len(ratings), batch_size):
        chunk = ratings[a:a + batch_size]
        q = torch.tensor([min(max(r.user, 0), n_users - 1) for r in chunk], dtype=torch.int64, device=dev)
        known = (table.pull(q)[:, k] == 1.0).cpu().tolist()
        exclude = None if window is None else \
            window.device_exclusions([r.user for r in chunk], [r.item for r in chunk], dev)
        sc, ids = serving.topk(q, K, workerK=max(workerK or K, K), exclude=exclude)
        sc, ids = sc.cpu().tolist(), ids.cpu().tolist()
        for j, r in enumerate(chunk):
            ok = known[j] and 0 <= r.user < n_users
            cand = [(s, i) for s, i in zip(sc[j], ids[j]) if i >= 0 and s > -1.0e38] if ok else []
            rows.append((r.item, r.getEventTime(), cand))
    table.close()
    return rows


class _LearnerModel:
    """The model the learner+generator leaves behind: user vectors on the PS table, this rank's item rows."""

    def __init__(self, users, items, world, rank, k):
        self.users, self.items, self.world, self.rank, self.k = users, items, world, rank, k

    def predict(self, users: torch.Tensor, items: torch.Tensor) -> torch.Tensor:
        """u.v for pairs whose ITEM is owned by this rank (user rows are pulled from the PS)."""
        rows = self.items[(items.to(torch.int64) // self.world)].contiguous()
        return self.users.pull_dot(users, rows)

    def close(self) -> None:
        self.users.close()


def ps_online_learner_and_generator_device(src, numFactors=10, rangeMin=-0.001, rangeMax=0.001,
                                           learningRate=0.01, negativeSampleRate=0, userMemory=65535,
                                           K=100, workerK=None, pullLimit=0, seed=0, plain_residual=False,
                                           numUsers: Optional[int] = None, numItems: Optional[int] = None,
                                           batch_size: int = 4096, group=None, loss: str = "pointwise",
                                           regularization: float = 0.0, margin: Optional[float] = None):
    """Online MF plus a top-K list for every incoming rating, computed BEFORE the model sees that rating
    (prequential evaluation; ``psOnlineLearnerAndGenerator``,
    PSOnlineMatrixFactorizationAndTopKGenerator.scala:51-101) on the device tier, any number of ranks.

    Roles as in the reference: **user vectors on the parameter server** (a sharded table), **item
    vectors on the workers** (rank ``item % N`` owns the item).  Every rank is handed the same rating
    stream (the reference broadcasts each rating to all workers, ``:84-101``).  Per micro-batch:

    1. every rank scores the batch's users -- pulled from the PS by the wgmma kernel's A-gather --
       against ITS item partition (``fps_topk_mma``) and keeps ``workerK`` candidates;
    2. the partial lists travel to the merge rank as one-sided stores (:class:`P2PGather`) and are
       merged by ``fps_row_topk`` (``CollectTopKFromEachWorker.scala:41-56``); the user's last
       ``userMemory`` items are excluded exactly inside the device top-K (per-query exclusion lists);
    3. the OWNER of each rated item trains: its local item row is updated in place and the user delta is
       pushed to the PS (``...AndTopKGeneratorWorker.scala:128-164``) -- the fused MF kernel with the
       roles swapped (worker-local rows = items, PS rows = users), negatives drawn from the owner's items.

    ``loss="warp"``: the owner examines its ``[n, negativeSampleRate]`` candidate draws in order until one is
    within ``margin`` (default 1.0) of the positive; the rank estimate uses ``numItems`` (the owner's items are a
    uniform subset of all items, so ``(numItems - 1) / n`` still estimates the global rank).

    Prequential at micro-batch granularity (``batch_size``; 1 reproduces the per-rating order).  The
    result is a pure function of the stream and the seed, whatever the number of ranks (init is Philox
    by id).  Rank 0 returns ``[(userId, itemId, timestamp, [(score, itemId)])]`` (other ranks ``[]``);
    the model is in ``.users`` (the PS table) / ``.items`` (local partition).  ``numFactors`` may be
    up to 512 (the widest row of the scoring kernel)."""
    import torch.distributed as dist

    from ...store.sharded_table import ShardedTable
    from .device_topk import DeviceTopK, DistributedTopK

    if loss not in ("pointwise", "bpr", "warp"):
        raise ValueError(f"loss must be 'pointwise', 'bpr' or 'warp', got {loss!r}")
    if loss == "pointwise" and regularization != 0:
        raise ValueError("regularization is only supported with loss='bpr' or loss='warp'")
    if loss != "pointwise" and negativeSampleRate < 1:
        raise ValueError(f"loss={loss!r} needs negativeSampleRate >= 1")
    margin = check_warp(loss, margin, optimizer="sgd", negative_sampling="uniform")
    recs = list(src.collect() if hasattr(src, "collect") else src)
    if numUsers is None:
        numUsers = 1 + max((r.user for r in recs), default=0)
    if numItems is None:
        numItems = 1 + max((r.item for r in recs), default=0)
    numUsers, numItems = _agree_max(numUsers, numItems, group)
    ready = dist.is_available() and dist.is_initialized()
    world = dist.get_world_size(group) if ready else 1
    rank = dist.get_rank(group) if ready else 0
    dev = torch.device("cuda", torch.cuda.current_device())
    users = ShardedTable(numUsers, numFactors, group=group, init="uniform", init_range=(rangeMin, rangeMax),
                         seed=seed * 2 + 2)
    n_local = -(-numItems // world)
    items = torch.empty((n_local, users.stride), dtype=torch.float32, device=dev)
    native.init_rows(items, numFactors, rank, world, native.PART_HASH, n_local, seed * 2 + 1, rangeMin, rangeMax)
    local_ids = torch.arange(n_local, device=dev, dtype=torch.int64) * world + rank
    n_valid = int((local_ids < numItems).sum())
    stats = torch.zeros(STATS_SIZE[loss], dtype=torch.float32, device=dev)
    nan_flag = torch.zeros(1, dtype=torch.int32, device=dev)
    err_mode = ERR_PLAIN if plain_residual else ERR_SIGMOID
    wk = max(workerK or K, K)
    window = _SeenWindow(userMemory) if userMemory != 0 else None    # same state on every rank
    gen = torch.Generator(device=dev).manual_seed(seed * 7919 + 13)
    rows = []
    users.barrier()
    # the scorer reads the item partition in place: the fused kernel's updates are seen by the next batch
    serving = DistributedTopK(users, items[:max(n_valid, 1)], local_ids[:max(n_valid, 1)], group=group)
    for bno, a in enumerate(range(0, len(recs), batch_size)):
        chunk = recs[a:a + batch_size]
        u = torch.tensor([r.user for r in chunk], dtype=torch.int32, device=dev)
        i = torch.tensor([r.item for r in chunk], dtype=torch.int32, device=dev)
        rt = torch.tensor([r.rating for r in chunk], dtype=torch.float32, device=dev)
        # 1 + 2: local top-workerK of every query on this rank's items, gathered + merged on rank 0
        exclude = None if window is None else \
            window.device_exclusions([r.user for r in chunk], [r.item for r in chunk], dev)
        sc, ids = serving.topk(u.long(), K, workerK=wk, dst=0, exclude=exclude)
        if sc is not None:
            sc, ids = sc.cpu().tolist(), ids.cpu().tolist()
            for j, r in enumerate(chunk):
                rows.append((r.user, r.item, r.getEventTime(),
                             [(s_, i_) for s_, i_ in zip(sc[j], ids[j]) if i_ >= 0 and s_ > -1.0e38]))
        users.barrier()                      # every rank has read the pre-update user vectors
        # 3: owner-only item update + pushed user delta (fused kernel, roles swapped)
        mine = (i % world) == rank
        ti = torch.where(mine, i, torch.full_like(i, -1))
        tu, tr = u, rt
        if negativeSampleRate > 0 and n_valid > 0:
            # negatives for the owned positives, drawn from the owner's items (reference: <= 32 retries to
            # avoid the positive; here a colliding draw is shifted to the next local item)
            neg_slot = torch.randint(0, n_valid, (len(chunk), negativeSampleRate), generator=gen, device=dev)
            neg_item = (neg_slot * world + rank).to(torch.int32)
            clash = neg_item == i[:, None]
            neg_item = torch.where(clash, ((neg_slot + 1) % n_valid * world + rank).to(torch.int32), neg_item)
            neg_item = torch.where(mine[:, None], neg_item, torch.full_like(neg_item, -1))
            if loss == "pointwise":
                ti = torch.cat([ti, neg_item.reshape(-1)])
                tu = torch.cat([u, u[:, None].expand(-1, negativeSampleRate).reshape(-1)])
                tr = torch.cat([rt, torch.zeros(neg_item.numel(), device=dev)])
        if loss == "bpr":
            if n_valid > 0:
                # anchors = users on the PS, candidates = this rank's item rows (slot = item // world)
                native.mf_bpr_fused(u, ti, rt, users.table_c, items, learningRate, regularization,
                                    negatives=neg_item.contiguous(), cand_div=world, stats=stats,
                                    nan_flag=nan_flag, max_inflight_rows=int(pullLimit or 0))
        elif loss == "warp":
            if n_valid > 0:
                native.mf_warp_fused(u, ti, rt, users.table_c, items, learningRate, regularization, margin=margin,
                                     rank_items=numItems, negatives=neg_item.contiguous(), cand_div=world,
                                     stats=stats, nan_flag=nan_flag, max_inflight_rows=int(pullLimit or 0))
        else:
            native.mf_sgd_fused(ti.contiguous(), tu.contiguous(), tr.contiguous(), items, world, users.table_c,
                                learningRate, err_mode=err_mode, stats=stats, nan_flag=nan_flag,
                                max_inflight_rows=int(pullLimit or 0), kernel="reg")
        users.barrier()                      # pushes of this micro-batch are in the PS before the next pulls
    if int(nan_flag.item()) != 0:
        from ...errors import FactorIsNotANumberException

        raise FactorIsNotANumberException("non-finite SGD update")
    out = _ListWithModel(rows if rank == 0 else [])
    out.users, out.items, out.item_ids, out.n_items = users, items, local_ids, n_valid
    out.model = _LearnerModel(users, items, world, rank, numFactors)
    if getattr(serving, "_p2p_gather", None) is not None:
        serving._p2p_gather.close()
    return out
