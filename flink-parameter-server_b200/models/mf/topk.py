"""Top-K recommendation on the parameter server (host tier).

* :func:`psTopKGenerator` -- serving-only top-K over a pre-trained model loaded with the double
  model load: item vectors -> workers, user vectors -> PS
  (M/matrix/factorization/PSTopKGenerator.scala:47-107, workers/PSTopKGeneratorWorker.scala:13-120).
* :func:`psOnlineLearnerAndGenerator` -- online MF *plus* a top-K list for every incoming rating;
  roles flipped: user vectors (with cached length) on the PS, item vectors on the workers
  (PSOnlineMatrixFactorizationAndTopKGenerator.scala:51-101, ...AndTopKGeneratorWorker.scala:28-195).
* :class:`CollectTopKFromEachWorker` -- parallelism-1 merge of the per-worker partial lists with the
  user's recent-items filter (utils/CollectTopKFromEachWorker.scala:24-75).

Every rating is broadcast to all workers (``RichRating(base, targetWorker, ratingId)``); worker w
scans its local items bucket by bucket in descending length order with LEMP pruning.
Device tier: models/mf/device_topk.py (pull user vectors + wgmma GEMM + top-K select).
"""
from __future__ import annotations

import math
import random
from collections import deque
from typing import Any, Dict, Iterable, List, Optional, Tuple

import numpy as np

from ...api import CtorFork, Left, Right, WorkerLogic
from ...limiter import addPullLimiter
from ...parallel.partitioner import stable_hash
from ...runtime.stream import DataStream, as_stream
from ...runtime.transform import transform, transformWithDoubleModelLoad
from ...server.logics import SimplePSLogic
from .common import (IDGenerator, Partitioner, RangedRandomFactorInitializerDescriptor, Rating, require_pointwise,
                     RichRating, SGDUpdater, TopKQueue, attachLength, vectorSum)
from .pruning import (COORD, INCR, LC, LENGTH, LI, LEMPPruningStrategy, coordPruning, focus_coordinate,
                      focus_set, incrPruning, lengthPruning)

INVALID_PARAM = (-1.0, np.zeros(0))


class BaseMFWorkerLogic(WorkerLogic):
    """``WorkerLogic`` + worker-local ``model`` + ``updateModel`` hook used by the double model load
    (workers/BaseMFWorkerLogic.scala:8-14)."""

    def __init__(self):
        self.model: Dict[int, Tuple[float, np.ndarray]] = {}

    def updateModel(self, id, param) -> None:
        self.model[id] = param


class _SortedItems:
    """Item ids ordered by vector length, descending (the reference's ``TreeSet[(length, id)]``)."""

    def __init__(self):
        self.length: Dict[int, float] = {}
        self._sorted: Optional[List[Tuple[float, int]]] = None

    def put(self, id: int, length: float) -> None:
        self.length[id] = length
        self._sorted = None

    def buckets(self, size: int):
        if self._sorted is None:
            self._sorted = sorted(((l, i) for i, l in self.length.items()), reverse=True)
        s = self._sorted
        for a in range(0, len(s), size):
            yield s[a:a + size]


def lemp_topk(user: Tuple[float, np.ndarray], items: _SortedItems, model, workerK: int,
              bucketSize: int, pruning: LEMPPruningStrategy) -> TopKQueue:
    """Bucketed MIPS with early stop ``maxLen_bucket * ||u|| <= theta`` and per-bucket pruning
    (PSTopKGeneratorWorker.scala:49-113)."""
    ulen, uvec = user
    topK = TopKQueue(workerK)
    if ulen <= 0 or uvec.size == 0:
        return topK
    focus = focus_coordinate(uvec)
    n_focus = pruning.numFocusCoordinates if isinstance(pruning, (INCR, LI)) else 0
    fset = focus_set(uvec, n_focus)
    for bucket in items.buckets(bucketSize):
        head_len = bucket[0][0]
        full = len(topK) >= workerK
        if full and head_len * ulen <= topK.min_score():
            break
        theta = topK.min_score() if full else -math.inf
        cand = [(i, model[i]) for _, i in bucket]
        if full and theta > 0:
            theta_b_q = theta / (head_len * ulen) if head_len * ulen > 0 else math.inf
            use_length = isinstance(pruning, LENGTH)
            if isinstance(pruning, (LC, LI)):
                use_length = head_len > bucket[-1][0] * pruning.algorithmSwitchThreshold
            if use_length:
                f = lengthPruning(theta / ulen)
            elif isinstance(pruning, (COORD, LC)):
                f = coordPruning(focus, user, theta_b_q)
            else:
                f = incrPruning(fset, user, theta)
            cand = [c for c in cand if f(c)]
        for i, (_, vec) in cand:
            topK.push(float(np.dot(uvec, vec)), i)
    return topK


class PSTopKGeneratorWorker(BaseMFWorkerLogic):
    def __init__(self, workerK: int, bucketSize: int, workerParallelism: int,
                 pruning: LEMPPruningStrategy):
        super().__init__()
        self.workerK, self.bucketSize, self.wP, self.pruning = workerK, bucketSize, workerParallelism, pruning
        self.items = _SortedItems()
        self.ratingBuffer: Dict[int, deque] = {}

    def onRecv(self, data: RichRating, ps):
        self.ratingBuffer.setdefault(data.base.user, deque()).append(data)
        ps.pull(data.base.user)

    def onPullRecv(self, paramId, userAndLen, ps):
        rate = self.ratingBuffer[paramId].popleft()
        if userAndLen[0] == -1:  # unknown user -> empty list (PSTopKGenerator.scala:62,74-76)
            ps.output((rate, []))
            return
        topK = lemp_topk(userAndLen, self.items, self.model, self.workerK, self.bucketSize, self.pruning)
        ps.output((rate, topK.sorted_desc()))

    def updateModel(self, id, param):
        self.model[id] = param
        self.items.put(id, param[0])


class CollectTopKFromEachWorker:
    """Merge ``workerParallelism`` partial lists per ``ratingId``; drop items in the user's recent
    set (bounded by ``memory``; -1 = unbounded); emit ``(user, item, time, topK)``."""

    def __init__(self, K: int, memory: int, workerParallelism: int):
        self.K, self.memory, self.wP = K, memory, workerParallelism
        self.outputs: Dict[int, Dict[int, list]] = {}
        self.seenSet: Dict[int, set] = {}
        self.seenList: Dict[int, deque] = {}

    def flatMap(self, value) -> List[Tuple[int, int, int, List[Tuple[float, int]]]]:
        if not value.is_left:
            return []
        rich, partial = value.value
        allTopK = self.outputs.setdefault(rich.ratingId, {})
        allTopK[rich.targetWorker] = partial
        if len(allTopK) < self.wP:
            return []
        base = rich.base
        seen = self.seenSet.setdefault(base.user, set())
        merged = [x for p in allTopK.values() for x in p if x[1] not in seen]
        merged.sort(key=lambda t: -t[0])
        del self.outputs[rich.ratingId]
        seen.add(base.item)
        sl = self.seenList.setdefault(base.user, deque())
        sl.append(base.item)
        if self.memory > -1 and len(sl) > self.memory:
            seen.discard(sl.popleft())
        return [(base.user, base.item, base.getEventTime(), merged[: self.K])]

    def run(self, results: Iterable[Any]):
        out = []
        for r in results:
            out.extend(self.flatMap(r))
        return out


def _broadcast_ratings(src, workerParallelism: int) -> DataStream:
    def enrich(r: Rating):
        rid = IDGenerator.next()
        return [r.enrich(i, rid) for i in range(workerParallelism)]

    return as_stream(src).flat_map(enrich).partition_custom(lambda k, n: k % n, lambda x: x.targetWorker)


def psTopKGenerator(src, model, numFactors: int = 10, rangeMin: float = -0.01, rangeMax: float = 0.01,
                    userMemory: int = 0, K: int = 100, workerK: int = 75, bucketSize: int = 100,
                    pruningAlgorithm: LEMPPruningStrategy = COORD(), pullLimit: int = 1600,
                    workerParallelism: int = 4, psParallelism: int = 4, iterationWaitTime: float = 10000,
                    backend: str = "local", **device_kw):
    """``model``: stream of ``Left((itemId, (len, vec)))`` (to workers) / ``Right((userId, (len, vec)))``
    (to the PS) -- note the reference's Either orientation is kept.  Returns
    ``[(itemId, timestamp, [(score, itemId)])]`` per rating.  ``backend="device"``: wgmma scoring
    against a length-sorted item table (``models/mf/device_api.py::ps_topk_generator_device``)."""
    if backend == "device":
        from .device_api import ps_topk_generator_device

        return ps_topk_generator_device(src, model, K=K, workerK=workerK, userMemory=userMemory, **device_kw)
    worker = addPullLimiter(PSTopKGeneratorWorker(workerK, bucketSize, workerParallelism, pruningAlgorithm),
                            pullLimit)
    psLogic = SimplePSLogic(lambda _i: INVALID_PARAM, lambda _old, new: new)
    # transformWithDoubleModelLoad expects Left = server parameter, Right = worker-local entry
    flipped = as_stream(model).map(lambda e: Right(e.value) if e.is_left else Left(e.value))
    part = Partitioner(psParallelism)
    res = transformWithDoubleModelLoad(flipped)(
        _broadcast_ratings(src, workerParallelism), worker, psLogic, part.workerToPSPartitioner,
        part.psToWorkerPartitioner, workerParallelism, psParallelism, iterationWaitTime,
        workerModelPartitioner=lambda itemId, n: stable_hash(itemId) % n)
    merged = CollectTopKFromEachWorker(K, userMemory, workerParallelism).run(res.collect())
    return [(item, ts, topK) for (_u, item, ts, topK) in merged]


class PSOnlineMatrixFactorizationAndTopKGeneratorWorker(CtorFork, BaseMFWorkerLogic):
    def __init__(self, negativeSampleRate, userMemory, workerK, bucketSize, pruningAlgorithm,
                 workerParallelism, factorInitDesc, factorUpdate, seed: Optional[int] = None):
        BaseMFWorkerLogic.__init__(self)
        self.neg, self.userMemory, self.workerK, self.bucketSize = negativeSampleRate, userMemory, workerK, bucketSize
        self.pruning, self.wP = pruningAlgorithm, workerParallelism
        self.factorInitDesc, self.factorUpdate = factorInitDesc, factorUpdate
        self._init = None
        self.items = _SortedItems()
        self.itemIdsBuffer: List[int] = []
        self.ratingBuffer: Dict[int, deque] = {}
        self.seenSet: Dict[int, set] = {}
        self.seenList: Dict[int, deque] = {}
        self.workerId = -1
        self.rnd = random.Random(seed)

    def onRecv(self, data: RichRating, ps):
        if self.workerId == -1:
            self.workerId = data.targetWorker
        self.ratingBuffer.setdefault(data.base.user, deque()).append(data)
        ps.pull(data.base.user)

    def _set_item(self, id, param):
        if id not in self.model:
            self.itemIdsBuffer.append(id)
        self.model[id] = param
        self.items.put(id, param[0])

    updateModel = _set_item

    def _initialize(self, id):
        if self._init is None:
            self._init = self.factorInitDesc.open()
        lv = attachLength(self._init.nextFactor(id))
        self._set_item(id, lv)
        return lv

    def onPullRecv(self, paramId, userAndLen, ps):
        rate = self.ratingBuffer[paramId].popleft()
        userVector = userAndLen[1]
        topK = lemp_topk(userAndLen, self.items, self.model, self.workerK, self.bucketSize, self.pruning)
        ps.output((rate, topK.sorted_desc()))
        base = rate.base
        if stable_hash(base.item) % self.wP != self.workerId:
            return  # only the owner worker of the item trains on this rating
        seen = self.seenSet.setdefault(base.user, set())
        if base.item not in seen:
            seen.add(base.item)
            sl = self.seenList.setdefault(base.user, deque())
            sl.append(base.item)
            if len(sl) > self.userMemory:
                seen.discard(sl.popleft())
        uDelta = np.zeros_like(userVector)
        for _ in range(min(len(self.model) - len(seen), self.neg)):
            negId = self.itemIdsBuffer[self.rnd.randrange(len(self.itemIdsBuffer))]
            counter = 32
            while counter > 0 and negId in seen:
                negId = self.itemIdsBuffer[self.rnd.randrange(len(self.itemIdsBuffer))]
                counter -= 1
            if counter > 0:
                _, negVec = self.model[negId]
                uu, iDelta = self.factorUpdate.delta(0.0, userVector, negVec)
                uDelta = vectorSum(uDelta, uu)
                self._set_item(negId, attachLength(vectorSum(negVec, iDelta)))
        _, itemVector = self.model.get(base.item) or self._initialize(base.item)
        userDelta, itemDelta = self.factorUpdate.delta(base.rating, userVector, itemVector)
        self._set_item(base.item, attachLength(vectorSum(itemVector, itemDelta)))
        ps.push(paramId, (float("nan"), vectorSum(uDelta, userDelta)))


def psOnlineLearnerAndGenerator(src, numFactors: int = 10, rangeMin: float = -0.001,
                                rangeMax: float = 0.001, learningRate: float = 0.01,
                                negativeSampleRate: int = 0, userMemory: int = 65535, K: int = 100,
                                workerK: int = 75, bucketSize: int = 100,
                                pruningAlgorithm: LEMPPruningStrategy = LI(5, 2.5), pullLimit: Optional[int] = None,
                                workerParallelism: int = 4, psParallelism: int = 4,
                                iterationWaitTime: float = 10000, seed: Optional[int] = None,
                                plain_residual: bool = False, backend: str = "local", **device_kw):
    """Returns ``[(userId, itemId, timestamp, [(score, itemId)])]`` -- one top-K per rating, computed
    BEFORE the model is updated with that rating (prequential evaluation).  ``backend="device"``:
    ``models/mf/device_api.py::ps_online_learner_and_generator_device``."""
    require_pointwise(backend, device_kw)
    if backend == "device":
        from .device_api import ps_online_learner_and_generator_device

        return ps_online_learner_and_generator_device(
            src, numFactors=numFactors, rangeMin=rangeMin, rangeMax=rangeMax, learningRate=learningRate,
            negativeSampleRate=negativeSampleRate, userMemory=userMemory, K=K, pullLimit=pullLimit,
            seed=seed or 0, plain_residual=plain_residual, **device_kw)
    initDesc = RangedRandomFactorInitializerDescriptor(numFactors, rangeMin, rangeMax, seed)
    worker = addPullLimiter(
        PSOnlineMatrixFactorizationAndTopKGeneratorWorker(
            negativeSampleRate, userMemory, workerK, bucketSize, pruningAlgorithm, workerParallelism,
            initDesc, SGDUpdater(learningRate, plain_residual), seed), 500 if pullLimit is None else pullLimit)
    holder = {}

    def init(x):
        if "f" not in holder:
            holder["f"] = RangedRandomFactorInitializerDescriptor(
                numFactors, rangeMin, rangeMax, None if seed is None else seed + 1).open()
        return attachLength(holder["f"].nextFactor(x))

    serverLogic = SimplePSLogic(init, lambda vec, d: attachLength(vectorSum(vec[1], d[1])))
    res = transform(_broadcast_ratings(src, workerParallelism), worker, serverLogic,
                    workerParallelism, psParallelism, iterationWaitTime)
    return CollectTopKFromEachWorker(K, userMemory, workerParallelism).run(res.collect())


ps_top_k_generator = psTopKGenerator
ps_online_learner_and_generator = psOnlineLearnerAndGenerator
