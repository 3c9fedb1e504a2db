"""Online SGD matrix factorisation -- ``psOnlineMF``.

Reference: M/matrix/factorization/PSOnlineMatrixFactorization.scala:39-75 and
workers/PSOnlineMatrixFactorizationWorker.scala:22-90.  Users live on workers
(``user % workerParallelism``), item vectors on the PS (``SimplePSLogic`` with ranged-random init
and ``vectorSum`` update); every rating = pull(item) -> SGD delta -> local user update ->
output((user, vec)) -> push(item, delta).

``backend="local"`` runs the per-record logic on the host tier (exact reference semantics incl.
per-user negative-sampling memory); ``backend="device"`` runs the same algorithm as fused
micro-batch kernels on the GPU (:class:`fps_b200.models.mf.device.DeviceOnlineMF`).

The reference passes ``(negativeSampleRate, userMemory)`` into a ctor declared
``(userMemory, negativeSampleRate)`` (SURVEY §7.4); here the arguments mean what they say.
"""
from __future__ import annotations

import random
from collections import deque
from typing import Dict, Optional

import numpy as np

from ...api import ParameterServerClient, WorkerLogic
from ...limiter import addPullLimiter
from ...runtime.stream import DataStream, ResultStream, as_stream
from ...runtime.transform import transform
from ...server.logics import SimplePSLogic
from .common import (Rating, RangedRandomFactorInitializerDescriptor, SGDUpdater, require_pointwise, vectorSum)


class NegativeSampler:
    """Per-user recent-item memory + uniform sampling over the items seen so far (K5;
    PSOnlineMatrixFactorizationWorker.scala:61-78)."""

    def __init__(self, userMemory: int, negativeSampleRate: int, seed: Optional[int] = None):
        self.userMemory, self.rate = userMemory, negativeSampleRate
        self.rnd = random.Random(seed)
        self.itemIds = []
        self.itemSet = set()
        self.seenSet: Dict[int, set] = {}
        self.seenQueue: Dict[int, deque] = {}

    def observe(self, user: int, item: int):
        ss = self.seenSet.setdefault(user, set())
        sq = self.seenQueue.setdefault(user, deque())
        if len(sq) >= self.userMemory:
            ss.discard(sq.popleft())
        ss.add(item)
        sq.append(item)
        return ss

    def register_item(self, item: int) -> None:
        if item not in self.itemSet:
            self.itemSet.add(item)
            self.itemIds.append(item)

    def sample(self, seen: set):
        out = []
        for _ in range(min(len(self.itemIds) - len(seen), self.rate)):
            r = self.itemIds[self.rnd.randrange(len(self.itemIds))]
            while r in seen:
                r = self.itemIds[self.rnd.randrange(len(self.itemIds))]
            out.append(r)
        return out


class PSOnlineMatrixFactorizationWorker(WorkerLogic):
    def __init__(self, numFactors: int, rangeMin: float, rangeMax: float, learningRate: float,
                 userMemory: int, negativeSampleRate: int, seed: Optional[int] = None,
                 plain_residual: bool = False):
        self._args = (numFactors, rangeMin, rangeMax, userMemory, negativeSampleRate, seed)
        self.factorInitDesc = RangedRandomFactorInitializerDescriptor(numFactors, rangeMin, rangeMax, seed)
        self._init = None
        self.factorUpdate = SGDUpdater(learningRate, plain_residual)
        self.userVectors: Dict[int, np.ndarray] = {}
        self.ratingBuffer: Dict[int, deque] = {}
        self.sampler = NegativeSampler(userMemory, negativeSampleRate, seed)

    def open(self):
        """Seeded runs: every worker subtask gets its OWN random stream (init + negative sampling); the
        engine tells the copy which subtask it is (``subtaskIndex``).  Identical streams would give the n-th
        new user of every worker the same vector and the same negatives."""
        numFactors, rangeMin, rangeMax, userMemory, rate, seed = self._args
        idx = getattr(self, "subtaskIndex", 0)
        if seed is not None and idx:
            sub = (int(seed) * 1000003 + 7919 * idx) & 0x7FFFFFFF
            self.factorInitDesc = RangedRandomFactorInitializerDescriptor(numFactors, rangeMin, rangeMax, sub)
            self._init = None
            self.sampler = NegativeSampler(userMemory, rate, sub + 1)

    def _factor_init(self):
        if self._init is None:
            self._init = self.factorInitDesc.open()
        return self._init

    def onPullRecv(self, paramId, paramValue, ps):
        rating = self.ratingBuffer[paramId].popleft()
        user = self.userVectors.get(rating.user)
        if user is None:
            user = self._factor_init().nextFactor(rating.user)
        userDelta, itemDelta = self.factorUpdate.delta(rating.rating, user, paramValue)
        self.userVectors[rating.user] = vectorSum(user, userDelta)
        ps.output((rating.user, self.userVectors[rating.user]))
        ps.push(paramId, itemDelta)

    def onRecv(self, data: Rating, ps):
        seen = self.sampler.observe(data.user, data.item)
        for neg in self.sampler.sample(seen):
            self.ratingBuffer[neg].append(Rating(data.user, neg, 0.0, data.timestamp))
            ps.pull(neg)
        if data.item not in self.ratingBuffer:
            self.sampler.register_item(data.item)
            self.ratingBuffer[data.item] = deque()
        self.ratingBuffer[data.item].append(data)
        ps.pull(data.item)


def psOnlineMF(src, numFactors: int = 10, rangeMin: float = -0.01, rangeMax: float = 0.01,
               learningRate: float = 0.01, negativeSampleRate: int = 0, userMemory: int = 128,
               pullLimit: Optional[int] = None, workerParallelism: int = 1, psParallelism: int = 1,
               iterationWaitTime: float = 10000, seed: Optional[int] = None,
               plain_residual: bool = False, backend: str = "local", **device_kw):
    """Returns the stream of ``Left((userId, userVector))`` / ``Right((itemId, itemVector))``.
    ``backend="local"``: arbitrary-logic Python engine; ``"native"``: the same protocol on the C++ host
    engine (threads + SPSC rings, ``ops/csrc/fps_host.cpp``); ``"device"``: fused GPU kernels."""
    hostPullLimit = 1600 if pullLimit is None else pullLimit   # reference default (JVM queue bound)
    require_pointwise(backend, device_kw)
    if backend == "native":
        from .native_api import ps_mf_native

        return ps_mf_native(src, numFactors, rangeMin, rangeMax, learningRate, hostPullLimit, workerParallelism,
                            psParallelism, seed or 0, plain_residual, epochs=1,
                            negativeSampleRate=negativeSampleRate, userMemory=userMemory)
    if backend == "device":
        from .device_api import ps_online_mf_device

        return ps_online_mf_device(src, numFactors=numFactors, rangeMin=rangeMin, rangeMax=rangeMax,
                                   learningRate=learningRate, negativeSampleRate=negativeSampleRate,
                                   pullLimit=pullLimit, seed=seed or 0, userMemory=userMemory,
                                   plain_residual=plain_residual, **device_kw)
    initDesc = RangedRandomFactorInitializerDescriptor(numFactors, rangeMin, rangeMax,
                                                       None if seed is None else seed + 1)
    holder = {}

    def paramInit(i):
        if seed is not None:
            # a pure function of (seed, id): deterministic whatever the interleaving of the PS shard
            # threads, which all share this closure (the device and native tiers do the same with Philox)
            rnd = random.Random((int(seed) + 1) * 1000003 + int(i))
            return np.array([rangeMin + (rangeMax - rangeMin) * rnd.random() for _ in range(numFactors)])
        if "f" not in holder:
            holder["f"] = initDesc.open()
        return holder["f"].nextFactor(i)

    workerLogic = addPullLimiter(
        PSOnlineMatrixFactorizationWorker(numFactors, rangeMin, rangeMax, learningRate, userMemory,
                                          negativeSampleRate, seed, plain_residual), hostPullLimit)
    serverLogic = SimplePSLogic(paramInit, vectorSum)
    partitioned = as_stream(src).partition_custom(lambda key, n: key % n, lambda r: r.user)
    return transform(partitioned, workerLogic, serverLogic, workerParallelism, psParallelism,
                     iterationWaitTime)


ps_online_mf = psOnlineMF
