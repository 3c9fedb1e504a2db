"""Offline (multi-epoch) SGD matrix factorisation -- ``psOfflineMF``.

Reference: M/matrix/factorization/PSOfflineMatrixFactorization.scala:46-107 and
workers/PSOfflineMatrixFactorizationWorker.scala:28-151: buffer all ratings (+negatives) until the
EOF of the finite input, then a background thread issues the pulls for ``iterations`` epochs while
the operator thread handles the answers.  ``shuffle=True`` actually reshuffles between epochs (the
reference discards the result of ``Random.shuffle``, SURVEY §7.4).
"""
from __future__ import annotations

import random
import threading
from collections import deque
from typing import Dict, List, Optional

import numpy as np

from ...api import CtorFork, WorkerLogic
from ...limiter import addPullLimiter
from ...runtime.stream import as_stream
from ...runtime.transform import transform
from ...utils.eof import EOF, with_eof
from .common import Rating, RangedRandomFactorInitializerDescriptor, SGDUpdater, require_pointwise, vectorSum
from .online import NegativeSampler


class PSOfflineMatrixFactorizationWorker(CtorFork, WorkerLogic):
    def __init__(self, numFactors, rangeMin, rangeMax, learningRate, negativeSampleRate, userMemory,
                 iterations, seed: Optional[int] = None, plain_residual: bool = False,
                 shuffle: bool = False):
        self.factorInitDesc = RangedRandomFactorInitializerDescriptor(numFactors, rangeMin, rangeMax, seed)
        self._init = None
        self.factorUpdate = SGDUpdater(learningRate, plain_residual)
        self.iterations = iterations
        self.shuffle = shuffle
        self.rbs: List[List[Rating]] = []
        self.userVectors: Dict[int, np.ndarray] = {}
        self.ratingBuffer: Dict[int, deque] = {}
        self.sampler = NegativeSampler(userMemory, negativeSampleRate, seed)
        self.workerThread: Optional[threading.Thread] = None
        self._lock = threading.Lock()
        self._rnd = random.Random(seed)
        self._seed_args = (numFactors, rangeMin, rangeMax, userMemory, negativeSampleRate, seed)

    def open(self):
        """Per-subtask random streams for seeded runs (see PSOnlineMatrixFactorizationWorker.open)."""
        numFactors, rangeMin, rangeMax, userMemory, rate, seed = self._seed_args
        idx = getattr(self, "subtaskIndex", 0)
        if seed is not None and idx:
            sub = (int(seed) * 1000003 + 7919 * idx) & 0x7FFFFFFF
            self.factorInitDesc = RangedRandomFactorInitializerDescriptor(numFactors, rangeMin, rangeMax, sub)
            self._init = None
            self.sampler = NegativeSampler(userMemory, rate, sub + 1)
            self._rnd = random.Random(sub + 2)

    def onRecv(self, value, ps):
        if isinstance(value, EOF):
            def run():
                for _ in range(self.iterations):
                    if self.shuffle:
                        self._rnd.shuffle(self.rbs)
                    for rs in self.rbs:
                        for rating in rs:
                            with self._lock:
                                self.ratingBuffer.setdefault(rating.item, deque()).append(
                                    (rating.user, rating.rating))
                            ps.pull(rating.item)

            self.workerThread = threading.Thread(target=run, daemon=True, name="fps-offline-mf")
            self.workerThread.start()
            return
        if self.workerThread is not None:
            raise RuntimeError("Should not have started worker thread while waiting for further elements.")
        rating: Rating = value
        self.sampler.register_item(rating.item)
        seen = self.sampler.observe(rating.user, rating.item)
        rs = [Rating(rating.user, neg, 0.0) for neg in self.sampler.sample(seen)]
        rs.append(rating)
        self.rbs.append(rs)

    def onPullRecv(self, item, itemVec, ps):
        with self._lock:
            user, rating = self.ratingBuffer[item].popleft()
        userVec = self.userVectors.get(user)
        if userVec is None:
            if self._init is None:
                self._init = self.factorInitDesc.open()
            userVec = self._init.nextFactor(user)
        du, dv = self.factorUpdate.delta(rating, userVec, itemVec)
        self.userVectors[user] = vectorSum(userVec, du)
        ps.output((user, self.userVectors[user]))
        ps.push(item, dv)

    def close(self):
        if self.workerThread is not None:
            self.workerThread.join(timeout=30)


def psOfflineMF(src, numFactors: int = 10, rangeMin: float = -0.01, rangeMax: float = 0.01,
                learningRate: float = 0.01, negativeSampleRate: int = 0, userMemory: int = 128,
                iterations: int = 10, pullLimit: Optional[int] = None, workerParallelism: int = 1,
                psParallelism: int = 1, iterationWaitTime: float = 10000, seed: Optional[int] = None,
                plain_residual: bool = False, shuffle: bool = False, backend: str = "local",
                **device_kw):
    hostPullLimit = 1600 if pullLimit is None else pullLimit   # reference default (JVM queue bound)
    require_pointwise(backend, device_kw)
    if backend == "native":
        from .native_api import ps_mf_native

        return ps_mf_native(src, numFactors, rangeMin, rangeMax, learningRate, hostPullLimit, workerParallelism,
                            psParallelism, seed or 0, plain_residual, epochs=iterations,
                            negativeSampleRate=negativeSampleRate, userMemory=userMemory)
    if backend == "device":
        from .device_api import ps_offline_mf_device

        return ps_offline_mf_device(src, numFactors=numFactors, rangeMin=rangeMin, rangeMax=rangeMax,
                                    learningRate=learningRate, negativeSampleRate=negativeSampleRate,
                                    iterations=iterations, pullLimit=pullLimit, seed=seed or 0,
                                    userMemory=userMemory, plain_residual=plain_residual, **device_kw)
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

    ratings = with_eof(src, lambda key, n: key % n, lambda r: r.user)
    worker = addPullLimiter(
        PSOfflineMatrixFactorizationWorker(numFactors, rangeMin, rangeMax, learningRate,
                                           negativeSampleRate, userMemory, iterations, seed,
                                           plain_residual, shuffle), hostPullLimit)
    return transform(ratings, worker, paramInit, vectorSum, workerParallelism, psParallelism,
                     iterationWaitTime)


ps_offline_mf = psOfflineMF
