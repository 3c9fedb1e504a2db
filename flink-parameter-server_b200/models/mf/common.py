"""Shared matrix-factorisation building blocks (host tier).

Capabilities of M/matrix/factorization/{factors,utils}/: vector helpers, ``Rating`` / ``RichRating``,
factor initialisers (incl. the descriptor/``open()`` factory pattern), ``SGDUpdater``, id generator,
top-K queue and the partitioner pair.  Vectors are ``numpy.float64`` arrays (the reference's
``Array[Double]``); the device tier uses fp32 rows in HBM.
"""
from __future__ import annotations

import heapq
import itertools
import math
import random
import threading
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np

from ...parallel.partitioner import stable_hash
from ...utils.input_source import EventWithTimestamp

Vector = np.ndarray
UserId = int
ItemId = int


from ...errors import FactorIsNotANumberException  # noqa: E402,F401  (re-exported; Vector.scala:78-80)


def vectorLengthSqr(v: Vector) -> float:
    return float(np.dot(v, v))


def dotProduct(u: Vector, v: Vector) -> float:
    return float(np.dot(u, v))


def vectorSum(u: Vector, v: Vector) -> Vector:
    res = u + v
    if np.isnan(res).any():
        raise FactorIsNotANumberException()
    return res


def attachLength(u: Vector) -> Tuple[float, Vector]:
    return math.sqrt(vectorLengthSqr(u)), u


@dataclass(frozen=True)
class Rating(EventWithTimestamp):
    user: int
    item: int
    rating: float
    timestamp: int = 0

    def enrich(self, workerId: int, ratingId: int) -> "RichRating":
        return RichRating(self, workerId, ratingId)

    def getEventTime(self) -> int:
        return self.timestamp


@dataclass(frozen=True)
class RichRating(EventWithTimestamp):
    """A rating with a target worker and a rating id (InputTypes.scala:44-49)."""

    base: Rating
    targetWorker: int
    ratingId: int

    def reduce(self) -> Rating:
        return self.base

    def getEventTime(self) -> int:
        return self.base.getEventTime()


def ratingFromTuple(t) -> Rating:
    return Rating(int(t[0]), int(t[1]), float(t[2]), 0)


class IDGenerator:
    _n = itertools.count()
    _lock = threading.Lock()

    @classmethod
    def next(cls) -> int:
        with cls._lock:
            return next(cls._n)


# ---- factor initialisers ------------------------------------------------------------------
class FactorInitializer:
    def nextFactor(self, id: int) -> Vector:
        raise NotImplementedError


class FactorInitializerDescriptor:
    """Serializable recipe; ``open()`` builds the (non-serialisable RNG holding) initialiser."""

    def open(self) -> FactorInitializer:
        raise NotImplementedError


class RandomFactorInitializer(FactorInitializer):
    """U[0,1) (RandomFactorInitializer.scala)."""

    def __init__(self, rnd: random.Random, numFactors: int):
        self.rnd, self.n = rnd, numFactors

    def nextFactor(self, id):
        return np.array([self.rnd.random() for _ in range(self.n)])


class RandomFactorInitializerDescriptor(FactorInitializerDescriptor):
    def __init__(self, numFactors: int):
        self.numFactors = numFactors

    def open(self):
        return RandomFactorInitializer(random.Random(), self.numFactors)


class RangedRandomFactorInitializer(FactorInitializer):
    """U[min,max) (RangedRandomFactorInitializer.scala:7-9)."""

    def __init__(self, rnd: random.Random, numFactors: int, rangeMin: float, rangeMax: float):
        self.rnd, self.n, self.lo, self.hi = rnd, numFactors, rangeMin, rangeMax

    def nextFactor(self, id):
        return np.array([self.lo + (self.hi - self.lo) * self.rnd.random() for _ in range(self.n)])


class RangedRandomFactorInitializerDescriptor(FactorInitializerDescriptor):
    def __init__(self, numFactors: int, rangeMin: float, rangeMax: float, seed: Optional[int] = None):
        self.numFactors, self.rangeMin, self.rangeMax, self.seed = numFactors, rangeMin, rangeMax, seed

    def open(self):
        return RangedRandomFactorInitializer(random.Random(self.seed), self.numFactors,
                                             self.rangeMin, self.rangeMax)


class PseudoRandomFactorInitializer(FactorInitializer):
    """Deterministic: RNG seeded by the id (PseudoRandomFactorInitializer.scala:7-20)."""

    def __init__(self, numFactors: int):
        self.n = numFactors

    def nextFactor(self, id):
        r = random.Random(int(id))
        return np.array([r.random() for _ in range(self.n)])


class PseudoRandomFactorInitializerDescriptor(FactorInitializerDescriptor):
    def __init__(self, numFactors: int):
        self.numFactors = numFactors

    def open(self):
        return PseudoRandomFactorInitializer(self.numFactors)


# ---- updaters ---------------------------------------------------------------------------
class FactorUpdater:
    def delta(self, rating: float, user: Vector, item: Vector) -> Tuple[Vector, Vector]:
        raise NotImplementedError


def _sigmoid(x: float) -> float:
    if x >= 0:
        return 1.0 / (1.0 + math.exp(-x))
    e = math.exp(x)
    return e / (1.0 + e)


class SGDUpdater(FactorUpdater):
    """``e = sigmoid(r - u.v)`` (parity, SGDUpdater.scala:8) or plain residual; no regulariser."""

    def __init__(self, learningRate: float, plain_residual: bool = False):
        self.lr = learningRate
        self.plain = plain_residual

    def delta(self, rating, user, item):
        resid = rating - float(np.dot(user, item))
        e = resid if self.plain else _sigmoid(resid)
        return self.lr * e * item, self.lr * e * user


def bpr_delta(u: Vector, vi: Vector, vj: Vector, lr: float, reg: float):
    """One BPR step (Rendle et al. 2009) on the triple ``(u, i, j)``: the SGD deltas of
    ``softplus(-x) + reg/2 * (|u|^2 + |vi|^2 + |vj|^2)`` with ``x = u . (vi - vj)``, all computed from the
    given values, and the triple's loss ``softplus(-x)``.  Returns ``(du, dvi, dvj, loss)``; the
    reference of the device kernel ``fps_mf_bpr``."""
    x = float(np.dot(u, vi - vj))
    g = lr * _sigmoid(-x)
    du = g * (vi - vj) - lr * reg * u
    dvi = g * u - lr * reg * vi
    dvj = -g * u - lr * reg * vj
    loss = max(-x, 0.0) + math.log1p(math.exp(-abs(x)))
    return du, dvi, dvj, loss


def warp_delta(u: Vector, vi: Vector, cand_rows, margin: float, lr: float, reg: float, rank_items: int):
    """One WARP step (Weston, Bengio and Usunier 2011) for the positive ``(u, i)`` and its candidates in draw order,
    ``cand_rows`` (``None`` = a void candidate: skipped, not counted); the reference of the device kernel
    ``fps_mf_warp``.  The first live ``t*`` with ``x = u . (vi - v_t*) < margin`` violates; with ``n`` the live
    candidates examined up to and including it, ``L = ln(max(1, (rank_items - 1) // n))`` and the deltas are those of
    ``L * (margin - x) + reg/2 * (|u|^2 + |vi|^2 + |vj|^2)`` at fixed ``L``, all computed from the given values.

    Returns ``(du, dvi, t*, dvj, n, L, loss)`` with ``loss = L * (margin - x)``; when no candidate violates (no
    update) ``du``, ``dvi``, ``t*`` and ``dvj`` are ``None``, ``L`` and ``loss`` are 0 and ``n`` counts every live
    candidate."""
    u, vi = np.asarray(u, dtype=np.float64), np.asarray(vi, dtype=np.float64)
    n = 0
    for t, vj in enumerate(cand_rows):
        if vj is None:
            continue
        n += 1
        vj = np.asarray(vj, dtype=np.float64)
        x = float(np.dot(u, vi - vj))
        if x < margin:
            L = math.log(max(1, (int(rank_items) - 1) // n))
            g = lr * L
            du = g * (vi - vj) - lr * reg * u
            dvi = g * u - lr * reg * vi
            dvj = -g * u - lr * reg * vj
            return du, dvi, t, dvj, n, L, L * (margin - x)
    return None, None, None, None, n, 0.0, 0.0


def rowwise_adagrad(row: Vector, G: float, delta: Vector, lr: float, k: int, eps: float = 1e-8):
    """One row-wise AdaGrad step of a row whose learning-rate-1 SGD delta is ``delta`` and whose accumulator
    reads ``G``: ``s = |delta|^2 / k``, ``row + lr * delta / (sqrt(G + s) + eps)``.  Returns ``(new_row, s)``; the
    accumulator becomes ``G + s``.  ``k`` is the logical factor count.  The reference of the device kernels'
    ``optimizer="adagrad"``."""
    delta = np.asarray(delta, dtype=np.float64)
    s = float(np.dot(delta, delta)) / k
    return np.asarray(row, dtype=np.float64) + lr * delta / (math.sqrt(G + s) + eps), s


def require_pointwise(backend: str, kw: dict) -> None:
    """The host tiers (``backend="local"`` / ``"native"``) train the pointwise loss with SGD only."""
    if backend != "device" and (kw.get("loss", "pointwise") != "pointwise" or kw.get("regularization", 0)):
        raise ValueError(f"loss={kw.get('loss')!r} / regularization need backend='device' "
                         f"(backend={backend!r} trains the pointwise loss only)")
    if backend != "device" and "margin" in kw:
        raise ValueError(f"margin (of loss='warp') needs backend='device' "
                         f"(backend={backend!r} trains the pointwise loss only)")
    if backend != "device" and kw.get("optimizer", "sgd") != "sgd":
        raise ValueError(f"optimizer={kw.get('optimizer')!r} needs backend='device' "
                         f"(backend={backend!r} trains with SGD only)")
    ns = kw.get("negativeSampling")
    if ns is not None and ns not in ("uniform", "seen"):
        raise ValueError(f"negativeSampling must be 'uniform' or 'seen', got {ns!r}")
    if backend != "device" and ns == "uniform":
        raise ValueError(f"negativeSampling='uniform' needs backend='device' (backend={backend!r} samples "
                         f"negatives from the items each worker has seen: negativeSampling='seen')")


class SeenRegistryOracle:
    """numpy reference of the device's seen-items registry (``negative_sampling="seen"``, DESIGN §2.11), the rule
    of PSOnlineMatrixFactorizationWorker.scala:61-88 and ops/csrc/fps_host.cpp:216-249 applied per micro-batch.

    :meth:`batch` takes one micro-batch ``(users, items)`` in stream order and returns, per record, ``|D_p|`` (the
    items seen before it: the registry before the batch plus the batch's items first seen at earlier
    positions), ``|ring_p|`` (the user's ratings so far, this one included, capped at ``user_memory``) and the
    negative count ``max(0, min(|D_p| - |ring_p|, neg_rate))``; then registers the batch's new items.  ``order``
    holds the registered items in first-occurrence order.  ``user_div``: users are counted per
    ``user // user_div`` slot, like the device ring."""

    def __init__(self, num_items: int, num_users: int, neg_rate: int, user_memory: int, user_div: int = 1):
        self.neg_rate, self.memory, self.user_div = int(neg_rate), int(user_memory), int(user_div)
        self.known = np.zeros(int(num_items), dtype=bool)
        self.order = np.zeros(0, dtype=np.int64)
        self.user_count = np.zeros(-(-int(num_users) // self.user_div), dtype=np.int64)

    def batch(self, users, items):
        users = np.asarray(users, dtype=np.int64) // self.user_div
        items = np.asarray(items, dtype=np.int64)
        n = items.size
        _, first = np.unique(items, return_index=True)
        flag = np.zeros(n, dtype=bool)
        flag[first] = True
        flag &= ~self.known[items]
        dom = self.order.size + np.cumsum(flag) - flag
        # ratings of the same user earlier in the batch: rank inside the stable sort by user
        by_user = np.argsort(users, kind="stable")
        su = users[by_user]
        start = np.r_[True, su[1:] != su[:-1]] if n else np.zeros(0, dtype=bool)
        rank = np.arange(n) - np.maximum.accumulate(np.where(start, np.arange(n), 0))
        within = np.empty(n, dtype=np.int64)
        within[by_user] = rank
        ring = np.minimum(self.user_count[users] + within + 1, self.memory)
        k_neg = np.clip(dom - ring, 0, self.neg_rate)
        np.add.at(self.user_count, users, 1)
        self.order = np.concatenate([self.order, items[flag]])
        self.known[items] = True
        return dom, ring, k_neg


# ---- top-K ------------------------------------------------------------------------------
class TopKQueue:
    """Bounded min-heap of ``(score, itemId)`` keeping the K largest (Utils.scala:13-18)."""

    def __init__(self, k: Optional[int] = None):
        self.k = k
        self.h: List[Tuple[float, int]] = []

    def push(self, score: float, item: int) -> None:
        if self.k is None or len(self.h) < self.k:
            heapq.heappush(self.h, (score, item))
        elif (score, item) > self.h[0]:
            heapq.heapreplace(self.h, (score, item))

    def min_score(self) -> float:
        return self.h[0][0] if self.h else -math.inf

    def __len__(self):
        return len(self.h)

    def sorted_desc(self) -> List[Tuple[float, int]]:
        return sorted(self.h, reverse=True)


class Partitioner:
    """``hash(id) % psParallelism`` / answer-to-worker pair (Utils.scala:44-63)."""

    def __init__(self, psParallelism: int):
        self.psP = psParallelism

    def workerToPSPartitioner(self, msg) -> int:
        m = msg[0] if isinstance(msg, (list, tuple)) else msg
        return stable_hash(m.paramId) % self.psP

    @staticmethod
    def psToWorkerPartitioner(msg) -> int:
        m = msg[0] if isinstance(msg, (list, tuple)) else msg
        return m.workerPartitionIndex
