"""Streaming sketches on the parameter server (M/sketch/**): Bloom filter, tug-of-war (AMS),
MinHash -- plain and time-aware -- with their train jobs, predict jobs and PS logics.

Train jobs are push-only (``onPullRecv`` is never called, ``???`` in the reference), keyed by
``word.hashCode``; the model is dumped at ``close()``.  Predict jobs load the model through
``transformWithModelLoad``, *pull* the query word's sketch, *push-broadcast* it to every PS shard
("push as RPC to shard i": ids 0..psParallelism-1 hash to themselves), every shard emits a local
top-K and a parallelism-1 merge produces the answer.

Device equivalents: models/sketch/device.py + ops/csrc/fps_sketch.cu (packed bitmaps with
``red.or``, int counters with ``red.add.s32``, packed (hash,id) ``atom.min.u64``).
"""
from __future__ import annotations

import math
from typing import Any, Dict, List, Sequence, Tuple

from ...api import Left, ParameterServerLogic, Right, WorkerLogic
from ...limiter import addPullLimiter
from ...runtime.stream import as_stream
from ...runtime.transform import (default_param_partitioner, default_worker_partitioner, transform,
                                  transformWithModelLoad)
from .hashing import floor_mod, hash64, hash64_signed, java_string_hash, murmur3_32
from .utils import bloomCoOccurrence, dotProduct, java_round, merge_topk


def _unsupported(*_a, **_k):
    raise NotImplementedError("push-only job: pulls are not part of the protocol")


def _ps_only(result) -> List[Any]:
    return result.ps_outputs()


def _device_train(kind: str, src, numHashes: int, arraySize: int = 0, capacity=None, group=None,
                  chunk: int = 65536, time_aware: bool = False) -> List[Any]:
    """``backend="device"`` of the push-only train jobs: the same ``(tweetId, [words])`` stream updates a
    :class:`~fps_b200.models.sketch.device.DeviceSketch` (one-sided ``red.or / red.add / red.min`` pushes)
    and the ``close()`` dump has the host jobs' shape.  Integer tweet ids; the hash family is the device
    one (``hashing.hash64``), not the reference's murmur3 / xxHash, so bit positions differ from the host
    tier while the sketch semantics (and the estimates) are the same.  In a multi-rank job every rank
    feeds its partition of the stream and gets the dump of its own shard."""
    from .device import DeviceSketch

    recs = [(int(r[0]), list(r[1])) + ((int(r[2]),) if time_aware else ())
            for r in (src.collect() if hasattr(src, "collect") else src)]
    if capacity is None:
        capacity = max(1, len({(w, r[2]) if time_aware else w for r in recs for w in r[1]}))
    sk = DeviceSketch(kind, int(capacity), numHashes, arraySize, group=group, time_aware=time_aware)
    try:
        for a in range(0, len(recs), chunk):
            sk.update(recs[a:a + chunk])
        return sk.model()
    finally:
        sk.close()


def _device_predict(kind: str, queries, model, numHashes: int, K: int, arraySize: int = 0, numMeans: int = 1,
                    time_aware: bool = False, counts=None, cooccurrence: bool = False, capacity=None,
                    group=None) -> List[Any]:
    """``backend="device"`` of the predict jobs: the model dump is loaded into a
    :class:`~fps_b200.models.sketch.device.DeviceSketch` (one-sided stores), every query word's sketch is
    pulled and scored against every shard by the scan kernels (popcount / median-of-means / equality
    count, ops/csrc/fps_sketch.cu), the local top-K lists are gathered by one-sided stores and merged on
    the device.  Output shape = the host jobs': ``[(queryId | (queryId, slot), [(score, key)] best first)]``."""
    from .device import DeviceSketch

    entries = list(model.collect() if hasattr(model, "collect") else model)
    if capacity is None:
        capacity = max(1, len(entries))
    sk = DeviceSketch(kind, int(capacity), numHashes, arraySize, group=group, time_aware=time_aware)
    try:
        sk.load_model(entries, counts)
        out = []
        for q in (queries.collect() if hasattr(queries, "collect") else queries):
            queryId, word = q if isinstance(q, (tuple, list)) else (java_string_hash(q), q)
            if time_aware:
                for slot in sk.slots_of(word):       # one pull -> one answer per time slot of the word
                    top = sk.query(word, K, num_means=numMeans, slot=slot)
                    out.append(((queryId, slot), [(sc, key[0]) for sc, key in top]))
            else:
                out.append((queryId, sk.query(word, K, num_means=numMeans, cooccurrence=cooccurrence)))
        return out
    finally:
        sk.close()


# =============================================================================================
# Bloom filter
# =============================================================================================
def bloom_positions(tweet_id: str, numHashes: int, arraySize: int) -> List[int]:
    return [floor_mod(murmur3_32(tweet_id, i), arraySize) for i in range(numHashes)]


class BloomPSLogic(ParameterServerLogic):
    """``word -> set of bit positions`` (BloomPSLogic.scala:10-27)."""

    def __init__(self):
        self.model: Dict[int, set] = {}

    onPullRecv = _unsupported

    def onPushRecv(self, id, deltaUpdate, ps):
        self.model.setdefault(id, set()).update(deltaUpdate)

    def close(self, ps):
        for id, c in self.model.items():
            ps.output((id, frozenset(c)))


class _BloomWorker(WorkerLogic):
    def __init__(self, arraySize, numHashes):
        self.m, self.k = arraySize, numHashes

    def onRecv(self, data, ps):
        tweet_id, words = data[0], data[1]
        AS = bloom_positions(tweet_id, self.k, self.m)
        for w in words:
            ps.push(java_string_hash(w), AS)

    onPullRecv = _unsupported


def bloomFilter(src, arraySize: int, numHashes: int, workerParallelism: int, psParallelism: int,
                iterationWaitTime: float = 10000, backend: str = "local", **device_kw) -> List[Tuple[int, frozenset]]:
    """Train: stream of ``(tweetId, [words])`` -> ``[(wordHash, bitset)]`` (BloomFilter.scala:32-98)."""
    if backend == "device":
        return _device_train("bloom", src, numHashes, arraySize, **device_kw)
    return _ps_only(transform(src, _BloomWorker(arraySize, numHashes), BloomPSLogic(),
                              workerParallelism, psParallelism, iterationWaitTime))


class BloomPredictPSLogic(ParameterServerLogic):
    """Model load by ``Right(bitset)`` pushes; ``Left((queryId, bitset))`` push = score the query
    against every local key: ``n(A) + n(B) - n(A u B)`` (BloomPredictPSLogic.scala:14-65)."""

    def __init__(self, arraySize: int, numHashes: int, K: int):
        self.m, self.k, self.K = arraySize, numHashes, K
        self.model: Dict[int, frozenset] = {}

    def onPullRecv(self, id, workerPartitionIndex, ps):
        ps.answerPull(id, Left((0, self.model.get(id, frozenset()))), workerPartitionIndex)

    def onPushRecv(self, id, deltaUpdate, ps):
        if deltaUpdate.is_left:
            queryId, target = deltaUpdate.value
            topK = []
            for k, v in self.model.items():     # a saturated union has no estimate: the key is skipped
                est = bloomCoOccurrence(self.m, self.k, len(target), len(v), len(target | v))
                if est is not None:
                    topK.append((est, k))
            ps.output((queryId, sorted(topK)[-self.K:]))
        else:
            self.model[id] = frozenset(deltaUpdate.value)


class _BroadcastQueryWorker(WorkerLogic):
    """pull(word) -> push the answered sketch to every shard (BloomFilterPredict.scala:44-65)."""

    def __init__(self, psParallelism: int):
        self.psP = psParallelism
        self.queryBuffer: Dict[int, int] = {}

    def onRecv(self, data, ps):
        queryId, word = data
        h = java_string_hash(word)
        self.queryBuffer[h] = queryId
        ps.pull(h)

    def onPullRecv(self, paramId, paramValue, ps):
        if paramValue.is_left:
            _, target = paramValue.value
            for i in range(self.psP):
                ps.push(i, Left((self.queryBuffer[paramId], target)))


def _int_hash_partitioner(psParallelism: int):
    def part(msg) -> int:
        m = msg[0] if isinstance(msg, (list, tuple)) else msg
        pid = m.paramId
        return abs(pid if isinstance(pid, int) else hash(pid)) % psParallelism

    return part


def _predict(src, model, workerLogic, serverLogic, K, workerParallelism, psParallelism, pullLimit,
             iterationWaitTime):
    res = transformWithModelLoad(model)(
        src, addPullLimiter(workerLogic, pullLimit), serverLogic,
        _int_hash_partitioner(psParallelism), default_worker_partitioner(workerParallelism),
        workerParallelism, psParallelism, iterationWaitTime)
    buf: Dict[Any, List] = {}
    for queryId, local in res.ps_outputs():
        buf.setdefault(queryId, []).append(local)
    return [(q, merge_topk(parts, K)) for q, parts in buf.items() if len(parts) == psParallelism]


def bloomPredict(src, model, arraySize: int, numHashes: int, K: int, workerParallelism: int,
                 psParallelism: int, pullLimit: int, iterationWaitTime: float = 10000,
                 backend: str = "local", **device_kw):
    """Predict: ``src`` = ``(queryId, word)``, ``model`` = ``(wordHash, bitset)`` pairs ->
    ``[(queryId, [(estimatedCoOccurrence, wordHash)] best-first)]`` (BloomFilterPredict.scala:33-139)."""
    if backend == "device":
        return _device_predict("bloom", src, model, numHashes, K, arraySize=arraySize, **device_kw)
    m = as_stream(model).map(lambda kv: (kv[0], Right(kv[1])))
    return _predict(src, m, _BroadcastQueryWorker(psParallelism),
                    BloomPredictPSLogic(arraySize, numHashes, K), K, workerParallelism,
                    psParallelism, pullLimit, iterationWaitTime)


# ---- time-aware Bloom -------------------------------------------------------------------------
class TimeAwareBloomPSLogic(ParameterServerLogic):
    """Keyed ``(wordHash, timeSlot)``; positions appended, de-duplicated at close
    (pslogic/TimeAwareBloomPSLogic.scala)."""

    def __init__(self):
        self.model: Dict[Tuple[int, int], List[int]] = {}

    onPullRecv = _unsupported

    def onPushRecv(self, id, deltaUpdate, ps):
        slot, positions = deltaUpdate
        self.model.setdefault((id, slot), []).extend(positions)

    def close(self, ps):
        for key, c in self.model.items():
            ps.output((key, frozenset(c)))


class _TimeAwareBloomWorker(WorkerLogic):
    def __init__(self, arraySize, numHashes):
        self.m, self.k = arraySize, numHashes

    def onRecv(self, data, ps):
        tweet_id, words, slot = data
        AS = bloom_positions(tweet_id, self.k, self.m)
        for w in words:
            ps.push(java_string_hash(w), (slot, AS))

    onPullRecv = _unsupported


def timeAwareBloomFilter(src, arraySize, numHashes, workerParallelism, psParallelism,
                         iterationWaitTime=10000, backend: str = "local", **device_kw):
    """(TimeAwareBloomFilter.scala:31-92) -> ``[((wordHash, slot), bitset)]``."""
    if backend == "device":
        return _device_train("bloom", src, numHashes, arraySize, time_aware=True, **device_kw)
    return _ps_only(transform(src, _TimeAwareBloomWorker(arraySize, numHashes), TimeAwareBloomPSLogic(),
                              workerParallelism, psParallelism, iterationWaitTime))


class TimeAwareBloomPredictPSLogic(ParameterServerLogic):
    """One pull -> one answer PER TIME SLOT of the word; queries are scored against same-slot
    keys only (pslogic/TimeAwareBloomPredictPSLogic.scala:14-60)."""

    def __init__(self, arraySize, numHashes, K):
        self.m, self.k, self.K = arraySize, numHashes, K
        self.model: Dict[Tuple[int, int], frozenset] = {}

    def onPullRecv(self, id, workerPartitionIndex, ps):
        for key, v in self.model.items():
            if key[0] == id:
                ps.answerPull(id, Left((key, v)), workerPartitionIndex)

    def onPushRecv(self, id, deltaUpdate, ps):
        if deltaUpdate.is_left:
            (queryId, slot), target = deltaUpdate.value
            topK = []
            for (k, s), v in self.model.items():
                if s == slot:
                    est = bloomCoOccurrence(self.m, self.k, len(target), len(v), len(target | v))
                    if est is not None:
                        topK.append((est, k))
            ps.output(((queryId, slot), sorted(topK)[-self.K:]))
        else:
            slot, bits = deltaUpdate.value
            self.model[(id, slot)] = frozenset(bits)


class _TimeAwareBroadcastWorker(WorkerLogic):
    def __init__(self, psParallelism):
        self.psP = psParallelism
        self.queryBuffer: Dict[int, int] = {}

    def onRecv(self, data, ps):
        queryId, word = data
        h = java_string_hash(word)
        self.queryBuffer[h] = queryId
        ps.pull(h)

    def onPullRecv(self, paramId, paramValue, ps):
        if paramValue.is_left:
            (_, slot), target = paramValue.value
            for i in range(self.psP):
                ps.push(i, Left(((self.queryBuffer[paramId], slot), target)))


def timeAwareBloomPredict(src, model, arraySize, numHashes, K, workerParallelism, psParallelism,
                          pullLimit, iterationWaitTime=10000, backend: str = "local", **device_kw):
    """``model`` = ``((wordHash, slot), bitset)`` pairs -> ``[((queryId, slot), topK)]``.
    The pull limiter must allow multi-answer pulls, so the limit is applied per query word."""
    if backend == "device":
        return _device_predict("bloom", src, model, numHashes, K, arraySize=arraySize, time_aware=True,
                               **device_kw)
    m = as_stream(model).map(lambda kv: (kv[0][0], Right((kv[0][1], kv[1]))))
    res = transformWithModelLoad(m)(
        src, _TimeAwareBroadcastWorker(psParallelism), TimeAwareBloomPredictPSLogic(arraySize, numHashes, K),
        _int_hash_partitioner(psParallelism), default_worker_partitioner(workerParallelism),
        workerParallelism, psParallelism, iterationWaitTime)
    buf: Dict[Any, List] = {}
    for key, local in res.ps_outputs():
        buf.setdefault(key, []).append(local)
    return [(q, merge_topk(parts, K)) for q, parts in buf.items() if len(parts) == psParallelism]


# =============================================================================================
# Tug-of-war (AMS) sketch
# =============================================================================================
def tow_hash_words(tweet_id: int, numHashes: int) -> List[int]:
    """``ceil(numHashes / 64)`` 64-bit hash words of the tweet id.  (The reference computes
    ``0 to ceil(numHashes/64)`` with integer division, i.e. one word too many or too few,
    TugOfWar.scala:38 -- SURVEY §7.4; here exactly enough bits are produced.)"""
    return [hash64(int(tweet_id), i) for i in range((numHashes + 63) // 64)]


def _bit(words: Sequence[int], j: int) -> int:
    return (words[j >> 6] >> (j & 63)) & 1


class BitSetBasedPSLogic(ParameterServerLogic):
    """``counter[j] += bit_j ? +1 : -1`` (pslogic/BitSetBasedPSLogic.scala:8-30)."""

    def __init__(self, numHashes: int):
        self.n = numHashes
        self.model: Dict[Any, List[int]] = {}

    onPullRecv = _unsupported

    def _key(self, id, deltaUpdate):
        return id, deltaUpdate

    def onPushRecv(self, id, deltaUpdate, ps):
        key, words = self._key(id, deltaUpdate)
        param = self.model.setdefault(key, [0] * self.n)
        for j in range(self.n):
            param[j] += 1 if _bit(words, j) else -1

    def close(self, ps):
        for id, c in self.model.items():
            ps.output((id, list(c)))


class TimeAwareToWPSLogic(BitSetBasedPSLogic):
    """Keyed ``(wordHash, slot)`` (pslogic/TimeAwareToWPSLogic.scala)."""

    def _key(self, id, deltaUpdate):
        slot, words = deltaUpdate
        return (id, slot), words


class _ToWWorker(WorkerLogic):
    def __init__(self, numHashes, time_aware=False):
        self.n, self.ta = numHashes, time_aware

    def onRecv(self, data, ps):
        words64 = tow_hash_words(int(data[0]), self.n)
        for w in data[1]:
            ps.push(java_string_hash(w), (data[2], words64) if self.ta else words64)

    onPullRecv = _unsupported


def tugOfWar(src, numHashes, workerParallelism, psParallelism, iterationWaitTime=10000,
             backend: str = "local", **device_kw):
    """(TugOfWar.scala:17-82) -> ``[(wordHash, int counters[numHashes])]``."""
    if backend == "device":
        return _device_train("tow", src, numHashes, **device_kw)
    return _ps_only(transform(src, _ToWWorker(numHashes), BitSetBasedPSLogic(numHashes),
                              workerParallelism, psParallelism, iterationWaitTime))


def timeAwareTugOfWar(src, numHashes, workerParallelism, psParallelism, iterationWaitTime=10000,
                      backend: str = "local", **device_kw):
    """(TimeAwareTugOfWar.scala:17-60) -> ``[((wordHash, slot), counters)]``."""
    if backend == "device":
        return _device_train("tow", src, numHashes, time_aware=True, **device_kw)
    return _ps_only(transform(src, _ToWWorker(numHashes, True), TimeAwareToWPSLogic(numHashes),
                              workerParallelism, psParallelism, iterationWaitTime))


def median_of_means(a: Sequence[int], b: Sequence[int], numHashes: int, numMeans: int) -> float:
    """Median over ``numMeans`` groups of the mean slice dot-product
    (SketchPredictPSLogic.scala:23-40)."""
    size = max(1, int(math.ceil(numHashes / numMeans)))
    means = []
    for i in range(0, numHashes, size):
        sa, sb = a[i:i + size], b[i:i + size]
        means.append(dotProduct(sa, sb) / len(sa))
    means.sort(reverse=True)
    n = len(means)
    return (means[n // 2] + means[n // 2 - 1]) / 2 if n % 2 == 0 else means[n // 2]


class SketchPredictPSLogic(ParameterServerLogic):
    def __init__(self, numHashes, numMeans, K):
        self.n, self.means, self.K = numHashes, numMeans, K
        self.model: Dict[int, List[int]] = {}

    def onPullRecv(self, id, workerPartitionIndex, ps):
        ps.answerPull(id, Left((0, self.model.setdefault(id, [0] * self.n))), workerPartitionIndex)

    def onPushRecv(self, id, deltaUpdate, ps):
        if deltaUpdate.is_left:
            queryId, target = deltaUpdate.value
            topK = [(median_of_means(v, target, self.n, self.means), k) for k, v in self.model.items()]
            ps.output((queryId, sorted(topK)[-self.K:]))
        else:
            self.model[id] = list(deltaUpdate.value)


class SketchPSLogic(ParameterServerLogic):
    """Generic dot-product sketch store with a top-100 query (pslogic/SketchPSLogic.scala:8-41;
    unused by the reference's jobs, kept for API parity)."""

    def __init__(self, numHashes: int, K: int = 100):
        self.n, self.K = numHashes, K
        self.model: Dict[int, List[int]] = {}

    def onPullRecv(self, id, workerPartitionIndex, ps):
        ps.answerPull(id, self.model.setdefault(id, [0] * self.n), workerPartitionIndex)

    def onPushRecv(self, id, deltaUpdate, ps):
        if isinstance(deltaUpdate, tuple) and deltaUpdate and deltaUpdate[0] == "query":
            _, queryId, target = deltaUpdate
            scores = [(dotProduct(v, target) / self.n, k) for k, v in self.model.items()]
            ps.output((queryId, sorted(scores)[-self.K:]))
        else:
            param = self.model.setdefault(id, [0] * self.n)
            for j, d in enumerate(deltaUpdate):
                param[j] += d


def tugOfWarPredict(src, model, numHashes, numMeans, K, workerParallelism, psParallelism, pullLimit,
                    iterationWaitTime=10000, backend: str = "local", **device_kw):
    """(TugOfWarPredict.scala:17-108) ``model`` = ``(wordHash, counters)`` pairs."""
    if backend == "device":
        return _device_predict("tow", src, model, numHashes, K, numMeans=numMeans, **device_kw)
    m = as_stream(model).map(lambda kv: (kv[0], Right(kv[1])))
    return _predict(src, m, _BroadcastQueryWorker(psParallelism),
                    SketchPredictPSLogic(numHashes, numMeans, K), K, workerParallelism, psParallelism,
                    pullLimit, iterationWaitTime)


class TimeAwareToWPredictPSLogic(ParameterServerLogic):
    """(pslogic/TimeAwareToWPredictPSLogic.scala) per-slot answers and per-slot scoring."""

    def __init__(self, numHashes, numMeans, K):
        self.n, self.means, self.K = numHashes, numMeans, K
        self.model: Dict[Tuple[int, int], List[int]] = {}

    def onPullRecv(self, id, workerPartitionIndex, ps):
        for key, v in self.model.items():
            if key[0] == id:
                ps.answerPull(id, Left((key, v)), workerPartitionIndex)

    def onPushRecv(self, id, deltaUpdate, ps):
        if deltaUpdate.is_left:
            (queryId, slot), target = deltaUpdate.value
            topK = [(median_of_means(v, target, self.n, self.means), k)
                    for (k, s), v in self.model.items() if s == slot]
            ps.output(((queryId, slot), sorted(topK)[-self.K:]))
        else:
            slot, vec = deltaUpdate.value
            self.model[(id, slot)] = list(vec)


def timeAwareTugOfWarPredict(src, model, numHashes, numMeans, K, workerParallelism, psParallelism,
                             pullLimit, iterationWaitTime=10000, backend: str = "local", **device_kw):
    """(TimeAwareTugOfWarPredict.scala:20-105) ``model`` = ``((wordHash, slot), counters)``."""
    if backend == "device":
        return _device_predict("tow", src, model, numHashes, K, numMeans=numMeans, time_aware=True,
                               **device_kw)
    m = as_stream(model).map(lambda kv: (kv[0][0], Right((kv[0][1], kv[1]))))
    res = transformWithModelLoad(m)(
        src, _TimeAwareBroadcastWorker(psParallelism), TimeAwareToWPredictPSLogic(numHashes, numMeans, K),
        _int_hash_partitioner(psParallelism), default_worker_partitioner(workerParallelism),
        workerParallelism, psParallelism, iterationWaitTime)
    buf: Dict[Any, List] = {}
    for key, local in res.ps_outputs():
        buf.setdefault(key, []).append(local)
    return [(q, merge_topk(parts, K)) for q, parts in buf.items() if len(parts) == psParallelism]


# =============================================================================================
# MinHash
# =============================================================================================
class SendHashPSLogic(ParameterServerLogic):
    """Worker sends ``(tweetId, numHashes hashes)``; the server keeps, per slot, the tweet with the
    smaller hash (pslogic/SendHashPSLogic.scala:11-44); close emits the arg-min tweet ids."""

    def __init__(self, numHashes):
        self.n = numHashes
        self.model: Dict[int, List[Tuple[int, int]]] = {}

    onPullRecv = _unsupported

    def onPushRecv(self, id, deltaUpdate, ps):
        tweetId, hashes = deltaUpdate
        cur = self.model.get(id)
        if cur is None:
            self.model[id] = [(tweetId, h) for h in hashes]
        else:
            self.model[id] = [(t, h) if h <= nh else (tweetId, nh) for (t, h), nh in zip(cur, hashes)]

    def close(self, ps):
        for id, c in self.model.items():
            ps.output((id, [t for t, _ in c]))


class StoredHashPSLogic(ParameterServerLogic):
    """Variation: the worker sends only the tweet id; the server re-hashes per slot and keeps the
    arg-min (pslogic/StoredHashPSLogic.scala:11-29).  ``seed_with_word_id=True`` reproduces the
    reference quirk of seeding a new key with the *word* id (``:24``)."""

    def __init__(self, numHashes, seed_with_word_id: bool = False):
        self.n = numHashes
        self.quirk = seed_with_word_id
        self.model: Dict[int, List[int]] = {}

    onPullRecv = _unsupported

    def onPushRecv(self, id, tweetId, ps):
        cur = self.model.get(id)
        if cur is None:
            self.model[id] = [id if self.quirk else tweetId] * self.n
        else:
            for i in range(self.n):
                if hash64_signed(tweetId, i) < hash64_signed(cur[i], i):
                    cur[i] = tweetId

    def close(self, ps):
        for id, c in self.model.items():
            ps.output((id, list(c)))


class _MinHashWorker(WorkerLogic):
    def __init__(self, numHashes, variation=False):
        self.n, self.var = numHashes, variation

    def onRecv(self, data, ps):
        tweet_id, words = data[0], data[1]
        if self.var:
            for w in words:
                ps.push(java_string_hash(w), int(tweet_id))
        else:
            a = [murmur3_32(tweet_id, i) for i in range(self.n)]
            for w in words:
                ps.push(java_string_hash(w), (int(tweet_id), a))

    onPullRecv = _unsupported


def minhash(src, numHashes, workerParallelism, psParallelism, iterationWaitTime=10000,
            backend: str = "local", **device_kw):
    """(MinHash.scala:15-74) -> ``[(wordHash, [argmin tweetId per slot])]``."""
    if backend == "device":
        return _device_train("minhash", src, numHashes, **device_kw)
    return _ps_only(transform(src, _MinHashWorker(numHashes), SendHashPSLogic(numHashes),
                              workerParallelism, psParallelism, iterationWaitTime))


def minhashVariation(src, numHashes, workerParallelism, psParallelism, iterationWaitTime=10000,
                     seed_with_word_id: bool = False):
    """(variation/MinHash.scala:16-67)."""
    return _ps_only(transform(src, _MinHashWorker(numHashes, True),
                              StoredHashPSLogic(numHashes, seed_with_word_id),
                              workerParallelism, psParallelism, iterationWaitTime))


class MinHashPredictPSLogic(ParameterServerLogic):
    """Jaccard ~ fraction of equal signature slots (pslogic/MinHashPredictPSLogic.scala:7-37)."""

    def __init__(self, numHashes, K):
        self.n, self.K = numHashes, K
        self.model: Dict[int, List[int]] = {}

    def onPullRecv(self, id, workerPartitionIndex, ps):
        ps.answerPull(id, Right(self.model.setdefault(id, [])), workerPartitionIndex)

    def _intersect(self, a, b) -> float:
        if a and b:
            return sum(1 for x, y in zip(a, b) if x == y) / self.n
        return 0.0

    def onPushRecv(self, id, deltaUpdate, ps):
        if deltaUpdate.is_left:
            queryId, target = deltaUpdate.value
            ps.output((queryId, [(self._intersect(target, v), k) for k, v in self.model.items()]))
        else:
            self.model[id] = list(deltaUpdate.value)


class _MinHashQueryWorker(WorkerLogic):
    def __init__(self, psParallelism):
        self.psP = psParallelism

    def onRecv(self, wordHash, ps):
        ps.pull(wordHash)

    def onPullRecv(self, paramId, paramValue, ps):
        if not paramValue.is_right:
            raise RuntimeError("PS should not send Left pull answers")
        for i in range(self.psP):
            ps.push(i, Left((paramId, paramValue.value)))


def word_count(train) -> Dict[int, int]:
    """Keyed word count of the training stream (MinHashPredict.scala:19-37), by word hash."""
    c: Dict[int, int] = {}
    for rec in as_stream(train).collect():
        for w in rec[1]:
            h = java_string_hash(w)
            c[h] = c.get(h, 0) + 1
    return c


def minhashPredict(words, train, model, numHashes, K, workerParallelism, psParallelism, pullLimit,
                   iterationWaitTime=10000, backend: str = "local", **device_kw):
    """(MinHashPredict.scala:60-141): Jaccard estimates converted to co-occurrence counts with the
    word frequencies of ``train``: ``java_round(J * (f_q + f_w) / (J + 1))`` in double, evaluated in that
    order and rounded like Java's ``Math.round`` (halves up, so J = 1 and f_q + f_w = 5 gives 3); per query the
    list is sorted by that count, best first."""
    if backend == "device":   # Jaccard scan + the Aggregate step (word frequencies) in one kernel
        res = _device_predict("minhash", list(as_stream(words).collect()), model, numHashes, K,
                              counts=word_count(train), cooccurrence=True, **device_kw)
        return [(q, [(key, int(c)) for c, key in lst]) for q, lst in res]
    searchWords = as_stream(words).map(java_string_hash)
    m = as_stream(model).map(lambda kv: (kv[0], Right(kv[1])))
    res = transformWithModelLoad(m)(
        searchWords, addPullLimiter(_MinHashQueryWorker(psParallelism), pullLimit),
        MinHashPredictPSLogic(numHashes, K), _int_hash_partitioner(psParallelism),
        default_worker_partitioner(workerParallelism), workerParallelism, psParallelism,
        iterationWaitTime)
    merged: Dict[int, List] = {}
    count: Dict[int, int] = {}
    for q, local in res.ps_outputs():
        merged.setdefault(q, []).extend(local)
        count[q] = count.get(q, 0) + 1
    freq = word_count(train)
    out = []
    for q, inter in merged.items():
        if count[q] < psParallelism:
            continue
        f = freq.get(q, 0)
        r = [(w, java_round((v * (f + freq.get(w, 0))) / (v + 1))) for v, w in inter]
        out.append((q, sorted(r, key=lambda t: t[1], reverse=True)))
    return out


# snake_case aliases
bloom_filter = bloomFilter
bloom_predict = bloomPredict
tug_of_war = tugOfWar
tug_of_war_predict = tugOfWarPredict
minhash_predict = minhashPredict
