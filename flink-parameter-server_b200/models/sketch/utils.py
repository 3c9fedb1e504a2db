"""Sketch helpers (M/sketch/utils/{Utils,TweetReader,TimeAwareTweetReader}.scala)."""
from __future__ import annotations

import math
from typing import Iterable, List, Optional, Sequence, Tuple


def dotProduct(u: Sequence[int], v: Sequence[int]) -> int:
    return int(sum(a * b for a, b in zip(u, v)))


def bloomEq(m: float, k: float, size: float) -> float:
    """Cardinality estimate of a Bloom filter with ``size`` set bits: ``-m/k * ln(1 - size/m)``."""
    return -m / k * math.log(1 - size / m)


def bloomCoOccurrence(m: float, k: float, sizeA: int, sizeB: int, sizeUnion: int) -> Optional[float]:
    """``n(A) + n(B) - n(A u B)`` from the set-bit counts, or None when the union has all ``m`` bits set: one of
    the estimates is then infinite and the score is not a number.  The device scan ranks such a key as not a
    key (``-3e38``), so both tiers leave it out of the top-K."""
    if sizeUnion >= m:
        return None
    return bloomEq(m, k, sizeA) + bloomEq(m, k, sizeB) - bloomEq(m, k, sizeUnion)


def java_round(x: float) -> int:
    """``Math.round`` on a double: the nearest integer, halves toward +inf.  ``floor(x + 0.5)`` would round
    0.49999999999999994 up, and Python's ``round`` takes halves to even."""
    f = math.floor(x)
    return int(f) + (x - f >= 0.5)


def bloomUnion(m: float, k: float, A: Iterable[int], B: Iterable[int]) -> float:
    """Estimate of |A u B| from the union of the two bit sets (BitSet or index-array form)."""
    return bloomEq(m, k, len(set(A) | set(B)))


class TweetReader:
    """``line -> (tweetId, [filtered lower-cased words])`` (TweetReader.scala): column 0 is the id,
    column 5 the text; only ``searchWords`` are kept, empty tweets are dropped."""

    def __init__(self, delimiter: str, searchWords: Sequence[str]):
        self.delimiter = delimiter
        self.words = set(searchWords)

    def __call__(self, line: str) -> List[Tuple[str, List[str]]]:
        cols = line.split(self.delimiter)
        tweet = [w for w in (x.lower() for x in cols[5].split(" ")) if w in self.words]
        return [(cols[0], tweet)] if tweet else []


class TimeAwareTweetReader(TweetReader):
    """Adds ``timeSlot = (col1 - timeStamp) // (windowSize hours)`` (TimeAwareTweetReader.scala)."""

    def __init__(self, delimiter: str, searchWords: Sequence[str], timeStamp: int, windowSize: int):
        super().__init__(delimiter, searchWords)
        self.timeStamp, self.windowSize = timeStamp, windowSize

    def __call__(self, line: str):
        cols = line.split(self.delimiter)
        tweet = [w for w in (x.lower() for x in cols[5].split(" ")) if w in self.words]
        slot = int((int(cols[1]) - self.timeStamp) // (self.windowSize * 60 * 60))
        return [(cols[0], tweet, slot)] if tweet else []


def merge_topk(partials: Iterable[Sequence[Tuple[float, int]]], K: int) -> List[Tuple[float, int]]:
    """Merge per-shard top-K lists: sorted descending, best K (the parallelism-1 sink of the
    predict jobs, e.g. BloomFilterPredict.scala:113-138)."""
    allv: List[Tuple[float, int]] = []
    for p in partials:
        allv.extend(p)
    return sorted(allv)[-K:][::-1]
