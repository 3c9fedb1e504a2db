"""LEMP candidate pruning for top-K maximum-inner-product search.

Strategies and their string form (M/matrix/factorization/pruning/LEMPPruningStrategy.scala:6-77):
``length`` | ``coord`` | ``incr:<n>`` | ``lc:<threshold>`` | ``li:<n>:<threshold>``.
Predicates (LEMPPruningFunctions.scala:20-89) take ``(itemId, (length, vector))`` and say whether
the item *may* still beat the current threshold (True = keep as candidate).

The device tier keeps the string-configurable strategies but realises pruning at tile
granularity inside the wgmma scoring kernel (length bound per 128-item tile of the
length-sorted item table; ops/csrc/fps_topk_mma.cu); every pruned result is validated against
brute force in the tests because the reference's bounds are themselves untested (SURVEY §7.4).
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass
from typing import Callable, Sequence, Tuple

import numpy as np

LengthAndVector = Tuple[float, np.ndarray]
Candidate = Tuple[int, LengthAndVector]


class LEMPPruningStrategy:
    @staticmethod
    def fromString(s: str) -> "LEMPPruningStrategy":
        if s == "length":
            return LENGTH()
        if s == "coord":
            return COORD()
        m = re.fullmatch(r"incr:(\d+)", s)
        if m:
            return INCR(int(m.group(1)))
        m = re.fullmatch(r"lc:([0-9.]+)", s)
        if m:
            return LC(float(m.group(1)))
        m = re.fullmatch(r"li:(\d+):([0-9.]+)", s)
        if m:
            return LI(int(m.group(1)), float(m.group(2)))
        raise ValueError(f"Invalid LEMP Pruning strategy string {s}")

    from_string = fromString


@dataclass(frozen=True)
class LENGTH(LEMPPruningStrategy):
    pass


@dataclass(frozen=True)
class COORD(LEMPPruningStrategy):
    pass


@dataclass(frozen=True)
class INCR(LEMPPruningStrategy):
    numFocusCoordinates: int


@dataclass(frozen=True)
class LC(LEMPPruningStrategy):
    algorithmSwitchThreshold: float


@dataclass(frozen=True)
class LI(LEMPPruningStrategy):
    numFocusCoordinates: int
    algorithmSwitchThreshold: float


def lengthPruning(minLength: float) -> Callable[[Candidate], bool]:
    """Keep items with ``||p|| >= theta / ||q||``.  (The reference compares ``||p||^2`` with
    the un-squared bound, LEMPPruningFunctions.scala:20-22 -- still a valid, looser filter for
    lengths <= 1; here the exact Cauchy-Schwarz bound is used.)"""
    return lambda v: v[1][0] >= minLength


def coordPruning(f: int, userVector: LengthAndVector, theta_b_q: float) -> Callable[[Candidate], bool]:
    """Feasible interval of the normalised focus coordinate ``p_f/||p||`` given that the cosine
    must reach ``theta_b_q`` (LEMPPruningFunctions.scala:31-52)."""
    qlen, q = userVector
    if theta_b_q <= 0 or qlen == 0:
        return lambda p: True
    if theta_b_q > 1:
        return lambda p: False
    q_bar_f = q[f] / qlen
    a = q_bar_f * theta_b_q
    b = math.sqrt(max(0.0, (1 - theta_b_q * theta_b_q) * (1 - q_bar_f * q_bar_f)))
    l_f, u_f = a - b, a + b

    def keep(p: Candidate) -> bool:
        plen, pv = p[1]
        if plen == 0:
            return False
        p_bar_f = pv[f] / plen
        return (l_f - 1e-12) <= p_bar_f <= (u_f + 1e-12)

    return keep


def incrPruning(F: Sequence[int], user: LengthAndVector, theta: float) -> Callable[[Candidate], bool]:
    """Partial dot over the focus set ``F`` plus Cauchy-Schwarz on the rest
    (LEMPPruningFunctions.scala:54-89)."""
    qlen, q = user
    F = list(F)
    qF = q[F] if F else np.zeros(0)
    q_mF_sqr = max(0.0, qlen * qlen - float(np.dot(qF, qF)))

    def keep(p: Candidate) -> bool:
        plen, pv = p[1]
        pF = pv[F] if F else np.zeros(0)
        u_bound = theta - float(np.dot(qF, pF))
        if u_bound < 0.0:
            return True
        return q_mF_sqr * max(0.0, plen * plen - float(np.dot(pF, pF))) >= u_bound * u_bound - 1e-12

    return keep


def focus_coordinate(q: np.ndarray) -> int:
    """Coordinate with the largest magnitude (all coordinates considered; the reference's fold
    starts at index 0 and its ``focusSet`` skips the last one, PSTopKGeneratorWorker.scala:55-66)."""
    return int(np.argmax(q * q))


def focus_set(q: np.ndarray, n: int) -> np.ndarray:
    return np.argsort(-(q * q), kind="stable")[:n]
