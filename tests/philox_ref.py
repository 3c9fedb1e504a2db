"""NumPy oracle of the Philox4x32-10 generator used by the init / sampling kernels."""
from fractions import Fraction

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)


def philox4x32(c0, c1, c2, c3, k0, k1):
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint32).copy() for x in np.broadcast_arrays(c0, c1, c2, c3))
    k0 = np.uint32(k0); k1 = np.uint32(k1)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & MASK).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & MASK).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0 = np.uint32((int(k0) + int(W0)) & 0xFFFFFFFF)
            k1 = np.uint32((int(k1) + int(W1)) & 0xFFFFFFFF)
    return c0, c1, c2, c3


def init_rows_ref(ids, dim, seed, lo, hi):
    """value(id, j) exactly as csrc/fps_core.cu::fps_init_rows_kernel computes it (fp32)."""
    ids = np.asarray(ids, dtype=np.int64)
    stride = (dim + 3) // 4 * 4
    out = np.zeros((len(ids), stride), dtype=np.float32)
    id_lo = (ids & 0xFFFFFFFF).astype(np.uint32)
    id_hi = ((ids >> 32) & 0xFFFFFFFF).astype(np.uint32)
    for q in range(stride // 4):
        r = philox4x32(id_lo, id_hi, np.uint32(q), np.uint32(0), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
        for j in range(4):
            col = 4 * q + j
            if col < dim:
                u = (r[j] >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
                out[:, col] = np.float32(lo) + np.float32(hi - lo) * u
    return out


def init_rows_f64_ref(ids, dim, seed, lo, hi):
    """value(id, j) exactly as csrc/fps_mf_f64.cu::fps_init_rows_f64_kernel computes it: with u the 53-bit uniform
    of Philox words (2 (j % 2), 2 (j % 2) + 1) at counter (id, j / 2, 1), ``lo + (hi - lo) * u`` rounded once (the
    kernel contracts it to one DFMA), padding columns 0."""
    ids = np.asarray(ids, dtype=np.int64)
    stride = (dim + 1) // 2 * 2
    out = np.zeros((len(ids), stride), dtype=np.float64)
    id_lo = (ids & 0xFFFFFFFF).astype(np.uint32)
    id_hi = ((ids >> 32) & 0xFFFFFFFF).astype(np.uint32)
    lo_q, sc_q = Fraction(lo), Fraction(hi - lo)
    for q in range(stride // 2):
        r = philox4x32(id_lo, id_hi, np.uint32(q), np.uint32(1), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
        for j in range(2):
            col = 2 * q + j
            if col < dim:
                w = (r[2 * j].astype(np.uint64) << np.uint64(32)) | r[2 * j + 1].astype(np.uint64)
                # float(Fraction) rounds the exact value to nearest-even, as the fused multiply-add does
                out[:, col] = [float(lo_q + sc_q * Fraction(int(m), 1 << 53)) for m in (w >> np.uint64(11))]
    return out


def k5_shift(neg, z, num_items):
    """Where a draw that hit the positive moves to: ``neg + 1 + (z % 7) % (num_items - 1)`` modulo ``num_items``,
    never back on ``neg`` (``num_items >= 2``)."""
    neg = np.asarray(neg, dtype=np.int64)
    z = np.asarray(z, dtype=np.uint32)
    return (neg + 1 + (z % np.uint32(7)).astype(np.int64) % (num_items - 1)) % num_items


def k5_negative(pos, j, items, num_items, step, seed):
    """Negative ``j >= 1`` of record ``pos`` whose positive is ``items``: the draw ``h % num_items`` of Philox key
    ``(pos, j, step, seed)`` (``h`` = words x:y), moved by :func:`k5_shift` when it is the positive.  The pointwise
    step (csrc/fps_core.cu, fps_mf_tma.cu) draws negative ``j`` of a record; BPR and WARP draw their negative
    ``t`` with ``j = t + 1``.  Returns (negatives, raw draws)."""
    pos = np.asarray(pos, dtype=np.int64)
    x, y, z, _ = philox4x32(pos & 0xFFFFFFFF, pos >> 32, np.uint32(j), np.uint32(step & 0xFFFFFFFF),
                            seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    h = (x.astype(np.uint64) << np.uint64(32)) | y.astype(np.uint64)
    raw = (h % np.uint64(num_items)).astype(np.int64)
    return np.where(raw == np.asarray(items, dtype=np.int64), k5_shift(raw, z, num_items), raw), raw
