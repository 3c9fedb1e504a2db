"""Exact host replays of the streaming-sketch kernels (ops/csrc/fps_sketch.cu).  numpy only, CPU.

Updates return the raw int32 rows a table holds after a batch of ``(key, tweet)`` occurrences:

* Bloom: bit ``hash64(t, j) % array_size`` of the row is set, for ``j < num_hashes``.
* tug-of-war: counter ``j`` adds +1 or -1 from bit ``j & 63`` of ``hash64(t, j >> 6)``.
* MinHash: slot ``j`` (two int32 words, little-endian u64) keeps the minimum of
  ``(hash64(t, j) >> 32) << 32 | (t & 0xFFFFFFFF)``; rows start all-ones.

Tweet ids are int64 and enter the hash as their two's-complement u64, like the kernel's cast.

Queries replay the per-key scans in fp64:

* Bloom: ``n(A) + n(B) - n(A u B)`` with ``n(X) = -m/k * ln(1 - |X|/m)`` (``utils.bloomEq``).  A row with no bit set
  is not a key, and a score that is not finite (some filter has all ``m`` bits set) is the not-a-key score too.
* tug-of-war: the median over groups of the mean slice dot product, grouped as ``jobs.median_of_means``.
* MinHash: the Jaccard ``float32(eq) / float32(n)``; with word frequencies, the co-occurrence count
  ``java_round(J * (f_q + f_w) / (J + 1))`` on the double ``J = eq / n``, in that order.  A row whose slots are
  all empty is not a key.

Rows whose ``key_slot`` differs from ``query_slot`` score ``NEG`` in every scan."""
import numpy as np

NEG = float(np.float32(-3.0e38))
GOLDEN = np.uint64(0x9E3779B97F4A7C15)
M1 = np.uint64(0xBF58476D1CE4E5B9)
M2 = np.uint64(0x94D049BB133111EB)
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
LOW32 = np.uint64(0xFFFFFFFF)


def as_u64(tweets):
    """Tweet ids as the kernel reads them: int64, reinterpreted as u64 (two's complement)."""
    return np.asarray(tweets, dtype=np.int64).view(np.uint64)


def hash64(x, seed):
    """``fps_hash64`` / ``hashing.hash64`` over a u64 (or int64) array, one seed."""
    x = np.asarray(x)
    if x.dtype != np.uint64:
        x = as_u64(x)
    with np.errstate(over="ignore"):
        z = x + GOLDEN * np.uint64(seed + 1)
        z = (z ^ (z >> np.uint64(30))) * M1
        z = (z ^ (z >> np.uint64(27))) * M2
    return z ^ (z >> np.uint64(31))


# ---- updates ------------------------------------------------------------------------------------------------------
def bloom_words(array_size):
    return (array_size + 31) // 32


def bloom_update(keys, tweets, n_keys, num_hashes, array_size):
    """int32 ``[n_keys, ceil(array_size / 32)]``: the Bloom rows after the batch, from zeroed rows."""
    keys = np.asarray(keys, dtype=np.int64)
    t = as_u64(tweets)
    words = bloom_words(array_size)
    bits = np.zeros((n_keys, words * 32), dtype=np.bool_)
    for j in range(num_hashes):
        bits[keys, (hash64(t, j) % np.uint64(array_size)).astype(np.int64)] = True
    return np.packbits(bits, axis=1, bitorder="little").view(np.int32).reshape(n_keys, words)


def tow_update(keys, tweets, n_keys, num_hashes):
    """int32 ``[n_keys, num_hashes]``: the tug-of-war counters after the batch, from zero."""
    keys = np.asarray(keys, dtype=np.int64)
    t = as_u64(tweets)
    out = np.zeros((n_keys, num_hashes), dtype=np.int64)
    for w in range((num_hashes + 63) // 64):
        h = hash64(t, w)
        for j in range(64 * w, min(num_hashes, 64 * w + 64)):
            up = ((h >> np.uint64(j & 63)) & np.uint64(1)).astype(bool)
            out[:, j] = (np.bincount(keys[up], minlength=n_keys)
                         - np.bincount(keys[~up], minlength=n_keys))
    return out.astype(np.int32)


def minhash_packed(tweets, j):
    t = as_u64(tweets)
    return ((hash64(t, j) >> np.uint64(32)) << np.uint64(32)) | (t & LOW32)


def minhash_update(keys, tweets, n_keys, num_hashes, init=None):
    """int32 ``[n_keys, 2 * num_hashes]``: the MinHash signatures (u64 slots, little-endian) after the batch,
    from all-ones rows or from ``init`` (u64 ``[n_keys, num_hashes]``)."""
    keys = np.asarray(keys, dtype=np.int64)
    sig = np.full((n_keys, num_hashes), ALL_ONES, dtype=np.uint64) if init is None else init.copy()
    for j in range(num_hashes):
        col = sig[:, j].copy()
        np.minimum.at(col, keys, minhash_packed(tweets, j))
        sig[:, j] = col
    return sig.view(np.int32).reshape(n_keys, 2 * num_hashes)


# ---- queries ------------------------------------------------------------------------------------------------------
def _slot_mask(n_rows, key_slot, query_slot):
    """True where the row takes part in the scan."""
    if key_slot is None:
        return np.ones(n_rows, dtype=bool)
    return np.asarray(key_slot) == query_slot


def bloom_eq(m, k, size):
    """``utils.bloomEq`` over an array of set-bit counts; ``+inf`` at ``size == m`` and NaN above."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return -m / k * np.log(1 - np.asarray(size, dtype=np.float64) / m)


def bloom_query(rows, n_words, query, m, k, key_slot=None, query_slot=0):
    """(est, n(A u B)) in fp64 for every row of ``rows`` (int32 ``[n_rows, >= n_words]``) against ``query``."""
    rows = np.asarray(rows).view(np.uint32)[:, :n_words]
    q = np.asarray(query).view(np.uint32)[:n_words]
    cq = int(np.bitwise_count(q).sum())
    cb = np.bitwise_count(rows).sum(axis=1, dtype=np.int64)
    cu = np.bitwise_count(rows | q[None, :]).sum(axis=1, dtype=np.int64)
    nU = bloom_eq(m, k, cu)
    with np.errstate(invalid="ignore"):
        est = bloom_eq(m, k, cq) + bloom_eq(m, k, cb) - nU
    keep = _slot_mask(len(rows), key_slot, query_slot) & (cb != 0) & np.isfinite(est)
    return np.where(keep, est, NEG), nU


def tow_groups(n_hashes, num_means):
    """(group size, groups formed) of ``median_of_means``."""
    size = max(1, -(-n_hashes // max(1, num_means)))
    return size, -(-n_hashes // size)


def tow_query(rows, query, n_hashes, num_means, key_slot=None, query_slot=0):
    """fp64 median of group means for every row (int32 ``[n_rows, >= n_hashes]``)."""
    a = np.asarray(rows, dtype=np.int64)[:, :n_hashes]
    b = np.asarray(query, dtype=np.int64)[:n_hashes]
    size, g = tow_groups(n_hashes, num_means)
    means = np.empty((len(a), g), dtype=np.float64)
    for i in range(g):
        lo, hi = i * size, min(n_hashes, i * size + size)
        means[:, i] = (a[:, lo:hi] @ b[lo:hi]) / (hi - lo)       # exact int64 dot, one correctly rounded division
    means = -np.sort(-means, axis=1)
    med = (means[:, g // 2] + means[:, g // 2 - 1]) / 2 if g % 2 == 0 else means[:, g // 2]
    return np.where(_slot_mask(len(a), key_slot, query_slot), med, NEG)


def java_round(x):
    """``Math.round`` on doubles: the nearest integer, halves toward +inf (``floor(x) + (x - floor(x) >= 0.5)``;
    ``floor(x + 0.5)`` would round 0.49999999999999994 up)."""
    x = np.asarray(x, dtype=np.float64)
    f = np.floor(x)
    return f + (x - f >= 0.5)


def minhash_query(rows, query, n_hashes, key_slot=None, query_slot=0, freq=None, query_freq=0.0):
    """Jaccard (float32 values in fp64) or, with ``freq``, the co-occurrence count, for every row
    (int32 ``[n_rows, >= 2 * n_hashes]``)."""
    a = np.ascontiguousarray(np.asarray(rows, dtype=np.int32)[:, :2 * n_hashes]).view(np.uint64)
    b = np.ascontiguousarray(np.asarray(query, dtype=np.int32)[:2 * n_hashes]).view(np.uint64)
    af, bf = a != ALL_ONES, b != ALL_ONES
    eq = (af & bf[None, :] & ((a & LOW32) == (b & LOW32)[None, :])).sum(axis=1)
    filled = af.sum(axis=1)
    both = (filled != 0) & bool(bf.any())
    if freq is None:
        est = np.where(both, np.float32(eq) / np.float32(n_hashes), np.float32(0)).astype(np.float64)
    else:
        J = np.where(both, eq / n_hashes, 0.0)
        est = java_round((J * (float(query_freq) + np.asarray(freq, dtype=np.float64))) / (J + 1))
    keep = _slot_mask(len(a), key_slot, query_slot) & (filled != 0)
    return np.where(keep, est, NEG)
