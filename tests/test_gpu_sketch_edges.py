"""The streaming-sketch kernels (ops/csrc/fps_sketch.cu) against the exact replays of tests/sketch_ref.py.

Updates (Bloom ``red.or``, tug-of-war ``red.add.s32``, MinHash ``red.min.u64``) are compared bit for bit on the raw
int32 rows, including the hash half of the MinHash slots and the rows and padding columns no occurrence touches.
The batches are larger than one grid-stride round of the capped grid, half of every batch goes to one key, the tweet
ids cover negative values and values past 2^32, and the hash counts cross the tug-of-war's 64-bit seed words.  The
same sweep runs through ``MultiShardTable`` with 1, 3 and 16 shards under hash, range and LUT layouts.

The per-key scans (``fps_bloom_query``, ``fps_sketch_query``) are called directly on crafted rows with padded strides,
``key_slot`` filters and, on the narrow rows, more rows than one warp-stride round.  The rows sit at the front of a
buffer twice their size that holds random words, so a row or stride error reads defined memory and shows as a wrong
score.  The tug-of-war and MinHash results must equal the replay exactly; the Bloom estimate must be within
``1e-6 * max(1, n(A u B))``.  Last, the two-level top-K of ``DeviceSketch`` over shards of more than 65 536 rows."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import rows_ref, sketch_ref
from tests.test_gpu_rows_edges import _layout

pytestmark = pytest.mark.gpu

NEG = sketch_ref.NEG
UPDATE_BLOCKS_PER_SM = 16            # fps_sketch_update caps its grid at num_sms * 16 blocks of 256
QUERY_WARPS_PER_SM = 64              # the scans: num_sms * 8 blocks of 8 warps, one warp per row
HASHES = [1, 3, 31, 32, 33, 63, 64, 65, 100, 128]
ARRAY_SIZES = [1, 31, 32, 33, 1000, 1024, 4096, 1_000_003]


def _sm():
    from fps_b200.ops import native

    torch.cuda.set_device(0)
    return native.sm_count(0)


def _dev():
    return torch.device("cuda", 0)


# ---- updates ------------------------------------------------------------------------------------------------------
def _words(kind, num_hashes, array_size):
    return {"bloom": sketch_ref.bloom_words(array_size), "tow": num_hashes, "minhash": 2 * num_hashes}[kind]


def _batch(rng, n_keys, num_hashes, sm):
    """(keys, tweets): more work items than one grid-stride round, half the occurrences on key 1, the last
    ``n_keys // 8`` keys untouched, tweet ids over the whole int64 range with small, negative and > 2^32 ids."""
    rounds = 2.5
    n = int(rounds * sm * UPDATE_BLOCKS_PER_SM * 256 / num_hashes) + 7
    assert n * num_hashes > 2 * sm * UPDATE_BLOCKS_PER_SM * 256
    touched = max(2, n_keys - n_keys // 8)
    keys = rng.integers(0, touched, n)
    keys[: n // 2] = 1
    base = rng.integers(0, 1 << 20, n)
    tweets = np.select([rng.random(n) < 0.25, rng.random(n) < 0.33, rng.random(n) < 0.5],
                       [base, -base - 1, base + (rng.integers(1, 1 << 30, n) << 32)],
                       rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64))
    tweets[:64] = base[:64] + (np.arange(64) << 32)                  # equal low halves, different high halves
    p = rng.permutation(n)
    return keys[p].astype(np.int32), tweets[p].astype(np.int64)


def _replay(kind, keys, tweets, n_keys, num_hashes, array_size):
    if kind == "bloom":
        return sketch_ref.bloom_update(keys, tweets, n_keys, num_hashes, array_size)
    if kind == "tow":
        return sketch_ref.tow_update(keys, tweets, n_keys, num_hashes)
    return sketch_ref.minhash_update(keys, tweets, n_keys, num_hashes)


def _init(kind):
    return -1 if kind == "minhash" else 0


def _update(tab, kind, keys, tweets, num_hashes, array_size):
    from fps_b200.ops import native

    native.sketch_update(tab, kind, torch.from_numpy(keys).to(_dev()), torch.from_numpy(tweets).to(_dev()),
                         num_hashes, array_size)


UPDATE_CASES = ([("bloom", h, 1000) for h in HASHES] + [("bloom", 3, a) for a in ARRAY_SIZES if a != 1000]
                + [("bloom", 65, 33), ("bloom", 33, 4096)]
                + [("tow", h, 0) for h in HASHES] + [("minhash", h, 0) for h in HASHES])


@pytest.mark.parametrize("kind,num_hashes,array_size", UPDATE_CASES)
def test_update_rows_bit_for_bit(kind, num_hashes, array_size):
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    sm = _sm()
    rng = np.random.default_rng(num_hashes * 7919 + array_size + len(kind))
    words = _words(kind, num_hashes, array_size)
    n_keys = 3 if array_size > 100_000 else 257
    capacity = n_keys + 5                                             # rows past the keys are never addressed
    t = ShardedTable(capacity, words, init="zeros")
    rows = t.local.view(torch.int32)
    rows.fill_(_init(kind))
    keys, tweets = _batch(rng, n_keys, num_hashes, sm)
    half = keys.size // 3                                             # two launches: the second folds into the first
    _update(t.table_c, kind, keys[:half], tweets[:half], num_hashes, array_size)
    _update(t.table_c, kind, keys[half:], tweets[half:], num_hashes, array_size)
    torch.cuda.synchronize()
    got = rows.cpu().numpy()
    want = np.full_like(got, _init(kind))
    want[:n_keys, :words] = _replay(kind, keys, tweets, n_keys, num_hashes, array_size)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (bad[:5], got[tuple(bad[0])], want[tuple(bad[0])])

    # n = 0 launches nothing and changes nothing; an unknown kind is refused before any launch
    before = rows.clone()
    empty = np.zeros(0, dtype=np.int32)
    _update(t.table_c, kind, empty, empty.astype(np.int64), num_hashes, array_size)
    k1 = torch.from_numpy(keys[:8]).to(_dev())
    t1 = torch.from_numpy(tweets[:8]).to(_dev())
    code = native.lib().fps_sketch_update(C.byref(t.table_c), 3, C.c_void_p(k1.data_ptr()), C.c_void_p(t1.data_ptr()),
                                          C.c_longlong(8), int(num_hashes), int(array_size), sm,
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert code == -1007
    torch.cuda.synchronize()
    assert torch.equal(rows, before)
    t.close()


SHARD_CASES = [("bloom", 3, 1000), ("bloom", 65, 33), ("tow", 65, 0), ("minhash", 33, 0)]


@pytest.mark.parametrize("kind,num_hashes,array_size", SHARD_CASES)
@pytest.mark.parametrize("partition", ["hash", "range", "lut"])
@pytest.mark.parametrize("num_shards", [1, 3, 16])
def test_update_through_shard_layouts(num_shards, partition, kind, num_hashes, array_size):
    sm = _sm()
    rng = np.random.default_rng(num_shards * 31 + num_hashes + len(partition))
    words = _words(kind, num_hashes, array_size)
    m, tc, loc, n_ids = _layout(num_shards, partition, words)
    for s in m.shards:
        s.view(torch.int32).fill_(_init(kind))
    keys, tweets = _batch(rng, n_ids, num_hashes, sm)
    _update(tc, kind, keys, tweets, num_hashes, array_size)
    torch.cuda.synchronize()
    got = np.stack([s.view(torch.int32).cpu().numpy() for s in m.shards])
    ids = np.arange(n_ids)
    owner, slot = rows_ref.locate(ids, **loc)
    assert rows_ref.place(ids, np.zeros((n_ids, 1), np.float32), owner, slot, num_shards, m.rows_per_shard,
                          m.stride) is not None                       # every id has a slot in some shard
    want = np.full((num_shards, m.rows_per_shard, m.stride), _init(kind), dtype=np.int32)
    want[owner, slot, :words] = _replay(kind, keys, tweets, n_ids, num_hashes, array_size)
    assert np.array_equal(got, want)
    m.close()


# ---- direct scans -------------------------------------------------------------------------------------------------
def _guarded(a, rng):
    """``a`` (int32, 2-D) on the device at the front of a buffer of twice its size plus slack, the rest random."""
    flat = torch.from_numpy(rng.integers(-2 ** 31, 2 ** 31 - 1, 2 * a.size + 256, dtype=np.int64).astype(np.int32))
    flat[: a.size] = torch.from_numpy(np.ascontiguousarray(a).ravel())
    return flat.to(_dev())[: a.size].view(a.shape)


def _row_counts(sm):
    return [1, 7, 2 * QUERY_WARPS_PER_SM * sm + 13]


def _bloom_rows(rng, n_rows, m, stride):
    """Bloom rows inside the first ``m`` bits with set-bit counts from 0 to all ``m``; junk in the padding words."""
    n_words = (m + 31) // 32
    kind = rng.integers(0, 5, n_rows)
    bits = np.zeros((n_rows, n_words * 32), dtype=bool)
    for r in range(n_rows):
        if kind[r] == 1:                                                # a few bits: where float cancels worst
            bits[r, rng.choice(m, min(m, int(rng.integers(1, 12))), replace=False)] = True
        elif kind[r] >= 2:
            bits[r, :m] = rng.random(m) < (0.02, 0.3, 0.9)[kind[r] - 2]
    rows = rng.integers(-2 ** 31, 2 ** 31 - 1, (n_rows, stride), dtype=np.int64).astype(np.int32)
    rows[:, :n_words] = np.packbits(bits, axis=1, bitorder="little").view(np.int32)
    return rows


def _full(m):
    bits = np.zeros(((m + 31) // 32) * 32, dtype=bool)
    bits[:m] = True
    return np.packbits(bits, bitorder="little").view(np.int32)


def _check_bloom(rows_np, n_words, q_np, m, k, key_slot=None, query_slot=0, rng=None):
    from fps_b200.ops import native

    rows = _guarded(rows_np, rng)
    q = torch.from_numpy(q_np.copy()).to(_dev())
    ks = None if key_slot is None else torch.from_numpy(key_slot).to(_dev())
    est = torch.full((len(rows_np),), 12345.0, device=_dev())
    native.bloom_query(rows, n_words, q, float(m), float(k), est, key_slot=ks, query_slot=query_slot)
    got = est.cpu().numpy().astype(np.float64)
    want, nU = sketch_ref.bloom_query(rows_np, n_words, q_np, float(m), float(k), key_slot, query_slot)
    neg = want == NEG
    assert np.array_equal(got == NEG, neg), np.nonzero((got == NEG) != neg)[0][:5]
    tol = 1e-6 * np.maximum(1.0, np.where(neg, 1.0, nU))
    err = np.abs(got - want)
    assert (err[~neg] <= tol[~neg]).all(), (np.max(err[~neg] / tol[~neg]), np.argmax(err[~neg] / tol[~neg]))
    return got


BLOOM_CASES = [(w, 32 * w - 5) for w in (1, 31, 32, 33, 128, 129)] + [(128, 4096), (31251, 1_000_003)]


@pytest.mark.parametrize("n_words,m", BLOOM_CASES)
def test_bloom_query(n_words, m):
    sm = _sm()
    rng = np.random.default_rng(m)
    k = 3
    assert (m + 31) // 32 == n_words
    counts = [1, 7, 300] if n_words > 1000 else _row_counts(sm)
    for n_rows in counts:
        for pad in (0, 3):
            rows = _bloom_rows(rng, n_rows, m, n_words + pad)
            if n_rows > 1:
                rows[0, :n_words] = 0                                   # empty: not a key
                rows[-1, :n_words] = _full(m)                           # saturated key row
            qb = np.zeros(n_words * 32, dtype=bool)
            qb[rng.choice(m, min(m, 5), replace=False)] = True
            q = np.packbits(qb, bitorder="little").view(np.int32)      # five bits, as in a rare word
            _check_bloom(rows, n_words, q, m, k, rng=rng)
            q2 = _bloom_rows(rng, 1, m, n_words)[0][:n_words].copy()
            ks = rng.integers(-1, 3, n_rows).astype(np.int32)
            _check_bloom(rows, n_words, q2, m, k, key_slot=ks, query_slot=1, rng=rng)
            got = _check_bloom(rows, n_words, _full(m), m, k, rng=rng)  # saturated query: nothing is a key
            assert (got == NEG).all()
            r0 = rows[n_rows // 2, :n_words].copy()                       # the union alone saturates for one row
            comp = ~r0 & _full(m)
            if r0.any() and comp.any():
                got = _check_bloom(rows, n_words, comp, m, k, rng=rng)
                assert got[n_rows // 2] == NEG


@pytest.mark.parametrize("m", [65537, 1_000_003])
def test_bloom_estimate_of_sparse_filters_does_not_cancel(m):
    """|A| = 5, |B| = 7, |A u B| = 10 bits of a filter whose width is not a power of two: c/m rounded in float
    before ``1 - c/m`` was off by 1.6e-5 (m = 65537) and 1.1% (m = 1000003) of the estimate."""
    _sm()
    rng = np.random.default_rng(m)
    n_words = (m + 31) // 32
    pos = rng.choice(m, 10, replace=False)
    q = np.zeros(n_words * 32, dtype=bool)
    q[pos[:5]] = True
    rows = np.zeros((3, n_words * 32), dtype=bool)
    rows[0, pos[3:]] = True                                               # shares two bits with the query
    rows[1, pos[5:]] = True                                               # disjoint
    rows[2, pos[:5]] = True                                               # equal
    def pack(bits):
        return np.packbits(bits, axis=-1, bitorder="little").view(np.int32)

    got = _check_bloom(pack(rows), n_words, pack(q), m, 3, rng=rng)
    assert got[1] != NEG and got[2] > got[0] > got[1]


def _tow_means(n_hashes):
    """num_means values forming 1, 2, 3, 31 and 32 groups where possible, one above ``n_hashes``, and one past the
    32-group limit where there is one."""
    out = set()
    for groups in (1, 2, 3, 31, 32):
        for nm in range(1, 200):
            if sketch_ref.tow_groups(n_hashes, nm)[1] == groups:
                out.add(nm)
                break
    out.add(n_hashes + 3)
    for nm in range(33, 200):
        if sketch_ref.tow_groups(n_hashes, nm)[1] > 32:
            out.add(nm)
            break
    return sorted(out)


TOW_HASHES = [1, 31, 32, 33, 64, 65, 200, 1024]


def test_tow_sweep_reaches_every_grouping():
    """1, 2, 3, 31 and 32 groups, a ragged last group, num_means above n_hashes and past the 32-group limit."""
    formed, ragged, over, refused = set(), False, False, False
    for n in TOW_HASHES:
        for nm in _tow_means(n):
            size, g = sketch_ref.tow_groups(n, nm)
            formed.add(g)
            ragged |= g <= 32 and n % size != 0
            over |= nm > n and g <= 32
            refused |= g > 32
    assert {1, 2, 3, 31, 32} <= formed and ragged and over and refused


@pytest.mark.parametrize("n_hashes", TOW_HASHES)
def test_tow_query_exact(n_hashes):
    from fps_b200.ops import native

    sm = _sm()
    rng = np.random.default_rng(n_hashes)
    means = _tow_means(n_hashes)
    limit = 2 ** 17
    for n_rows in _row_counts(sm):
        stride = n_hashes + (5 if n_rows > 1 else 0)
        rows = rng.integers(-limit - 9, limit + 9, (n_rows, stride)).astype(np.int32)
        rows[0, :n_hashes] = limit                                     # every group mean tied
        if n_rows > 2:
            rows[1, :n_hashes] = 0
            rows[2, :n_hashes] = -limit - 3
        d_rows = _guarded(rows, rng)
        for q in (rng.integers(-limit - 9, limit + 9, n_hashes).astype(np.int32),
                  np.full(n_hashes, limit + 1, dtype=np.int32)):
            ks = rng.integers(-1, 2, n_rows).astype(np.int32)
            for key_slot in (None, ks):
                for nm in means:
                    est = torch.full((n_rows,), 12345.0, device=_dev())
                    args = ("tow", d_rows, n_hashes, n_hashes, torch.from_numpy(q).to(_dev()), est)
                    kw = dict(num_means=nm, key_slot=None if key_slot is None else torch.from_numpy(key_slot).to(
                        _dev()), query_slot=1)
                    if sketch_ref.tow_groups(n_hashes, nm)[1] > 32:
                        with pytest.raises(RuntimeError, match="-1008"):
                            native.sketch_query(*args, **kw)
                        continue
                    native.sketch_query(*args, **kw)
                    want = sketch_ref.tow_query(rows, q, n_hashes, nm, key_slot, 1).astype(np.float32)
                    got = est.cpu().numpy()
                    assert np.array_equal(got, want), (nm, np.nonzero(got != want)[0][:5])


def _mh_rows(rng, n_rows, n_hashes, q, stride):
    """u64 signature rows sharing tweet halves with ``q`` at random slots, with empty slots and one never-filled row."""
    sig = np.full((n_rows, stride // 2), sketch_ref.ALL_ONES, dtype=np.uint64)
    hi = rng.integers(0, 2 ** 32, (n_rows, n_hashes), dtype=np.uint64) << np.uint64(32)
    lo = rng.integers(0, 2 ** 32, (n_rows, n_hashes), dtype=np.uint64)
    share = rng.random((n_rows, n_hashes)) < rng.random((n_rows, 1))
    lo = np.where(share, q[None, :n_hashes] & sketch_ref.LOW32, lo)
    body = hi | lo
    body[rng.random((n_rows, n_hashes)) < 0.1] = sketch_ref.ALL_ONES
    sig[:, :n_hashes] = body
    sig[:, n_hashes:] = rng.integers(0, 2 ** 63, (n_rows, stride // 2 - n_hashes), dtype=np.uint64)
    if n_rows > 1:
        sig[-1, :n_hashes] = sketch_ref.ALL_ONES                        # never filled: not a key
    return sig.view(np.int32)


def _mh_query(rows_np, q_np, n_hashes, rng, key_slot=None, freq=None, query_freq=0.0):
    from fps_b200.ops import native

    est = torch.full((len(rows_np),), 12345.0, device=_dev())
    native.sketch_query("minhash", _guarded(rows_np, rng), 2 * n_hashes, n_hashes,
                        torch.from_numpy(q_np.view(np.int32).copy()).to(_dev()), est,
                        key_slot=None if key_slot is None else torch.from_numpy(key_slot).to(_dev()), query_slot=2,
                        freq=None if freq is None else torch.from_numpy(freq).to(_dev()), query_freq=query_freq)
    want = sketch_ref.minhash_query(rows_np, q_np.view(np.int32), n_hashes, key_slot, 2, freq, query_freq)
    got = est.cpu().numpy()
    assert np.array_equal(got, want.astype(np.float32)), np.nonzero(got != want.astype(np.float32))[0][:5]
    return got


def _float_count(eq, n, F):
    """The co-occurrence count as a float kernel rounds it: ``rintf(j * F / (j + 1))`` in fp32."""
    j = np.asarray(eq, dtype=np.float32) / np.float32(n)
    return np.rint(j * np.asarray(F, dtype=np.float32) / (j + np.float32(1)))


@pytest.mark.parametrize("n_hashes", [1, 3, 31, 32, 33, 100])
def test_minhash_query_exact(n_hashes):
    sm = _sm()
    rng = np.random.default_rng(n_hashes + 99)
    q = rng.integers(0, 2 ** 64 - 1, n_hashes, dtype=np.uint64)
    q[rng.random(n_hashes) < 0.1] = sketch_ref.ALL_ONES
    for n_rows in _row_counts(sm):
        stride = 2 * n_hashes + (4 if n_rows > 1 else 0)
        rows = _mh_rows(rng, n_rows, n_hashes, q, stride)
        freq = rng.integers(0, 3000, n_rows).astype(np.float32)
        ks = rng.integers(0, 4, n_rows).astype(np.int32)
        for key_slot in (None, ks):
            _mh_query(rows, q, n_hashes, rng, key_slot)
            _mh_query(rows, q, n_hashes, rng, key_slot, freq=freq, query_freq=17.0)
        _mh_query(rows, np.full(n_hashes, sketch_ref.ALL_ONES), n_hashes, rng)     # empty query: J = 0
        if n_rows > 1:
            got = _mh_query(rows, q, n_hashes, rng)
            assert got[-1] == NEG

    # exact halves: rows equal to a full query (J = 1) with odd frequency sums
    full = rng.integers(0, 2 ** 63, n_hashes, dtype=np.uint64)
    same = np.tile(full, (6, 1))
    same[:, :] ^= np.uint64(1) << np.uint64(40)                          # other hash halves, same tweet ids
    freq = np.array([0, 1, 2, 4, 6, 1000], dtype=np.float32)
    got = _mh_query(same.view(np.int32), full, n_hashes, rng, freq=freq, query_freq=3.0)
    assert got.tolist() == [(3 + f + 1) // 2 for f in freq.astype(int)]

    # every (eq, F) whose float rounding differs from the double one, as far as n_hashes gives any
    eq, F = np.meshgrid(np.arange(1, n_hashes + 1), np.arange(2, 2000), indexing="ij")
    J = eq / n_hashes
    differ = _float_count(eq, n_hashes, F) != sketch_ref.java_round((J * F) / (J + 1))
    pairs = list(zip(eq[differ].tolist(), F[differ].tolist()))
    if n_hashes == 100:
        assert (4, 819) in pairs and len(pairs) > 100
    pairs = pairs[:: max(1, len(pairs) // 64)]
    if pairs:
        rows = np.empty((len(pairs), n_hashes), dtype=np.uint64)
        for r, (eq, _) in enumerate(pairs):
            rows[r] = full ^ (np.uint64(1) << np.uint64(45))
            rows[r, eq:] = full[eq:] ^ np.uint64(1)                      # another tweet id past the first eq slots
        freq = np.array([F - 1 for _, F in pairs], dtype=np.float32)
        got = _mh_query(rows.view(np.int32), full, n_hashes, rng, freq=freq, query_freq=1.0)
        assert np.array_equal(got, sketch_ref.java_round([(e / n_hashes * F) / (e / n_hashes + 1) for e, F in pairs]))


# ---- top-K over a large shard ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_local,n_keys", [(2 * 32768 - 1, 65000), (2 * 32768 + 1, 1500), (100_003, 99_000)])
def test_two_level_topk(n_local, n_keys):
    from fps_b200.models.sketch.device import DeviceSketch
    from fps_b200.models.sketch.hashing import java_string_hash

    _sm()
    rng = np.random.default_rng(n_local)
    m, k = 1000, 3
    sk = DeviceSketch("bloom", n_local, k, m)
    words = sk.words
    assert sk.rows_i32.shape[0] == n_local
    names = [f"w{i}" for i in range(n_keys)]
    for w in names:
        sk.interner(java_string_hash(w))
    assert len(sk.interner) == n_keys
    rows = _bloom_rows(rng, n_local, m, sk.rows_i32.shape[1])
    rows[:, words:] = 0
    dup = rng.choice(n_keys, 200, replace=False)
    rows[dup[100:]] = rows[dup[:100]]                                   # tied scores
    sat = int(rng.integers(10, n_keys))
    rows[sat, :words] = _full(m)
    qslot = 5
    rows[qslot, :words] = 0
    rows[qslot, :words] = np.packbits(rng.random(words * 32) < 0.05, bitorder="little").view(np.int32)
    rows[qslot, words - 1] &= (1 << (m % 32)) - 1
    sk.rows_i32.copy_(torch.from_numpy(rows))
    est = sk._local_scores(names[qslot], 1, None, False)
    want, nU = sketch_ref.bloom_query(rows, words, rows[qslot], float(m), float(k))
    want[n_keys:] = NEG
    got = est.cpu().numpy().astype(np.float64)
    assert got[sat] == NEG
    assert np.array_equal(got == NEG, want == NEG)
    fin = want != NEG
    assert (np.abs(got - want)[fin] <= 1e-6 * np.maximum(1.0, nU[fin])).all()
    ids = sk.table.local_ids().cpu().numpy()
    n_finite = int((got > -1e38).sum())
    for K in (1, 50, 2048):
        s, gid = sk._local_topk(est, K)
        tv, ti = torch.topk(est, K)
        assert torch.equal(s, tv)
        s, gid, ti = s.cpu().numpy(), gid.cpu().numpy(), ti.cpu().numpy()
        real = s > -1e38
        assert (gid[real] >= 0).all()
        uniq = real & np.array([(got == v).sum() == 1 for v in s])
        assert np.array_equal(gid[uniq], ids[ti[uniq]])
        out = sk.query_local(names[qslot], K)
        assert len(out) == min(K, n_finite)
        assert [sc for sc, _ in out] == s[: len(out)].tolist()
        assert java_string_hash(names[sat]) not in {key for _, key in out}
    sk.close()
