"""The sketch replays of tests/sketch_ref.py against the scalar host oracles they vectorise (CPU only)."""
import math

import numpy as np
import pytest

from tests import sketch_ref

TWEETS = np.array([0, 1, 7, 1000, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 7, 7 + 2 ** 40,
                   7 + 2 ** 62, 2 ** 63 - 1, -1, -7, -(2 ** 32), -(2 ** 63), 123456789012345], dtype=np.int64)


def test_ids_that_differ_above_bit_32_hash_apart():
    h = [sketch_ref.hash64(TWEETS[TWEETS == t], 0)[0] for t in (7, 2 ** 32 + 7, 2 ** 40 + 7)]
    assert len(set(h)) == 3


@pytest.mark.parametrize("seed", [0, 1, 5, 63, 64, 1000])
def test_hash64_equals_scalar(seed):
    from fps_b200.models.sketch.hashing import hash64

    got = sketch_ref.hash64(TWEETS, seed)
    assert got.dtype == np.uint64
    assert [int(v) for v in got] == [hash64(int(t), seed) for t in TWEETS]


@pytest.mark.parametrize("num_hashes", [1, 3, 63, 64, 65, 130])
def test_update_replays_equal_scalar_oracles(num_hashes):
    from fps_b200.models.sketch.device import bloom_positions64, minhash_packed64, tow_bits64

    rng = np.random.default_rng(num_hashes)
    n_keys = 5
    keys = rng.integers(0, n_keys - 1, 3 * TWEETS.size)            # the last key stays untouched
    tweets = np.tile(TWEETS, 3)
    for array_size in (1, 31, 33, 1000, 4096, 1_000_003):
        got = sketch_ref.bloom_update(keys, tweets, n_keys, num_hashes, array_size)
        assert got.shape == (n_keys, sketch_ref.bloom_words(array_size)) and got.dtype == np.int32
        bits = np.unpackbits(got.view(np.uint8), axis=1, bitorder="little")
        for key in range(n_keys):
            want = set()
            for t in tweets[keys == key]:
                want.update(bloom_positions64(int(t), num_hashes, array_size))
            assert set(np.nonzero(bits[key])[0].tolist()) == want
    got = sketch_ref.tow_update(keys, tweets, n_keys, num_hashes)
    for key in range(n_keys):
        want = np.zeros(num_hashes, dtype=np.int64)
        for t in tweets[keys == key]:
            want += tow_bits64(int(t), num_hashes)
        assert got[key].tolist() == want.tolist()
    got = sketch_ref.minhash_update(keys, tweets, n_keys, num_hashes)
    assert got.shape == (n_keys, 2 * num_hashes)
    sig = got.view(np.uint64)
    for key in range(n_keys):
        want = [2 ** 64 - 1] * num_hashes
        for t in tweets[keys == key]:
            want = [min(a, b) for a, b in zip(want, minhash_packed64(int(t), num_hashes))]
        assert [int(v) for v in sig[key]] == want
    assert (got[n_keys - 1] == -1).all()


@pytest.mark.parametrize("n_hashes", [1, 5, 31, 32, 33, 64, 65, 200, 1024])
def test_tow_query_equals_median_of_means(n_hashes):
    from fps_b200.models.sketch.jobs import median_of_means

    rng = np.random.default_rng(n_hashes)
    rows = rng.integers(-2 ** 17, 2 ** 17, (6, n_hashes)).astype(np.int32)
    rows[1] = rows[0]                                              # tied rows
    rows[2, : n_hashes // 2] = 0
    q = rng.integers(-2 ** 17, 2 ** 17, n_hashes).astype(np.int32)
    for num_means in sorted({1, 2, 3, 4, 7, 31, 32, n_hashes, n_hashes + 5}):
        got = sketch_ref.tow_query(rows, q, n_hashes, num_means)
        want = [median_of_means(r.tolist(), q.tolist(), n_hashes, num_means) for r in rows]
        assert got.tolist() == want, num_means
    slots = np.array([0, 2, -1, 2, 2, 0], dtype=np.int32)
    got = sketch_ref.tow_query(rows, q, n_hashes, 3, key_slot=slots, query_slot=2)
    assert (got[slots != 2] == sketch_ref.NEG).all() and (got[slots == 2] > sketch_ref.NEG).all()


def test_tow_groups_match_median_of_means():
    for n in (1, 5, 33, 200, 1024):
        for means in range(1, 70):
            size, g = sketch_ref.tow_groups(n, means)
            assert size == max(1, int(math.ceil(n / means)))
            assert g == len(range(0, n, size))


def _bits(m, n_rows, rng, density):
    words = (m + 31) // 32
    b = rng.random((n_rows, words * 32)) < density
    b[:, m:] = False
    return np.packbits(b, axis=1, bitorder="little").view(np.int32)


@pytest.mark.parametrize("m", [1000, 1024, 65537, 1_000_003])
def test_bloom_query_equals_bloomEq_where_finite(m):
    from fps_b200.models.sketch.utils import bloomEq

    rng = np.random.default_rng(m)
    k = 3
    rows = _bits(m, 8, rng, 0.3)
    rows[0] = 0                                                      # empty: not a key
    q = _bits(m, 1, rng, 0.2)[0]
    full = _bits(m, 1, rng, 1.0)[0]
    rows[1] = full                                                   # saturated row
    n_words = (m + 31) // 32
    est, nU = sketch_ref.bloom_query(rows, n_words, q, float(m), float(k))
    assert est[0] == sketch_ref.NEG and est[1] == sketch_ref.NEG
    qa = set(np.nonzero(np.unpackbits(q.view(np.uint8), bitorder="little"))[0].tolist())
    for r in range(2, len(rows)):
        b = set(np.nonzero(np.unpackbits(rows[r].view(np.uint8), bitorder="little"))[0].tolist())
        want = bloomEq(m, k, len(qa)) + bloomEq(m, k, len(b)) - bloomEq(m, k, len(qa | b))
        assert est[r] == want
        assert nU[r] == bloomEq(m, k, len(qa | b))
    with pytest.raises(ValueError):
        bloomEq(m, k, m)                                             # the host formula has no value there
    est, _ = sketch_ref.bloom_query(rows, n_words, full, float(m), float(k))   # saturated query
    assert (est == sketch_ref.NEG).all()
    slots = np.arange(8, dtype=np.int32) % 3 - 1
    est, _ = sketch_ref.bloom_query(rows, n_words, q, float(m), float(k), key_slot=slots, query_slot=1)
    assert (est[slots != 1] == sketch_ref.NEG).all() and (est[slots == 1] > sketch_ref.NEG).all()


def test_bloom_union_saturation_alone_is_not_a_key():
    m, k = 64, 2
    q = np.array([-1, 0], dtype=np.int32)                           # low half set
    rows = np.array([[0, -1], [0, 1]], dtype=np.int32)              # high half: the union fills every bit
    est, nU = sketch_ref.bloom_query(rows, 2, q, float(m), float(k))
    assert est[0] == sketch_ref.NEG and math.isinf(nU[0])
    assert math.isfinite(est[1])


def test_java_round():
    cases = {2.5: 3, 3.5: 4, 0.49999999999999994: 0, 12.499999999999998: 12, 0.5: 1, 1.4999999999999998: 1,
             -0.5: 0, -2.5: -2, 0.0: 0, 7.0: 7}
    got = sketch_ref.java_round(np.array(list(cases)))
    assert got.tolist() == list(cases.values())
    from fps_b200.models.sketch.utils import java_round

    assert [java_round(x) for x in cases] == list(cases.values())
    assert all(isinstance(java_round(x), int) for x in cases)


def test_minhash_query_jaccard_and_count():
    n = 100
    rows = np.full((5, n), sketch_ref.ALL_ONES, dtype=np.uint64)
    q = np.full(n, sketch_ref.ALL_ONES, dtype=np.uint64)
    q[:80] = np.arange(80, dtype=np.uint64) | (np.uint64(9) << np.uint64(32))
    rows[0, :4] = q[:4] ^ (np.uint64(5) << np.uint64(32))          # equal tweet halves, other hash halves
    rows[1, :60] = np.arange(60, dtype=np.uint64) + np.uint64(1)     # filled, no match
    rows[2, 81:] = 7                                                 # filled where the query is empty
    rows[3] = q                                                      # row 4: never filled
    r32, q32 = rows.view(np.int32), q.view(np.int32)
    jac = sketch_ref.minhash_query(r32, q32, n)
    assert jac.tolist() == [np.float32(4) / np.float32(n), 0.0, 0.0, np.float32(80) / np.float32(n), sketch_ref.NEG]
    freq = np.array([819, 3, 5, 20, 1], dtype=np.float32)
    cnt = sketch_ref.minhash_query(r32, q32, n, freq=freq, query_freq=0.0)
    assert cnt.tolist() == [31.0, 0.0, 0.0, 9.0, sketch_ref.NEG]     # 0.04 * 819 / 1.04 is 31.499999999999996
    cnt = sketch_ref.minhash_query(r32[3:4], q32, n, freq=np.array([1.0]), query_freq=4.0)
    assert cnt.tolist() == [math.floor(0.8 * 5 / 1.8 + 0.5)]
    same = np.arange(n, dtype=np.uint64).view(np.int32)               # J = 1: the count is half the sum, halves up
    for fq, fw in ((2, 3), (0, 1), (4, 7)):
        got = sketch_ref.minhash_query(same[None, :], same, n, freq=np.array([fw]), query_freq=fq)
        assert got.tolist() == [(fq + fw + 1) // 2]
    slots = np.array([3, 3, 1, 3, 3], dtype=np.int32)
    got = sketch_ref.minhash_query(r32, q32, n, key_slot=slots, query_slot=3)
    assert got[2] == sketch_ref.NEG and got[:2].tolist() == jac[:2].tolist()


def test_minhash_predict_rounds_halves_up():
    from fps_b200.models.sketch.jobs import minhashPredict

    train = [("1", ["a", "b"]), ("2", ["a"]), ("3", ["a", "b"]), ("4", ["c"])]     # f = 3, 2, 1
    model = [(h, [11, 12]) for h in _hashes("a", "b", "c")]                  # every signature equal: J = 1
    a, b, c = _hashes("a", "b", "c")
    res = dict(minhashPredict(["a", "b"], train, model, 2, 3, 1, 1, 100))
    assert dict(res[a]) == {a: 3, b: 3, c: 2}                                  # 6/2, 5/2 = 2.5 up, 4/2
    assert dict(res[b]) == {a: 3, b: 2, c: 2}                                  # 5/2 up, 4/2, 3/2 = 1.5 up


def _hashes(*words):
    from fps_b200.models.sketch.hashing import java_string_hash

    return [java_string_hash(w) for w in words]


def test_bloom_predict_skips_saturated_candidates():
    from fps_b200.models.sketch.jobs import bloomPredict, timeAwareBloomPredict
    from fps_b200.models.sketch.utils import bloomEq

    m, k = 64, 2
    a, b, c = _hashes("a", "b", "c")
    sets = {a: frozenset({1, 2, 3}), b: frozenset(range(m)), c: frozenset({2, 3, 40})}
    res = dict(bloomPredict([(1, "a"), (2, "b")], list(sets.items()), m, k, 5, 1, 1, 100))
    nA = bloomEq(m, k, 3)
    assert res[1] == [(nA, a), (nA + bloomEq(m, k, 3) - bloomEq(m, k, 4), c)]     # b's union is saturated
    assert res[2] == []                                                          # a saturated query
    res = dict(timeAwareBloomPredict([(1, "a")], [((h, 0), v) for h, v in sets.items()], m, k, 5, 1, 1, 100))
    assert [h for _, h in res[(1, 0)]] == [a, c]
