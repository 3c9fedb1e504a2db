"""Sketch update kernels (red.or / red.add.s32 / red.min.u64) vs the host oracle with the same hashes."""
import pytest
import torch

pytestmark = pytest.mark.gpu

_W = [["cat", "dog"], ["cat", "dog"], ["cat", "dog", "fish"], ["cat", "dog"], ["bird"], ["bird", "fish"],
      ["cat", "dog"], ["fish"], ["cat", "dog"], ["bird"], ["cat", "dog"], ["cat", "fish"]] * 5
TWEETS = [(str(1000 + i), ws) for i, ws in enumerate(_W)]


def _by_word(model):
    from fps_b200.models.sketch.hashing import java_string_hash
    d = dict(model)
    return {w: d[java_string_hash(w)] for w in ["cat", "dog", "fish", "bird"]}


def test_bloom_device_equals_oracle_and_ranks_cooccurrence():
    from fps_b200.models.sketch.device import DeviceSketch, bloom_positions64
    from fps_b200.models.sketch.hashing import java_string_hash

    torch.cuda.set_device(0)
    sk = DeviceSketch("bloom", 64, 3, 1024)
    sk.update(TWEETS[:30]); sk.update(TWEETS[30:])
    got = _by_word(sk.model())
    for w in got:
        ref = set()
        for tid, ws in TWEETS:
            if w in ws:
                ref.update(bloom_positions64(int(tid), 3, 1024))
        assert got[w] == frozenset(ref)
    top = sk.query_local("cat", 2)
    assert {k for _, k in top} == {java_string_hash("cat"), java_string_hash("dog")}
    sk.close()


def test_tow_and_minhash_device_equal_oracle():
    from fps_b200.models.sketch.device import DeviceSketch, minhash_packed64, tow_bits64
    from fps_b200.models.sketch.hashing import java_string_hash

    torch.cuda.set_device(0)
    tow = DeviceSketch("tow", 64, 96)
    tow.update(TWEETS)
    got = _by_word(tow.model())
    for w in got:
        ref = [0] * 96
        for tid, ws in TWEETS:
            if w in ws:
                ref = [a + b for a, b in zip(ref, tow_bits64(int(tid), 96))]
        assert got[w] == ref
    assert {k for _, k in tow.query_local("dog", 2)} == {java_string_hash("cat"), java_string_hash("dog")}
    tow.close()
    mh = DeviceSketch("minhash", 64, 32)
    mh.update(TWEETS)
    got = _by_word(mh.model())
    for w in got:
        ref = None
        for tid, ws in TWEETS:
            if w in ws:
                p = minhash_packed64(int(tid), 32)
                ref = p if ref is None else [min(a, b) for a, b in zip(ref, p)]
        assert got[w] == [r & 0xFFFFFFFF for r in ref]
    top = mh.query_local("cat", 2)
    assert top[0][1] == java_string_hash("cat") and top[1][1] == java_string_hash("dog")
    mh.close()


# ---- device predict == host predict (the host scoring functions on the device hash family) -----------------
SLOTTED = [(tid, ws, i % 3) for i, (tid, ws) in enumerate(TWEETS)]


def _rank_close(dev_list, host_list, K, tol=1e-4):
    """Same scores best-first; keys equal wherever the scores are not tied."""
    assert len(dev_list) == min(K, len(host_list))
    for (ds, dk), (hs, hk) in zip(dev_list, host_list):
        assert abs(ds - hs) <= tol * max(1.0, abs(hs)), (dev_list, host_list[:K])
    strict = [i for i in range(len(dev_list))
              if all(abs(host_list[i][0] - host_list[j][0]) > 1e-6 for j in range(len(host_list)) if j != i)]
    for i in strict:
        assert dev_list[i][1] == host_list[i][1]


def test_tow_median_of_means_query_equals_host_predict():
    from fps_b200.models.sketch.device import DeviceSketch
    from fps_b200.models.sketch.hashing import java_string_hash
    from fps_b200.models.sketch.jobs import median_of_means, tugOfWarPredict

    torch.cuda.set_device(0)
    n, means, K = 96, 6, 3
    sk = DeviceSketch("tow", 64, n)
    sk.update(TWEETS)
    model = sk.model()
    d = dict(model)
    for w in ["cat", "fish", "bird"]:
        target = d[java_string_hash(w)]
        host = sorted(((median_of_means(v, target, n, means), k) for k, v in d.items()), reverse=True)
        _rank_close(sk.query_local(w, K, num_means=means), host, K)
    sk.close()
    out = dict(tugOfWarPredict([(7, "cat"), (8, "bird")], model, n, means, K, 1, 1, 100, backend="device"))
    target = d[java_string_hash("cat")]
    host = sorted(((median_of_means(v, target, n, means), k) for k, v in d.items()), reverse=True)
    _rank_close(out[7], host, K)
    assert set(out) == {7, 8}


def test_minhash_jaccard_and_cooccurrence_query_equal_host_predict():
    from fps_b200.models.sketch.device import DeviceSketch
    from fps_b200.models.sketch.hashing import java_string_hash
    from fps_b200.models.sketch.jobs import minhashPredict, word_count
    from fps_b200.models.sketch.utils import java_round

    torch.cuda.set_device(0)
    n = 32
    mh = DeviceSketch("minhash", 64, n)
    mh.update(TWEETS)
    model = mh.model()
    d = dict(model)
    freq = word_count(TWEETS)
    assert mh.word_count() == freq                             # keyed occurrence count on the device
    for w in ["cat", "fish"]:
        q = java_string_hash(w)
        jac = {k: sum(1 for a, b in zip(v, d[q]) if a == b) / n for k, v in d.items()}
        host_j = sorted(((j, k) for k, j in jac.items()), reverse=True)
        _rank_close(mh.query_local(w, 4), host_j, 4)
        host_c = sorted(((float(java_round(j * (freq[q] + freq[k]) / (j + 1))), k) for k, j in jac.items()),
                        reverse=True)
        _rank_close(mh.query_local(w, 4, cooccurrence=True), host_c, 4)
    mh.close()
    res = dict(minhashPredict(["cat"], TWEETS, model, n, 4, 1, 1, 100, backend="device"))
    q = java_string_hash("cat")
    got = res[q]
    assert got[0][0] == q and got[0][1] == java_round(1.0 * (2 * freq[q]) / 2.0)     # J(cat, cat) = 1
    assert [c for _, c in got] == sorted((c for _, c in got), reverse=True)


@pytest.mark.parametrize("kind", ["bloom", "tow"])
def test_time_aware_sketches_score_same_slot_keys_only(kind):
    from fps_b200.models.sketch.device import DeviceSketch
    from fps_b200.models.sketch.hashing import java_string_hash
    from fps_b200.models.sketch.jobs import (median_of_means, timeAwareBloomFilter, timeAwareBloomPredict,
                                             timeAwareTugOfWar, timeAwareTugOfWarPredict)
    from fps_b200.models.sketch.utils import bloomEq

    torch.cuda.set_device(0)
    n, m, K = (96, 0, 3) if kind == "tow" else (3, 1024, 3)
    if kind == "tow":
        model = timeAwareTugOfWar(SLOTTED, n, 1, 1, backend="device")
    else:
        model = timeAwareBloomFilter(SLOTTED, m, n, 1, 1, backend="device")
    d = dict(model)
    assert all(isinstance(k, tuple) and len(k) == 2 for k in d)                 # keyed (wordHash, slot)
    cat = java_string_hash("cat")
    slots = sorted(s for (h, s) in d if h == cat)
    assert slots == [0, 1, 2]
    if kind == "tow":
        out = dict(timeAwareTugOfWarPredict([(5, "cat")], model, n, 4, K, 1, 1, 100, backend="device"))
    else:
        out = dict(timeAwareBloomPredict([(5, "cat")], model, m, n, K, 1, 1, 100, backend="device"))
    assert sorted(out) == [(5, s) for s in slots]                                # one answer per time slot
    for s in slots:
        target = d[(cat, s)]
        if kind == "tow":
            host = sorted(((median_of_means(v, target, n, 4), k) for (k, ks), v in d.items() if ks == s), reverse=True)
        else:
            nA = bloomEq(m, n, len(target))
            host = sorted(((nA + bloomEq(m, n, len(v)) - bloomEq(m, n, len(target | v)), k)
                           for (k, ks), v in d.items() if ks == s), reverse=True)
        _rank_close(out[(5, s)], host, K, tol=1e-3)


def test_device_train_adapters_and_bloom_predict_job():
    from fps_b200.models.sketch.device import DeviceSketch
    from fps_b200.models.sketch.hashing import java_string_hash
    from fps_b200.models.sketch.jobs import bloomFilter, bloomPredict, minhash, tugOfWar
    from fps_b200.models.sketch.utils import bloomEq

    torch.cuda.set_device(0)
    for job, kind, args in ((bloomFilter, "bloom", (1024, 3)), (tugOfWar, "tow", (64,)), (minhash, "minhash", (16,))):
        model = job(TWEETS, *args, 1, 1, backend="device")
        nh, arr = (args[1], args[0]) if kind == "bloom" else (args[0], 0)
        sk = DeviceSketch(kind, 64, nh, arr)
        sk.update(TWEETS)
        assert dict(model) == dict(sk.model())
        sk.close()
    model = bloomFilter(TWEETS, 1024, 3, 1, 1, backend="device")
    d = dict(model)
    out = dict(bloomPredict([(1, "dog"), (2, "unknown-word")], model, 1024, 3, 2, 1, 1, 100, backend="device"))
    target = d[java_string_hash("dog")]
    nA = bloomEq(1024, 3, len(target))
    host = sorted(((nA + bloomEq(1024, 3, len(v)) - bloomEq(1024, 3, len(target | v)), k) for k, v in d.items()),
                  reverse=True)
    _rank_close(out[1], host, 2, tol=1e-3)
    assert out[2] == []
