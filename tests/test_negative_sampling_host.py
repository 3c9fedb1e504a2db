"""Negatives from the items each worker has seen, and unigram noise, without a GPU: the numpy reference of the
seen-items registry against a record-by-record replay of the host tier's rule, and every refusal."""
import math

import numpy as np
import pytest

import fps_b200  # noqa: F401
from fps_b200.models.mf.common import Rating, SeenRegistryOracle, require_pointwise
from fps_b200.models.mf.device import check_negative_sampling
from fps_b200.models.w2v import check_noise


def _replay(batches, neg_rate, memory):
    """The rule of ops/csrc/fps_host.cpp:235-249, one record at a time: append to the user's queue, draw
    max(0, min(|item_ids| - |queue|, neg_rate)) negatives, then register the record's item."""
    item_ids, known, queues, out = [], set(), {}, []
    for users, items in batches:
        dom, ring, k = [], [], []
        for u, i in zip(users, items):
            q = queues.setdefault(int(u), [])
            if len(q) >= memory and q:
                q.pop(0)
            if memory > 0:
                q.append(int(i))
            dom.append(len(item_ids)); ring.append(len(q))
            k.append(max(0, min(len(item_ids) - len(q), neg_rate)))
            if int(i) not in known:
                known.add(int(i)); item_ids.append(int(i))
        out.append((dom, ring, k))
    return item_ids, out


@pytest.mark.parametrize("memory", [0, 1, 4, 128])
@pytest.mark.parametrize("neg_rate", [1, 3])
def test_registry_oracle_matches_the_record_by_record_rule(memory, neg_rate):
    rng = np.random.default_rng(7)
    batches = [(rng.integers(0, 40, size=n), rng.integers(0, 60, size=n)) for n in (1, 17, 200, 0, 55)]
    oracle = SeenRegistryOracle(num_items=60, num_users=40, neg_rate=neg_rate, user_memory=memory)
    got = [oracle.batch(u, i) for u, i in batches]
    order, want = _replay(batches, neg_rate, memory)
    np.testing.assert_array_equal(oracle.order, order)
    for (dom, ring, k), (wd, wr, wk) in zip(got, want):
        np.testing.assert_array_equal(dom, wd)
        np.testing.assert_array_equal(ring, wr)
        np.testing.assert_array_equal(k, wk)


def test_registry_oracle_by_hand():
    """Items 5, 5, 7 then 7, 9: a record's own first-seen item joins the domain from the next record on."""
    o = SeenRegistryOracle(num_items=10, num_users=4, neg_rate=2, user_memory=0)
    dom, ring, k = o.batch([0, 1, 2], [5, 5, 7])
    assert dom.tolist() == [0, 1, 1] and ring.tolist() == [0, 0, 0] and k.tolist() == [0, 1, 1]
    dom, ring, k = o.batch([3, 0], [7, 9])
    assert dom.tolist() == [2, 2] and k.tolist() == [2, 2]
    assert o.order.tolist() == [5, 7, 9]


def test_registry_oracle_ring_counts_the_users_ratings():
    o = SeenRegistryOracle(num_items=10, num_users=2, neg_rate=5, user_memory=2)
    dom, ring, k = o.batch([0, 0, 0, 1], [1, 2, 3, 4])
    assert dom.tolist() == [0, 1, 2, 3]
    assert ring.tolist() == [1, 2, 2, 1]
    assert k.tolist() == [0, 0, 0, 2]


def test_registry_oracle_counts_users_per_worker_slot():
    """With two workers, users 0 and 2 are slots 0 and 1 of worker 0."""
    o = SeenRegistryOracle(num_items=10, num_users=4, neg_rate=1, user_memory=8, user_div=2)
    _, ring, _ = o.batch([0, 2, 0], [1, 2, 3])
    assert ring.tolist() == [1, 1, 2]


def test_negative_sampling_accepts_uniform_and_seen():
    check_negative_sampling("uniform", 0)
    check_negative_sampling("uniform", 0, negatives=object())
    check_negative_sampling("seen", 1)


@pytest.mark.parametrize("args, fix", [
    (("frequency", 1), "'uniform' or 'seen'"),
    (("seen", 0), "negative_sample_rate >= 1"),
    (("seen", 2, object()), "without negatives="),
])
def test_negative_sampling_refusals_name_the_fix(args, fix):
    with pytest.raises(ValueError, match=fix):
        check_negative_sampling(*args)


@pytest.mark.parametrize("backend", ["local", "native"])
def test_host_tiers_take_seen_and_refuse_uniform(backend):
    require_pointwise(backend, {"negativeSampling": "seen"})
    require_pointwise(backend, {})
    with pytest.raises(ValueError, match="backend='device'"):
        require_pointwise(backend, {"negativeSampling": "uniform"})
    require_pointwise("device", {"negativeSampling": "uniform"})
    require_pointwise("device", {"negativeSampling": "seen"})


@pytest.mark.parametrize("backend", ["local", "native", "device"])
def test_unknown_negative_sampling_is_refused(backend):
    with pytest.raises(ValueError, match="'uniform' or 'seen'"):
        require_pointwise(backend, {"negativeSampling": "popular"})


@pytest.mark.parametrize("entry", ["online", "offline"])
def test_host_entry_points_refuse_uniform(entry):
    from fps_b200.models.mf.offline import psOfflineMF
    from fps_b200.models.mf.online import psOnlineMF

    recs = [Rating(0, 1, 1.0), Rating(1, 0, 0.5)]
    fn = psOnlineMF if entry == "online" else psOfflineMF
    with pytest.raises(ValueError, match="negativeSampling='uniform' needs backend='device'"):
        fn(recs, numFactors=4, backend="local", negativeSampleRate=1, negativeSampling="uniform")


def test_noise_counts_are_returned_as_float64():
    c = check_noise([3, 0, 1], 3, 0.75)
    assert c.dtype == np.float64 and c.tolist() == [3.0, 0.0, 1.0]
    check_noise(np.ones(4), 4, 0.0)


@pytest.mark.parametrize("counts, power, fix", [
    ([1, 2], 0.75, "one count per word"),
    ([1, -1, 2], 0.75, ">= 0"),
    ([1, math.nan, 2], 0.75, "finite"),
    ([1, math.inf, 2], 0.75, "finite"),
    ([0, 0, 0], 0.75, "positive count"),
    ([1, 2, 3], -0.5, "noise_power"),
    ([1, 2, 3], math.nan, "noise_power"),
])
def test_noise_refusals_name_the_fix(counts, power, fix):
    with pytest.raises(ValueError, match=fix):
        check_noise(counts, 3, power)
