"""The replica-mode replay (``tests/replica_ref.py``) against the host protocol and the textbook exchange, and the
argument refusals of the replica bindings.  No GPU: the refusals come before the kernel library is loaded."""
import itertools
import random

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from fps_b200.protocol.combination import CombinationLogic, CountLogic, TimerLogic, all_of, any_of

from . import replica_ref as ref


# ---- slices --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("slices", range(1, 10))
def test_slices_cover_the_range_once(slices):
    for rps in sorted({1, 7, max(1, slices - 1), 4 * slices}):
        for slot_lo, slot_hi in [(0, rps), (rps // 3, rps)]:
            for offset, o in itertools.product(range(4), (0, 3, 15)):
                seen = np.zeros(rps, dtype=int)
                for flushes in range(1, slices + 1):
                    lo, hi = ref.slice_range(o, flushes, slot_lo, slot_hi, slices, offset, slices > 1)
                    assert slot_lo <= lo <= hi <= slot_hi
                    seen[lo:hi] += 1
                assert (seen[slot_lo:slot_hi] == 1).all() and seen[:slot_lo].sum() == 0


def test_slices_past_the_range_are_empty():
    # 3 slots in 5 slices of one slot: two successive flushes move nothing
    got = [ref.slice_range(0, f, 0, 3, 5, 0, True) for f in range(5)]
    assert got == [(0, 1), (1, 2), (2, 3), (3, 3), (3, 3)]


# ---- policy against the host CountLogic / TimerLogic -----------------------------------------------------------

def _host_fires(events, count_max, timer, require_all):
    """Fire pattern of the host CombinationLogic: 'm' is one message, 't' one timer tick."""
    trig = ([CountLogic(count_max)] if count_max else []) + ([TimerLogic(1e9)] if timer else [])
    logic = CombinationLogic(all_of if require_all else any_of, trig)
    out, fires = [], []
    try:
        for e in events:
            n = len(out)
            if e == "m":
                logic.logic(lambda data: data.append(1), out.append)
            else:
                for t in trig:
                    if isinstance(t, TimerLogic):
                        with logic._lock:            # the body of the timer thread, one tick
                            if t.sendCondition():
                                t.send(logic.checkAndSend, out.append)
                                t.containsData = False
            fires.append(len(out) > n)
    finally:
        logic.close()
    return fires


def _device_fires(events, count_max, timer, require_all):
    """The device deadline stays passed until the next flush; the host timer notices it at a tick with data
    buffered and keeps its flag until the next flush, so a deadline counts from such a tick on."""
    st, fires, passed = np.zeros(ref.STATE_WORDS, dtype=np.int64), [], False
    for e in events:
        tick = e == "t"
        passed = passed or (tick and int(st[ref.PENDING]) != 0)
        st = ref.policy(st, 1, count_max=count_max, interval_passed=[passed] if timer else None,
                        require_all=require_all, add_uniform=0 if tick else 1)
        fires.append(bool(ref.mask_word(st) & 1))
        passed = passed and not fires[-1]
    return fires, st


@pytest.mark.parametrize("count_max, timer", [(1, False), (3, False), (0, True), (2, True), (4, True)])
@pytest.mark.parametrize("require_all", [False, True])
def test_policy_matches_host_count_timer_logic(count_max, timer, require_all):
    rnd = random.Random(count_max * 10 + timer + 2 * require_all)
    events = [rnd.choice("mmmt" if timer else "m") for _ in range(60)]
    fires, st = _device_fires(events, count_max, timer, require_all)
    assert fires == _host_fires(events, count_max, timer, require_all)
    assert int(st[ref.COUNT]) == sum(fires) and ref.evals(st) == len(events)


def test_policy_counters():
    st = np.zeros(ref.STATE_WORDS, dtype=np.int64)
    st = ref.policy(st, 3, count_max=5, add_uniform=4)
    assert ref.mask_word(st) == 0 and list(st[:3]) == [4, 4, 4]
    st = ref.policy(st, 3, count_max=5, add_uniform=1)
    assert ref.mask_word(st) == 0b111 and list(st[:3]) == [0, 0, 0] and list(st[ref.COUNT:ref.COUNT + 3]) == [1] * 3
    st = ref.policy(st, 2, force=True)
    assert ref.mask_word(st) == 0b11 and list(st[ref.COUNT:ref.COUNT + 3]) == [2, 2, 1] and ref.evals(st) == 3
    # AND with nothing enabled never fires; the timer needs a message pending
    assert ref.mask_word(ref.policy(st, 3, require_all=True, add_uniform=9)) == 0
    assert ref.mask_word(ref.policy(st, 3, interval_passed=[True] * 3)) == 0


# ---- exchange ------------------------------------------------------------------------------------------------

def _textbook(masters, cache, base, mask, num_shards, ranges):
    masters = [m.copy() for m in masters]; cache = cache.copy(); base = base.copy()
    rps = cache.shape[0] // num_shards
    for o in range(num_shards):
        lo, hi = ranges[o]
        if not (mask >> o) & 1:
            continue
        for s in range(lo, hi):
            v, c, b = masters[o][s].copy(), cache[o * rps + s].copy(), base[o * rps + s].copy()
            d, f = c - b, v - b
            masters[o][s] = v + d
            cache[o * rps + s] = c + f
            base[o * rps + s] = v + d
    return masters, cache, base


def _tables(num_shards, rps, stride, seed, subnormal=False):
    g = np.random.default_rng(seed)
    scale = np.float32(1e-39) if subnormal else np.float32(1)
    masters = [(g.standard_normal((rps, stride)) * scale).astype(np.float32) for _ in range(num_shards)]
    base = np.concatenate(masters) + (g.standard_normal((num_shards * rps, stride)) * scale).astype(np.float32)
    cache = base + (g.standard_normal(base.shape) * scale).astype(np.float32)
    return masters, cache.astype(np.float32), base.astype(np.float32)


def _same(a, b):
    return all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(a, b))


@pytest.mark.parametrize("num_shards, stride", [(1, 4), (3, 8), (5, 12)])
def test_exchange_without_ftz_is_the_textbook_update(num_shards, stride):
    rps = 9
    masters, cache, base = _tables(num_shards, rps, stride, num_shards)
    ranges = [(1, rps - 1)] * num_shards
    mask = 0b10111
    got = ref.exchange(masters, cache, base, mask, 0, num_shards, ranges, flush=False)
    want = _textbook(masters, cache, base, mask, num_shards, ranges)
    assert _same(got[0], want[0]) and _same([got[1], got[2]], [want[1], want[2]])
    # normal values: FTZ changes nothing
    got_ftz = ref.exchange(masters, cache, base, mask, 0, num_shards, ranges)
    assert _same(got_ftz[0], want[0]) and _same([got_ftz[1], got_ftz[2]], [want[1], want[2]])


def _sub(x):
    return (x != 0) & (np.abs(x) < ref.TINY)


def test_exchange_ftz_differs_only_on_subnormals():
    num_shards, rps, stride = 2, 16, 8
    masters, cache, base = _tables(num_shards, rps, stride, 7)
    g = np.random.default_rng(8)
    for t in masters + [cache, base]:
        pick = g.random(t.shape) < 0.3
        t[pick] = (g.standard_normal(pick.sum()) * 1e-39).astype(np.float32)
    ranges = [(0, rps)] * num_shards
    plain = ref.exchange(masters, cache, base, 0b11, 0, num_shards, ranges, flush=False)
    ftz = ref.exchange(masters, cache, base, 0b11, 0, num_shards, ranges)
    v, c, b = np.concatenate(masters), cache, base
    d, f = c - b, v - b
    for p, q, x, y in [(np.concatenate(plain[0]), np.concatenate(ftz[0]), v, d), (plain[1], ftz[1], c, f)]:
        differs = p.view(np.int32) != q.view(np.int32)
        assert differs.any()
        assert not (differs & ~(_sub(x) | _sub(y) | _sub(p))).any()
        assert not _sub(q[differs]).any()
    assert _same([plain[2]], [ftz[2]])          # b = v + d is not flushed


def test_exchange_gates_per_float4_group():
    tiny = np.float32(1e-39)
    masters = [np.full((1, 8), tiny, np.float32)]
    base, cache = np.full((1, 8), tiny, np.float32), np.full((1, 8), tiny, np.float32)
    cache[0, 1] = 2.0                                      # only lane 1 of group 0 changed
    m, c, b = ref.exchange(masters, cache, base, 1, 0, 1, [(0, 1)])
    assert list(m[0][0, :4]) == [0, 2, 0, 0]              # the group pushed: its subnormal lanes were flushed
    assert (m[0][0, 4:] == tiny).all()                     # group 1 did not push: untouched
    assert list(b[0, :4]) == [tiny, 2, tiny, tiny]         # b = v + d keeps the subnormal
    assert _same([c], [cache])
    c2, b2 = cache.copy(), base.copy()
    c2[0, 1], b2[0, 1] = -0.0, 0.0                         # d = -0 gates nothing
    assert _same(ref.exchange(masters, c2, b2, 1, 0, 1, [(0, 1)])[0], masters)
    c3 = cache.copy(); c3[0, 5] = np.nan
    m3, _, b3 = ref.exchange(masters, c3, base, 1, 0, 1, [(0, 1)])
    assert np.isnan(m3[0][0, 5]) and np.isnan(b3[0, 5]) and list(m3[0][0, [4, 6, 7]]) == [0, 0, 0]


def test_exchange_mask_clamp_and_skip():
    masters, cache, base = _tables(3, 4, 4, 3)
    ranges = [(0, 4)] * 3
    got = ref.exchange(masters, cache, base, 0xFFFF_FFF8 | 0b101, 0b100, 3, ranges)
    want = ref.exchange(masters, cache, base, 0b001, 0, 3, ranges)
    assert _same(got[0], want[0]) and _same(got[1:], want[1:])


def test_sequential_workers_conserve_dyadic_deltas():
    W, rps, stride = 3, 11, 8
    g = np.random.default_rng(4)
    masters = [(g.integers(-512, 512, (rps, stride)) / 256).astype(np.float32) for _ in range(W)]
    init = np.concatenate(masters).copy()
    for own in (False, True):
        wk = ref.Workers(W, rps, stride, own, masters)
        total = np.zeros((W * rps, stride))
        for step in range(6):
            for w in range(W):
                ids = g.choice(W * rps, 10, replace=False)
                delta = (g.integers(-256, 256, (10, stride)) / 256).astype(np.float32)
                wk.push(w, ids, delta)
                for i, d in zip(ids, delta):
                    total[(i % W) * rps + i // W] += d
                wk.policy(w, count_max=1, add_uniform=1)
                wk.exchange(w, slices=3, slice_offset=w)
        for _ in range(2):
            for w in range(W):
                wk.policy(w, force=True)
                wk.exchange(w)
        assert np.array_equal(np.concatenate(wk.masters), (init + total).astype(np.float32))
        for w in range(W):
            keep = np.ones(W * rps, bool)
            if own:
                keep[w * rps:(w + 1) * rps] = False
            assert np.array_equal(wk.cache[w][keep], np.concatenate(wk.masters)[keep])
            assert np.array_equal(wk.base[w][keep], wk.cache[w][keep])


def test_deal_replay():
    items = np.array([0, 1, 2, 3, 7, -7, 100, -100])
    bucket, feed = ref.deal(items, 3, 5, 1, 4)
    owner = np.abs(items) % 3
    assert list(feed) == list(np.bincount(owner, minlength=3))
    assert list(bucket) == list(np.minimum((owner * 5 + np.abs(items) // 3) >> 1, 3))
    assert list(ref.deal(items, 1, 0, 2, 64)[0]) == list(np.abs(items) >> 2)


# ---- refusals, before the library loads ----------------------------------------------------------------------

@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the kernel library was loaded before the arguments were refused")
    monkeypatch.setattr(native, "lib", refuse)


def _master(num_shards=2, stride=8, rps=4):
    t = native.ShardTableC()
    t.num_shards = num_shards; t.stride = stride; t.dim = stride; t.rows_per_shard = rps
    return t


def _cpu(num_shards=2, stride=8, rps=4):
    return torch.zeros(max(1, num_shards) * rps, stride), torch.zeros(max(1, num_shards) * rps, stride)


@pytest.mark.parametrize("num_shards", [0, -1, 17, 32])
def test_exchange_refuses_shard_counts(no_library, num_shards):
    with pytest.raises(ValueError, match="num_shards"):
        native.replica_exchange(_master(num_shards), *_cpu(num_shards), mask=1)


@pytest.mark.parametrize("stride", [0, 2, 6, 66])
def test_exchange_refuses_strides(no_library, stride):
    with pytest.raises(ValueError, match="stride"):
        native.replica_exchange(_master(stride=stride), *_cpu(stride=max(stride, 1)), mask=1)


@pytest.mark.parametrize("lo, hi", [(-1, 4), (0, 5), (-3, -1), (2, 9)])
def test_exchange_refuses_slot_ranges(no_library, lo, hi):
    with pytest.raises(ValueError, match="slot range"):
        native.replica_exchange(_master(), *_cpu(), mask=1, slot_lo=lo, slot_hi=hi)


@pytest.mark.parametrize("num_shards", [0, 17])
def test_bucket_by_item_refuses_shard_counts(no_library, num_shards):
    u = torch.zeros(4, dtype=torch.int32)
    with pytest.raises(ValueError, match="num_shards"):
        native.bucket_by_item(u, u, torch.ones(4), 0, 1, torch.zeros(128, dtype=torch.int32),
                              num_shards=num_shards, rows_per_shard=1)


@pytest.mark.parametrize("num_dest", [0, 17])
def test_flush_policy_refuses_destination_counts(no_library, num_dest):
    with pytest.raises(ValueError, match="num_dest"):
        native.flush_policy(torch.zeros(native.FLUSH_STATE_WORDS, dtype=torch.int64), num_dest)


def test_flush_policy_refuses_a_short_state(no_library):
    with pytest.raises(ValueError, match="state must hold"):
        native.flush_policy(torch.zeros(native.FLUSH_STATE_WORDS - 1, dtype=torch.int64), 1)


def test_replay_constants_match_the_bindings():
    assert (ref.MAX_SHARDS, ref.STATE_WORDS) == (native.FPS_MAX_SHARDS, native.FLUSH_STATE_WORDS)
    assert (ref.PENDING, ref.LAST_NS, ref.COUNT, ref.MASK) == (native.FLUSH_PENDING, native.FLUSH_LAST_NS,
                                                               native.FLUSH_COUNT, native.FLUSH_MASK)
