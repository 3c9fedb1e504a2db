"""Replica (item-cache) kernels against the exact replay of ``tests/replica_ref.py`` on one GPU.

Master shards are separate device tensors behind a hand-built ``ShardTableC``; every master, replica and base
table carries sentinel guard rows before and after its rows.  Within one launch the exchange is deterministic
per element, so masters, replica and base must equal the replay bit for bit, guards included (NaNs compare by
class, not payload), and the flush state words (all but the ``last_ns`` clocks) exactly."""
import ctypes as C

import numpy as np
import pytest
import torch

from fps_b200.ops import native
from tests import replica_ref as ref

pytestmark = pytest.mark.gpu

GUARD = 3
SENTINEL = np.float32(-12345.5)
CHUNK_VEC = 512                 # float4 vectors per pipeline stage (EX_CHUNK_VEC)


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def chunk_rows(stride):
    return max(1, CHUNK_VEC // (stride // 4))


def _guarded(rows, stride, dev, fill):
    buf = torch.full((rows + 2 * GUARD, stride), float(SENTINEL), dtype=torch.float32, device=dev)
    buf[GUARD:GUARD + rows] = torch.from_numpy(np.ascontiguousarray(fill)).to(dev)
    return buf


def _bits(a):
    a = np.array(a, dtype=np.float32, copy=True)
    a[np.isnan(a)] = np.float32("nan")
    return a.view(np.int32)


def _assert_same(got, want, what):
    g, w = _bits(got), _bits(want)
    bad = np.argwhere(g != w)
    assert bad.size == 0, f"{what}: {len(bad)} elements differ, first at {bad[0].tolist()}: " \
                          f"{got[tuple(bad[0])]!r} != {want[tuple(bad[0])]!r}"


def _pad(a):
    s = np.full((a.shape[0] + 2 * GUARD, a.shape[1]), SENTINEL, dtype=np.float32)
    s[GUARD:GUARD + a.shape[0]] = a
    return s


def _state_words(st):
    st = np.asarray(st, dtype=np.int64).copy()
    st[ref.LAST_NS:ref.LAST_NS + ref.MAX_SHARDS] = 0
    return st


class Setup:
    """W master shards, one replica / base pair and a flush state on the device, and their host copies."""

    def __init__(self, dev, num_shards, rps, stride, masters, cache, base, state=None):
        self.num_shards, self.rps, self.stride = num_shards, rps, stride
        self.m_dev = [_guarded(rps, stride, dev, m) for m in masters]
        self.c_dev = _guarded(num_shards * rps, stride, dev, cache)
        self.b_dev = _guarded(num_shards * rps, stride, dev, base)
        self.state = torch.zeros(ref.STATE_WORDS, dtype=torch.int64, device=dev) if state is None else \
            torch.from_numpy(np.asarray(state, dtype=np.int64)).to(dev)
        t = native.ShardTableC()
        for o in range(num_shards):
            t.base[o] = self.m_dev[o].data_ptr() + GUARD * stride * 4
        t.rows_per_shard = rps; t.div = rps; t.num_shards = num_shards; t.dim = stride; t.stride = stride
        t.mode = native.PART_HASH; t.shard_shift = native.log2_or_neg(num_shards)
        self.tc = t
        self.masters = [np.array(m, np.float32) for m in masters]
        self.cache, self.base = np.array(cache, np.float32), np.array(base, np.float32)
        self.st = np.asarray(self.state.cpu().numpy(), dtype=np.int64)

    def cache_view(self):
        return self.c_dev[GUARD:GUARD + self.num_shards * self.rps]

    def base_view(self):
        return self.b_dev[GUARD:GUARD + self.num_shards * self.rps]

    def policy(self, **kw):
        """flush_policy on the device and in the replay (the timer is off or never due)."""
        due = kw.pop("interval_passed", None)
        native.flush_policy(self.state, self.num_shards, **kw)
        self.st = ref.policy(self.st, self.num_shards, count_max=kw.get("count_max", 0),
                             interval_passed=due, require_all=kw.get("require_all", False),
                             force=kw.get("force", False), add_uniform=kw.get("add_uniform", 0))

    def exchange(self, use_state=False, mask=0, skip_mask=0, slot_lo=0, slot_hi=None, slices=1, slice_offset=0,
                 **kw):
        hi = self.rps if slot_hi is None else slot_hi
        native.replica_exchange(self.tc, self.cache_view(), self.base_view(), state=self.state if use_state else None,
                                mask=mask, skip_mask=skip_mask, slot_lo=slot_lo, slot_hi=hi, slices=slices,
                                slice_offset=slice_offset, **kw)
        st = self.st if use_state else None
        ranges = ref.ranges_for(self.num_shards, slot_lo, hi, st, slices, slice_offset)
        m = ref.mask_word(self.st) if use_state else mask
        self.masters, self.cache, self.base = ref.exchange(self.masters, self.cache, self.base, m, skip_mask,
                                                           self.num_shards, ranges)
        return ranges

    def check(self):
        torch.cuda.synchronize()
        for o in range(self.num_shards):
            _assert_same(self.m_dev[o].cpu().numpy(), _pad(self.masters[o]), f"master {o}")
        _assert_same(self.c_dev.cpu().numpy(), _pad(self.cache), "replica")
        _assert_same(self.b_dev.cpu().numpy(), _pad(self.base), "base")
        assert np.array_equal(_state_words(self.state.cpu().numpy()), _state_words(self.st))


def tables(num_shards, rps, stride, seed, p=0.5):
    """Masters, replica and base where about a fraction ``p`` of the float4 groups have a local delta and,
    independently, a foreign one (single lanes as well as whole groups)."""
    g = np.random.default_rng(seed)
    n = num_shards * rps
    base = g.standard_normal((n, stride)).astype(np.float32)
    groups = (n, stride // 4, 1)

    def delta():
        lanes = g.random((n, stride // 4, 4)) < 0.5
        on = (g.random(groups) < p) & lanes
        return (g.standard_normal((n, stride // 4, 4)) * on).astype(np.float32).reshape(n, stride)

    cache = base + delta()
    master = base + delta()
    return [master[o * rps:(o + 1) * rps] for o in range(num_shards)], cache, base


def run(dev, num_shards, rps, stride, seed=0, state=None, **kw):
    s = Setup(dev, num_shards, rps, stride, *tables(num_shards, rps, stride, seed), state=state)
    s.exchange(**kw)
    s.check()
    return s


# ---- geometry ------------------------------------------------------------------------------------------------

def _rps_list(stride):
    if stride // 4 > CHUNK_VEC:
        return [1, 2, 7]
    cr = chunk_rows(stride)
    return sorted({1, max(1, cr - 1), cr + 1, 3 * cr + 5})


@pytest.mark.parametrize("sequential", [False, True], ids=["interleaved", "sequential"])
@pytest.mark.parametrize("stride", [4, 64, 68, 300, 2048, 2052, 4100])
@pytest.mark.parametrize("num_shards", [1, 2, 3, 5, 16])
def test_exchange_geometry(dev, num_shards, stride, sequential):
    for k, rps in enumerate(_rps_list(stride)):
        run(dev, num_shards, rps, stride, seed=k, mask=(1 << num_shards) - 1, sequential=sequential, n_ctas=7)


# ---- pipeline ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_stages", [0, 1, 2, 3, 4, 8, 9])
@pytest.mark.parametrize("shape", [(5, 68, 95), (16, 64, 32 * 40 + 5)], ids=["20-chunks", "656-chunks"])
def test_exchange_pipeline_depth_and_grid(dev, shape, n_stages):
    """Every stage depth (0 and 9 clamp to 4 and 8) and CTA count, down to one CTA through one stage (the phase
    wraps on every chunk), gives the replayed tables."""
    num_shards, stride, rps = shape
    chunks = num_shards * -(-rps // chunk_rows(stride))
    sms = native.sm_count(0)
    for n_ctas in [1, 2, 7, 64, 2 * sms, chunks + 5]:
        for sequential in (False, True):
            run(dev, num_shards, rps, stride, seed=n_ctas, mask=(1 << num_shards) - 1, n_ctas=n_ctas,
                n_stages=n_stages, sequential=sequential)


# ---- selection -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("stride", [68, 2052])
@pytest.mark.parametrize("mask, skip", [(0xFFFF, 0), (1 | 1 << 5 | 1 << 15, 0), (0, 0), (0xFFFF, 0xFFFF),
                                        (0xFFFF, 1 << 5 | 1 << 6), (1 << 5, 1 << 5)],
                         ids=["full", "sparse", "empty", "all-skipped", "skip-overlap", "skip-only-bit"])
def test_exchange_masks(dev, stride, mask, skip):
    run(dev, 16, 7, stride, seed=mask, mask=mask, skip_mask=skip, n_ctas=5)


@pytest.mark.parametrize("stride", [68, 2052])
@pytest.mark.parametrize("num_shards", [1, 3, 5])
def test_exchange_ignores_mask_bits_past_the_shard_count(dev, stride, num_shards):
    run(dev, num_shards, 9, stride, seed=1, mask=0xFFFFFFFF ^ 0b10, skip_mask=0b100, n_ctas=3)


@pytest.mark.parametrize("stride", [68, 2052])
def test_exchange_state_mask_against_override(dev, stride):
    st = np.zeros(ref.STATE_WORDS, dtype=np.int64)
    st[ref.MASK] = 0b0110 | (7 << 32)
    st[ref.COUNT:ref.COUNT + 4] = [3, 1, 4, 1]
    run(dev, 4, 31, stride, seed=2, state=st, use_state=True, mask=0b1001)          # the state wins
    run(dev, 4, 31, stride, seed=3, state=st, use_state=True, slices=3, slice_offset=1)
    run(dev, 4, 31, stride, seed=4, state=st, mask=0b1011, slices=3, slice_offset=1)  # override: not sliced


@pytest.mark.parametrize("stride", [68, 2052])
@pytest.mark.parametrize("lo, hi", [(0, 1), (5, 6), (3, 40), (0, 61), (60, 61), (7, 7), (9, 2)])
def test_exchange_slot_subranges(dev, stride, lo, hi):
    run(dev, 3, 61, stride, seed=lo * 100 + hi, mask=0b111, slot_lo=lo, slot_hi=hi, n_ctas=4)


# ---- slices --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("slice_offset", range(4))
@pytest.mark.parametrize("slices", range(1, 10))
@pytest.mark.parametrize("stride", [64, 2052], ids=["tma", "wide"])
def test_exchange_slices_rotate_through_the_range(dev, stride, slices, slice_offset):
    """Each forced flush moves exactly its replayed slice, rows outside it stay bitwise unchanged in all three
    arrays, and ``slices`` successive flushes cover every slot once."""
    num_shards = 3
    rps = 3 * chunk_rows(stride) + 5 if stride <= 4 * CHUNK_VEC else 11
    s = Setup(dev, num_shards, rps, stride, *tables(num_shards, rps, stride, slices, p=1.0))
    covered = np.zeros((num_shards, rps), dtype=int)
    for _ in range(slices):
        s.cache_view()[:] += 0.5                          # every row has a local delta again
        s.cache += np.float32(0.5)
        before = [m.copy() for m in s.masters], s.cache.copy(), s.base.copy()
        s.policy(force=True)
        ranges = s.exchange(use_state=True, slices=slices, slice_offset=slice_offset, n_ctas=3)
        s.check()
        for o, (lo, hi) in enumerate(ranges):
            rows = slice(o * rps, (o + 1) * rps)
            moved = ~(s.masters[o] == before[0][o]).all(axis=1)
            assert moved[lo:hi].all() and not moved[:lo].any() and not moved[hi:].any()
            for now, old in [(s.cache[rows], before[1][rows]), (s.base[rows], before[2][rows])]:
                keep = np.ones(rps, bool); keep[lo:hi] = False
                _assert_same(now[keep], old[keep], f"rows outside the slice of {o}")
            covered[o, lo:hi] += 1
    assert (covered == 1).all()


# ---- values --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("stride", [8, 2052])
def test_exchange_values(dev, stride):
    """Single-lane deltas, local and foreign deltas together, subnormal master / replica / base lanes (flushed
    by the reductions of a gated group, kept by ``b = v + d``), inf and NaN in the replica, and -0."""
    rps = 12
    masters, cache, base = tables(2, rps, stride, 9, p=0.0)
    m = np.concatenate(masters)
    tiny = np.float32(3e-39)
    m[0, :] = base[0, :]; cache[0, :] = base[0, :]; cache[0, 2] += 1   # one lane of one group, local
    m[1, 1] = base[1, 1] + 2                                            # one lane, foreign
    cache[2, :4] += 1; m[2, :4] -= 3                                    # both
    m[3, :4] = tiny; base[3, :4] = tiny; cache[3, :4] = tiny; cache[3, 0] = 1   # subnormal master lanes pushed into
    m[3, 4:8] = tiny; base[3, 4:8] = tiny; cache[3, 4:8] = tiny          # ... and left alone
    cache[4, :4] = -tiny; base[4, :4] = 0; m[4, :4] = 0                  # subnormal replica delta
    base[5, :4] = tiny; cache[5, :4] = 1; m[5, :4] = 0                   # subnormal base
    cache[6, 1] = np.inf; cache[7, 2] = np.nan; cache[8, 3] = -np.inf
    cache[9, :4] = -0.0; base[9, :4] = 0.0; m[9, :4] = 0.0               # -0: no delta
    base[10, :4] = -0.0; m[10, :4] = 0.0; cache[10, :4] = 0.0            # f = 0 - (-0) = +0: no delta
    masters = [m[:rps], m[rps:]]
    s = Setup(dev, 2, rps, stride, masters, cache, base)
    s.exchange(mask=0b11)
    s.check()
    assert s.masters[0][3, 1] == 0 and s.base[3, 1] == tiny and s.masters[0][3, 5] == tiny


# ---- policy --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("num_dest", range(1, 17))
def test_policy_counts_force_and_feed(dev, num_dest):
    count_max = 5
    g = np.random.default_rng(num_dest)
    st0 = np.zeros(ref.STATE_WORDS, dtype=np.int64)
    st0[:num_dest] = g.integers(0, 2 * count_max, num_dest)     # destinations start at different counts
    state = torch.from_numpy(st0).to(dev)
    st = st0
    for add, force, feed in [(count_max - 1, False, 0), (0, False, 0), (1, False, 0), (count_max + 1, False, 3),
                             (count_max, False, 0), (0, True, 0), (2, False, 0), (0, False, count_max)]:
        if feed:                                              # the bucket histogram feeds between evaluations
            state[:num_dest] += feed
            st = st.copy(); st[:num_dest] += feed
        native.flush_policy(state, num_dest, count_max=count_max, force=force, add_uniform=add)
        st = ref.policy(st, num_dest, count_max=count_max, force=force, add_uniform=add)
        torch.cuda.synchronize()
        assert np.array_equal(_state_words(state.cpu().numpy()), _state_words(st))


@pytest.mark.parametrize("require_all", [False, True], ids=["or", "and"])
@pytest.mark.parametrize("count_max", [0, 3])
@pytest.mark.parametrize("interval", [0, 1, 1 << 62], ids=["no-timer", "timer-due", "timer-never"])
def test_policy_count_and_timer(dev, require_all, count_max, interval):
    """The timer without sleeping: ``interval_ns = 1`` is due from the second evaluation on (the first one
    starts the clock), ``2^62`` never; it fires only with messages pending."""
    num_dest = 4
    state = torch.zeros(ref.STATE_WORDS, dtype=torch.int64, device=dev)
    st = np.zeros(ref.STATE_WORDS, dtype=np.int64)
    for k, add in enumerate([1, 0, 2, 1, 0, 0, 3, 1]):
        due = None if interval == 0 else [interval == 1 and k > 0] * num_dest
        native.flush_policy(state, num_dest, count_max=count_max, interval_ns=interval, require_all=require_all,
                            add_uniform=add)
        st = ref.policy(st, num_dest, count_max=count_max, interval_passed=due, require_all=require_all,
                        add_uniform=add)
        torch.cuda.synchronize()
        assert np.array_equal(_state_words(state.cpu().numpy()), _state_words(st)), f"evaluation {k}"


@pytest.mark.parametrize("num_dest", [0, 17])
def test_policy_c_entry_refuses_destination_counts(dev, num_dest):
    p = native.FlushPolicyC(); p.num_dest = num_dest; p.force = 1
    state = torch.zeros(ref.STATE_WORDS, dtype=torch.int64, device=dev)
    assert native.lib().fps_flush_policy(C.byref(p), C.c_void_p(state.data_ptr()), native._stream()) == -1401
    torch.cuda.synchronize()
    assert not state.any()


def test_exchange_c_entry_refuses_bad_arguments(dev):
    """The C entry refuses what the binding refuses, before any launch."""
    s = Setup(dev, 2, 4, 8, *tables(2, 4, 8, 0))

    def code(**kw):
        a = native.ExchArgsC()
        a.master = native.ShardTableC.from_buffer_copy(s.tc)
        a.cache = s.cache_view().data_ptr(); a.base = s.base_view().data_ptr(); a.rps = 4
        a.slot_lo, a.slot_hi, a.mask_override = 0, 4, 0b11
        for k, v in kw.items():
            if k in ("num_shards", "stride"):
                setattr(a.master, k, v)
            else:
                setattr(a, k, v)
        return native.lib().fps_replica_exchange(C.byref(a), 4, native._stream())

    assert [code(num_shards=0), code(num_shards=17)] == [-1403, -1403]
    assert [code(stride=6), code(stride=0)] == [-1404, -1404]
    assert [code(slot_lo=-1), code(slot_hi=5)] == [-1405, -1405]
    s.check()                                                       # nothing moved


def test_bucket_c_entry_refuses_shard_counts(dev):
    a = native.BucketArgsC(); a.n = 4; a.n_buckets = 1
    for n in (0, 17):
        a.num_shards = n
        assert native.lib().fps_bucket_by_item(C.byref(a), 1, native._stream()) == -1302


# ---- bucket deal ---------------------------------------------------------------------------------------------

def _deal_case(dev, form, num_shards, n, n_buckets, g, scratch, pending):
    n_items = 40_000
    rps = -(-n_items // num_shards)
    rows = rps * num_shards
    shift = max(0, int(np.ceil(np.log2(max(1, rows / n_buckets)))))
    items = g.integers(0, n_items + n_items // 8, n)          # past the table: clamps to the last bucket
    users = g.integers(0, 1 << 20, n)
    ratings = g.integers(0, 64, n).astype(np.float32)
    if form != "packed64":
        items = np.where(g.random(n) < 0.05, -items, items)   # void (negative) ids bucket by |item|
    if form == "packed64":
        recs = (users << 38) | (items << 16) | np.float16(ratings).view(np.int16).astype(np.int64) & 0xFFFF
        out, _, _ = native.bucket_by_item(torch.from_numpy(recs).to(dev), None, None, shift, n_buckets, scratch,
                                          num_shards=num_shards, rows_per_shard=rps, pending=pending)
        got = out.cpu().numpy()
        got_items, key_in, key_out = (got >> 16) & 0x3FFFFF, recs, got
    else:
        dt = torch.int32 if form == "int32" else torch.int64
        ou, oi, orat = native.bucket_by_item(torch.from_numpy(users).to(dt).to(dev),
                                             torch.from_numpy(items).to(dt).to(dev),
                                             torch.from_numpy(ratings).to(dev), shift, n_buckets, scratch,
                                             num_shards=num_shards, rows_per_shard=rps, pending=pending)
        got_items = oi.cpu().numpy().astype(np.int64)
        key_in = (users << 40) ^ ((items & 0xFFFFFF) << 16) ^ ratings.astype(np.int64)
        key_out = (ou.cpu().numpy().astype(np.int64) << 40) ^ ((got_items & 0xFFFFFF) << 16) ^ \
            orat.cpu().numpy().astype(np.int64)
    bucket, feed = ref.deal(items, num_shards, rps, shift, n_buckets)
    out_bucket, _ = ref.deal(got_items, num_shards, rps, shift, n_buckets)
    assert np.array_equal(np.sort(key_in), np.sort(key_out)), "not a permutation"
    assert (np.diff(out_bucket) >= 0).all(), "bucket keys decrease"
    counts = np.bincount(bucket, minlength=n_buckets)
    ends = np.cumsum(counts)
    for k, want in enumerate(ref.bucket_groups(key_in, bucket, n_buckets)):
        assert np.array_equal(np.sort(key_out[ends[k] - counts[k]:ends[k]]), want), f"bucket {k}"
    return feed


@pytest.mark.parametrize("form", ["int32", "int64", "packed64"])
@pytest.mark.parametrize("num_shards", [1, 2, 3, 5, 8, 16])
def test_bucket_deal(dev, num_shards, form):
    g = np.random.default_rng(num_shards * 7 + len(form))
    grid = 4 * native.sm_count(0)                # every CTA resident: up to 4 per SM for this kernel
    sizes = [1, 255, 256, 257, grid * 256 - 1, grid * 256 + 1, grid * 1000 - 1, grid * 1000 + 1]
    if num_shards in (5, 16):
        sizes.append(5_000_000)
    scratch = torch.randint(-1000, 1000, (2 * native.BUCKET_MAX,), dtype=torch.int32, device=dev)   # dirty
    for k, n in enumerate(sizes):
        n_buckets = [1, 2, 63, 64][k % 4]
        start = g.integers(0, 1000, num_shards)
        pending = torch.from_numpy(start).to(dev)
        feed = _deal_case(dev, form, num_shards, n, n_buckets, g, scratch, pending)
        feed = feed + _deal_case(dev, form, num_shards, max(1, n // 3), n_buckets, g, scratch, pending)
        assert np.array_equal(pending.cpu().numpy(), start + feed), f"feed, n={n}"


# ---- W workers on one device ---------------------------------------------------------------------------------

def _workers(dev, W, rps, stride, own, seed, dyadic=False):
    g = np.random.default_rng(seed)
    if dyadic:
        masters = [(g.integers(-512, 512, (rps, stride)) / 256).astype(np.float32) for _ in range(W)]
    else:
        masters = [g.standard_normal((rps, stride)).astype(np.float32) for _ in range(W)]
    rep = ref.Workers(W, rps, stride, own, masters)
    m_dev = [_guarded(rps, stride, dev, m) for m in masters]
    t = native.ShardTableC()
    for o in range(W):
        t.base[o] = m_dev[o].data_ptr() + GUARD * stride * 4
    t.rows_per_shard = rps; t.div = rps; t.num_shards = W; t.dim = stride; t.stride = stride
    t.mode = native.PART_HASH; t.shard_shift = native.log2_or_neg(W)
    full = np.concatenate(masters)
    caches = [_guarded(W * rps, stride, dev, full) for _ in range(W)]
    bases = [_guarded(W * rps, stride, dev, full) for _ in range(W)]
    states = [torch.zeros(ref.STATE_WORDS, dtype=torch.int64, device=dev) for _ in range(W)]
    views = [c[GUARD:GUARD + W * rps] for c in caches], [b[GUARD:GUARD + W * rps] for b in bases]
    segs = [native.segment_table(views[0][w], t, alias=w if own else None) for w in range(W)]
    return g, rep, m_dev, t, caches, bases, states, views, segs


def _check_workers(rep, m_dev, caches, bases, states):
    torch.cuda.synchronize()
    for o, m in enumerate(m_dev):
        _assert_same(m.cpu().numpy(), _pad(rep.masters[o]), f"master {o}")
    for w in range(rep.W):
        _assert_same(caches[w].cpu().numpy(), _pad(rep.cache[w]), f"replica of worker {w}")
        _assert_same(bases[w].cpu().numpy(), _pad(rep.base[w]), f"base of worker {w}")
        assert np.array_equal(_state_words(states[w].cpu().numpy()), _state_words(rep.state[w]))


@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("own", [False, True], ids=["replicated", "own-in-place"])
@pytest.mark.parametrize("mode", ["sliced", "count"])
def test_workers_one_stream_match_the_replay(dev, W, own, mode):
    rps, stride, n, sync_every = 53, 68, 48, 3
    g, rep, m_dev, t, caches, bases, states, views, segs = _workers(dev, W, rps, stride, own, W * 10 + own)
    per_dest = max(1, n // W)
    if mode == "sliced":       # ReplicaCache with sync_every: every step fires, one rotating slice per flush
        count_max, slices = max(1, per_dest // 2), sync_every
    else:                      # ReplicaCache with a count: head start (o - rank) % sync_every steps
        count_max, slices = max(1, int((sync_every - 0.5) * per_dest)), 1
        for w in range(W):
            head = np.array([((o - w) % sync_every) * per_dest for o in range(W)])
            states[w][:W] += torch.from_numpy(head).to(dev)
            rep.state[w][:W] += head
    for step in range(7):
        for w in range(W):
            ids = g.choice(W * rps, n, replace=False)
            delta = g.standard_normal((n, stride)).astype(np.float32)
            native.push_add(segs[w], torch.from_numpy(ids).to(dev), torch.from_numpy(delta).to(dev))
            rep.push(w, ids, delta)
            native.flush_policy(states[w], W, count_max=count_max, add_uniform=per_dest)
            rep.policy(w, count_max=count_max, add_uniform=per_dest)
            native.replica_exchange(t, views[0][w], views[1][w], state=states[w], n_ctas=5, slices=slices,
                                    slice_offset=w, skip_mask=rep.skip_mask(w))
            rep.exchange(w, slices=slices, slice_offset=w)
    _check_workers(rep, m_dev, caches, bases, states)


@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("own", [False, True], ids=["replicated", "own-in-place"])
def test_workers_overlapping_exchanges_conserve_exactly(dev, W, own):
    """Exchanges on a side stream overlap the pushes on the main stream.  With dyadic deltas every partial sum
    is exact in any interleaving, so after two forced rounds every master is ``init + sum of deltas`` exactly
    and every replica and base equals its master."""
    rps, stride, n = 211, 64, 200
    g, rep, m_dev, t, caches, bases, states, views, segs = _workers(dev, W, rps, stride, own, W + 50 * own,
                                                                    dyadic=True)
    init = np.concatenate(rep.masters)
    total = np.zeros_like(init, dtype=np.float64)
    side = torch.cuda.Stream()
    main = torch.cuda.current_stream()
    for step in range(12):
        for w in range(W):
            ids = g.choice(W * rps, n, replace=False)
            delta = (g.integers(-256, 257, (n, stride)) / 256).astype(np.float32)
            total[(ids % W) * rps + ids // W] += delta
            ev = torch.cuda.Event(); ev.record(main); side.wait_event(ev)
            with torch.cuda.stream(side):
                native.flush_policy(states[w], W, count_max=1, add_uniform=1)
                native.replica_exchange(t, views[0][w], views[1][w], state=states[w], n_ctas=3, slices=3,
                                        slice_offset=w, skip_mask=rep.skip_mask(w))
            native.push_add(segs[w], torch.from_numpy(ids).to(dev), torch.from_numpy(delta).to(dev))
    main.wait_stream(side)
    for _ in range(2):
        for w in range(W):
            native.flush_policy(states[w], W, force=True)
            native.replica_exchange(t, views[0][w], views[1][w], state=states[w], n_ctas=16,
                                    skip_mask=rep.skip_mask(w))
    torch.cuda.synchronize()
    assert np.abs(total).max() < 2 ** 14
    want = (init + total).astype(np.float32)
    got = np.concatenate([m[GUARD:GUARD + rps].cpu().numpy() for m in m_dev])
    assert np.array_equal(got, want)
    for w in range(W):
        keep = np.ones(W * rps, bool)
        if own:
            keep[w * rps:(w + 1) * rps] = False
        assert np.array_equal(views[0][w].cpu().numpy()[keep], want[keep])
        assert np.array_equal(views[1][w].cpu().numpy()[keep], want[keep])
        for buf in (caches[w], bases[w]):
            b = buf.cpu().numpy()
            assert (b[:GUARD] == SENTINEL).all() and (b[-GUARD:] == SENTINEL).all()
    for m in m_dev:
        b = m.cpu().numpy()
        assert (b[:GUARD] == SENTINEL).all() and (b[-GUARD:] == SENTINEL).all()


# ---- ReplicaCache on one GPU ---------------------------------------------------------------------------------

@pytest.mark.parametrize("sync_every", [2, 3, 4, 7])
def test_replica_cache_exchanges_every_row_once_per_cycle(dev, sync_every):
    from fps_b200.store.replica_cache import ReplicaCache
    from fps_b200.store.sharded_table import ShardedTable

    t = ShardedTable(1001, 16, seed=sync_every)
    rc = ReplicaCache(t, sync_every=sync_every, own_inplace=False)
    rps = rc.rps
    rc.cache[:, :16] += 0.25                                  # every row has a pending local delta
    moved = np.zeros(rps, dtype=int)
    for step in range(sync_every):
        before = t.local.clone()
        rc.after_step(1000)
        torch.cuda.synchronize()
        now = (t.local != before).any(dim=1).cpu().numpy()
        lo, hi = ref.slice_range(0, step + 1, 0, rps, sync_every, 0, True)
        assert now[lo:hi].all() and not now[:lo].any() and not now[hi:].any(), f"step {step}"
        moved += now
    assert (moved == 1).all()
    assert rc.flush_counts() == [sync_every]
    t.close()
