"""Exact replay of the replica (item-cache) kernels of ``ops/csrc/fps_replica.cu`` and ``fps_bucket.cu``.

numpy only, float32, bitwise: within one launch every element of the exchange is computed by one thread with
plain ``FADD`` (no flush) for ``d = c - b``, ``f = v - b`` and ``b = v + d``, and both reductions are
``REDG.E.ADD.F32x4.FTZ``: inputs and result flushed, ``ftz(ftz(x) + ftz(y))``.  So a kernel that is right
matches the replay bit for bit, and no tolerance is needed.

* :func:`policy` -- ``fps_flush_policy_kernel`` on a copy of the 49-word ``FlushState``; the clock is an input
  (``interval_passed`` per destination).
* :func:`slice_range` -- the per-destination ``[lo, hi)`` of one launch, shared by both exchange kernels.
* :func:`exchange` -- one exchange launch.
* :func:`deal` -- the bucket and owner of every record of ``fps_bucket_deal_kernel`` and the per-owner feed.
  The order inside a bucket depends on the schedule and is not replayed.
* :class:`Workers` -- W workers with a replica each against W master shards, replayed in stream order.
"""
import numpy as np

MAX_SHARDS = 16
STATE_WORDS = 3 * MAX_SHARDS + 1
PENDING, LAST_NS, COUNT, MASK = 0, MAX_SHARDS, 2 * MAX_SHARDS, 3 * MAX_SHARDS   # word 48: mask | evals << 32
U64 = (1 << 64) - 1
TINY = np.finfo(np.float32).tiny


def ftz(x):
    """Flush float32 subnormals to zero of the same sign (NaN and inf pass)."""
    x = np.array(x, dtype=np.float32, copy=True)
    sub = (x != 0) & (np.abs(x) < TINY)
    x[sub] = np.copysign(np.float32(0), x[sub])
    return x


def red_add(x, y, flush=True):
    """``red.global.add.f32``: both operands and the sum flushed."""
    with np.errstate(all="ignore"):
        if not flush:
            return np.asarray(x, np.float32) + np.asarray(y, np.float32)
        return ftz(ftz(x) + ftz(y))


# ---- flush policy --------------------------------------------------------------------------------------------

def mask_word(state):
    return int(state[MASK]) & 0xFFFFFFFF


def evals(state):
    return (int(state[MASK]) >> 32) & 0xFFFFFFFF


def policy(state, num_dest, count_max=0, interval_passed=None, require_all=False, force=False, add_uniform=0):
    """One ``fps_flush_policy_kernel`` launch on a copy of ``state`` (int64 ``[49]``); returns the copy.

    ``interval_passed``: ``None`` when the timer is off, else per destination whether its deadline has passed.
    Per destination ``o < num_dest``: ``pending += add_uniform``; the count trigger is ``pending >= count_max``
    (``count_max`` 0: off); the timer trigger needs a message pending; AND needs every enabled trigger and at
    least one enabled; ``force`` fires everything.  On fire ``pending`` drops by what was counted, ``flushes``
    rises by one.  The mask word gets the fired bits and ``evals`` one more.  ``last_ns`` is a clock and is not
    replayed."""
    st = [int(w) & U64 for w in np.asarray(state, dtype=np.int64)]
    has_count, has_timer = count_max != 0, interval_passed is not None
    m = 0
    for o in range(num_dest):
        pend = (st[PENDING + o] + add_uniform) & U64
        st[PENDING + o] = pend
        cnt = has_count and pend >= count_max
        tim = has_timer and pend != 0 and bool(interval_passed[o])
        if force:
            fire = True
        elif require_all:
            fire = (has_count or has_timer) and (not has_count or cnt) and (not has_timer or tim)
        else:
            fire = cnt or tim
        if fire:
            st[PENDING + o] = (st[PENDING + o] - pend) & U64
            st[COUNT + o] = (st[COUNT + o] + 1) & U64
            m |= 1 << o
    ev = (((st[MASK] >> 32) + 1) & 0xFFFFFFFF)
    st[MASK] = m | (ev << 32)
    return np.array([w - (1 << 64) if w >= 1 << 63 else w for w in st], dtype=np.int64)


# ---- exchange ------------------------------------------------------------------------------------------------

def slice_range(o, flushes, slot_lo, slot_hi, slices, slice_offset, sliced):
    """``[lo, hi)`` of destination ``o`` in one launch; ``flushes`` is its counter after the policy ran."""
    lo, hi = slot_lo, slot_hi
    if sliced:
        length = -(-(slot_hi - slot_lo) // slices)
        sl = ((flushes + ((o + slice_offset) & U64)) & U64) % slices
        lo = slot_lo + sl * length
        hi = min(lo + length, slot_hi)
        lo = min(lo, hi)
    return lo, hi


def ranges_for(num_shards, slot_lo, slot_hi, state=None, slices=1, slice_offset=0):
    """The ``[lo, hi)`` of every destination for a launch with these arguments (slicing needs ``state``)."""
    sliced = slices > 1 and state is not None
    fl = [0] * num_shards if state is None else [int(state[COUNT + o]) & U64 for o in range(num_shards)]
    return [slice_range(o, fl[o], slot_lo, slot_hi, slices, slice_offset, sliced) for o in range(num_shards)]


def launch_mask(mask, skip_mask, num_shards):
    return mask & ((1 << num_shards) - 1) & ~skip_mask & 0xFFFFFFFF


def exchange(master_list, cache, base, mask, skip_mask, num_shards, ranges, flush=True):
    """One exchange launch; returns new ``(masters, cache, base)``.  ``master_list[o]``: ``[rps, stride]``;
    ``cache`` / ``base``: ``[num_shards * rps, stride]``; ``ranges[o]``: ``(lo, hi)`` slots of destination o.

    Gating is per float4 group: a group pushes when any lane of ``d`` is nonzero (NaN counts, -0 does not),
    folds when any lane of ``f`` is, and writes ``b = v + d`` (no flush) when it did either.  ``flush=False``
    gives the textbook update without FTZ."""
    masters = [np.array(m, dtype=np.float32, copy=True) for m in master_list]
    cache = np.array(cache, dtype=np.float32, copy=True)
    base = np.array(base, dtype=np.float32, copy=True)
    stride = cache.shape[1]
    rps = cache.shape[0] // num_shards
    m = launch_mask(mask, skip_mask, num_shards)
    with np.errstate(all="ignore"):
        for o in range(num_shards):
            lo, hi = ranges[o]
            if not (m >> o) & 1 or hi <= lo:
                continue
            rows = slice(o * rps + lo, o * rps + hi)
            v = masters[o][lo:hi].reshape(hi - lo, stride // 4, 4)
            c = cache[rows].reshape(hi - lo, stride // 4, 4)
            b = base[rows].reshape(hi - lo, stride // 4, 4)
            d = c - b
            f = v - b
            has_d = (d != 0).any(axis=-1, keepdims=True)
            has_f = (f != 0).any(axis=-1, keepdims=True)
            nm = np.where(has_d, red_add(v, d, flush), v)
            nc = np.where(has_f, red_add(c, f, flush), c)
            nb = np.where(has_d | has_f, v + d, b)
            masters[o][lo:hi] = nm.reshape(hi - lo, stride)
            cache[rows] = nc.reshape(hi - lo, stride)
            base[rows] = nb.reshape(hi - lo, stride)
    return masters, cache, base


# ---- bucket deal ---------------------------------------------------------------------------------------------

def deal(items, num_shards, rps, shift, n_buckets):
    """Bucket of every record and the per-owner feed of ``fps_bucket_deal_kernel``.  ``items``: the decoded
    item ids (int64).  The owner and slot come from ``|item|``; the bucket is the owner-major row
    ``owner * rps + slot`` (plain ``|item|`` for one shard) ``>> shift``, clamped to the last bucket."""
    a = np.abs(np.asarray(items, dtype=np.int64))
    if num_shards > 1:
        owner = a % num_shards
        row = owner * rps + a // num_shards
    else:
        owner = np.zeros_like(a)
        row = a
    bucket = np.minimum(row >> shift, n_buckets - 1)
    return bucket, np.bincount(owner, minlength=num_shards)


def bucket_groups(records, bucket, n_buckets):
    """Sorted multiset of the records of every bucket."""
    records = np.asarray(records)
    return [np.sort(records[bucket == k]) for k in range(n_buckets)]


# ---- W workers on one device ---------------------------------------------------------------------------------

class Workers:
    """W workers, each with an owner-major replica, its base and a flush state, against W master shards (hash
    partition: id ``i`` lives in shard ``i % W`` at slot ``i // W``).  ``own_inplace``: worker w pushes the ids of
    shard w straight into the master and never exchanges that segment.  Replays, in stream order, the
    operations of :meth:`push` (``push_add``), :meth:`policy` (``flush_policy``) and :meth:`exchange`."""

    def __init__(self, W, rps, stride, own_inplace, masters):
        self.W, self.rps, self.stride, self.own_inplace = W, rps, stride, own_inplace
        self.masters = [np.array(m, dtype=np.float32, copy=True) for m in masters]
        full = np.concatenate(self.masters)
        self.cache = [full.copy() for _ in range(W)]
        self.base = [full.copy() for _ in range(W)]
        self.state = [np.zeros(STATE_WORDS, dtype=np.int64) for _ in range(W)]

    def skip_mask(self, w):
        return 1 << w if self.own_inplace else 0

    def push(self, w, ids, delta):
        """``push_add`` of distinct ``ids`` with ``delta`` (``[n, <= stride]``, zero padded) by worker w."""
        delta = np.asarray(delta, dtype=np.float32)
        full = np.zeros((len(ids), self.stride), dtype=np.float32)
        full[:, : delta.shape[1]] = delta
        for i, r in zip(np.asarray(ids, dtype=np.int64), full):
            o, s = int(i) % self.W, int(i) // self.W
            if self.own_inplace and o == w:
                self.masters[o][s] = red_add(self.masters[o][s], r)
            else:
                self.cache[w][o * self.rps + s] = red_add(self.cache[w][o * self.rps + s], r)

    def policy(self, w, **kw):
        self.state[w] = policy(self.state[w], self.W, **kw)

    def exchange(self, w, slices=1, slice_offset=0):
        rng = ranges_for(self.W, 0, self.rps, self.state[w], slices, slice_offset)
        self.masters, self.cache[w], self.base[w] = exchange(
            self.masters, self.cache[w], self.base[w], mask_word(self.state[w]), self.skip_mask(w), self.W, rng)
