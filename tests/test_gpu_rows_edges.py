"""The row primitives of the generic tensor tier (ops/csrc/fps_core.cu: ``fps_pull_gather`` with and without the
pull limiter, ``fps_push_add``, ``fps_push_assign``, ``fps_pull_dot``, ``fps_push_add_fetch`` and the wide-row kernel)
against exact and fp64 replays.

The row widths reach every lane rung of ``pick_lpr`` (1 to 32 lanes per row, one or several 16-byte chunks per lane)
and the wide-row kernel with a partial last segment; the narrow batches are at least three times the capped grid's
lane-groups, so every lane-group runs several grid-stride rounds.  Pushes use dyadic data, whose sums are exact in
any order, so the table must come back bit for bit even under heavy duplication.  The layouts cover one shard and
``MultiShardTable`` with 2 to 16 shards under hash, range (with and without the last-shard clamp) and LUT
partitioning, checked element by element against the host ``locate`` of tests/rows_ref.py with both id widths."""
import numpy as np
import pytest
import torch

from tests import rows_ref
from tests.philox_ref import init_rows_ref

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
MARGIN = 2.0
DIMS = [1, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 300, 1024]
WIDE_DIMS = [1025, 1028, 2048, 4100]
IDTS = [torch.int32, torch.int64]
SHARDS = [2, 3, 4, 5, 16]
NUM_IDS = 1001                      # not a multiple of any shard count above
HOT_REPEATS = 3000


def _sm():
    from fps_b200.ops import native

    torch.cuda.set_device(0)
    return native.sm_count(0)


def _nvec(dim):
    return rows_ref.stride_of(dim) // 4


def _n_rows(dim, sm):
    """Batch rows: three times the capped grid's lane-groups (narrow kernels) or warps over segments (wide kernel)."""
    nvec = _nvec(dim)
    if nvec > rows_ref.WIDE_SEG_VEC:
        n_seg = -(-nvec // rows_ref.WIDE_SEG_VEC)
        return 3 * sm * rows_ref.CTAS_PER_SM * (rows_ref.BLOCK // 32) // n_seg + 5
    return 3 * rows_ref.lane_groups(sm, rows_ref.pick_lpr(nvec)) + 37


def test_sweep_reaches_every_rung():
    sm = _sm()
    lprs = {rows_ref.pick_lpr(_nvec(d)) for d in DIMS}
    assert lprs == {1, 2, 4, 8, 16, 32}
    # a lane with several chunks, and rungs with idle lanes
    assert any(_nvec(d) > 32 for d in DIMS) and any(_nvec(d) < rows_ref.pick_lpr(_nvec(d)) for d in DIMS)
    assert any(_nvec(d) > 64 for d in DIMS) and any(_nvec(d) == 256 for d in DIMS)
    for d in DIMS:
        s = rows_ref.stride_of(d)
        assert not rows_ref.use_wide(s, s, False)
    for d in WIDE_DIMS:
        s = rows_ref.stride_of(d)
        assert rows_ref.use_wide(s, s, False) and not rows_ref.use_wide(s, s, True)
        assert not rows_ref.use_wide(s, d if d % 4 else d - 1, False)
    assert any(_nvec(d) % rows_ref.WIDE_SEG_VEC for d in WIDE_DIMS)
    assert any(_nvec(d) % rows_ref.WIDE_SEG_VEC == 0 for d in WIDE_DIMS)
    # grid-stride rounds at LPR 1, 4 and 32
    for lpr in (1, 4, 32):
        ds = [d for d in DIMS if rows_ref.pick_lpr(_nvec(d)) == lpr]
        assert ds and all(_n_rows(d, sm) >= 3 * rows_ref.lane_groups(sm, lpr) for d in ds)
    assert any(s & (s - 1) for s in SHARDS) and any(not s & (s - 1) for s in SHARDS)   # division and shift paths
    assert max(SHARDS) == 16
    assert all(NUM_IDS % s for s in SHARDS)


def _ids(rng, n, n_ids, hot=True):
    """Zipf and uniform ids, plus one id repeated ``HOT_REPEATS`` times."""
    z = np.minimum(rng.zipf(1.2, n), n_ids) - 1
    u = rng.integers(0, n_ids, n)
    ids = np.where(rng.random(n) < 0.5, z, u)
    if hot:
        ids[:HOT_REPEATS] = n_ids // 2
    return rng.permutation(ids)


def _widths(dim):
    s = rows_ref.stride_of(dim)
    return sorted({dim, s, 1, max(dim - 1, 1), s - 1})


def _dyadic(rng, shape, k, unit):
    return (rng.integers(-k, k + 1, shape) * unit).astype(np.float32)


@pytest.mark.parametrize("idt", IDTS)
@pytest.mark.parametrize("dim", DIMS + WIDE_DIMS)
def test_rows_at_every_rung(dim, idt):
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    sm = _sm()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(dim * 3 + (idt == torch.int32))
    stride = rows_ref.stride_of(dim)
    n_ids = 3000 if dim > 1024 else 4999
    n = _n_rows(dim, sm)
    t = ShardedTable(n_ids, dim, seed=dim, init_range=(-1.0, 1.0))
    tab = t.table_c
    t.local[:, :dim] = torch.from_numpy(_dyadic(rng, (t.local.shape[0], dim), 128, 2.0 ** -8)).to(dev)
    ids_np = _ids(rng, n, n_ids)
    ids = torch.from_numpy(ids_np).to(dev).to(idt)
    il = ids.long()

    # pull: bitwise at every out width (the wide kernel at width == stride, the LPR-32 path otherwise / with touch)
    table0 = t.local.clone()
    for w in _widths(dim):
        out = torch.full((n, w), 7.5, device=dev)
        native.pull_gather(tab, ids, out)
        assert torch.equal(out, table0[il, :w]), w
    out = torch.full((n, stride), 7.5, device=dev)
    native.pull_gather(tab, ids, out, touch=True)
    assert torch.equal(out, table0[il])

    # push_add, exact: dyadic data, every summation order gives the same bits
    for scale in (1.0, 0.5, -2.0):
        for w in (stride, dim, _widths(dim)[-2]):
            before = t.local.clone()
            delta = torch.from_numpy(_dyadic(rng, (n, w), 7, 2.0 ** -7)).to(dev)
            flag = torch.zeros(1, dtype=torch.int32, device=dev)
            native.push_add(tab, ids, delta, scale=scale, nan_flag=flag)
            mag = before.double().abs()
            mag[:, :w].index_add_(0, il, (scale * delta.double()).abs())
            assert float(mag.max()) * 2 ** 8 < 2 ** 24              # every partial sum fits 24 bits of 2^-8
            want = before.double()
            want[:, :w].index_add_(0, il, scale * delta.double())
            assert torch.equal(t.local, want.float()), (scale, w)
            assert torch.equal(t.local.double(), want), (scale, w)     # every partial sum was exact
            assert int(flag) == 0

    # push_add, random values: within the order-independent bound
    before = t.local.clone().double()
    delta = torch.randn(n, stride, device=dev, generator=torch.Generator(device=dev).manual_seed(dim))
    native.push_add(tab, ids, delta, scale=0.75)
    terms = (0.75 * delta.double())
    want = before.clone().index_add_(0, il, terms)
    mag = before.abs().index_add_(0, il, terms.abs())
    cnt = torch.zeros(t.local.shape[0], device=dev, dtype=torch.float64).index_add_(
        0, il, torch.ones(n, device=dev, dtype=torch.float64))[:, None]
    tol = (cnt + 2) * EPS * mag
    assert ((t.local.double() - want).abs() <= MARGIN * tol).all()

    # push_assign: exact; a value width narrower than the stride zeroes the rest of the row
    uniq = torch.from_numpy(rng.permutation(n_ids)[: min(n_ids, 2000)]).to(dev).to(idt)
    for w in (stride, dim, 1):
        vals = torch.from_numpy(_dyadic(rng, (uniq.numel(), w), 1000, 2.0 ** -6)).to(dev)
        keep = t.local.clone()
        native.push_assign(tab, uniq, vals)
        want = keep.clone()
        want[uniq.long()] = 0.0
        want[uniq.long(), :w] = vals
        assert torch.equal(t.local, want), w

    # pull_dot: fp64 replay, local vectors as wide as the row and narrower
    table1 = t.local.double()
    for w in sorted({stride, max(dim - 1, 1), 1}):
        loc = torch.randn(n, w, device=dev)
        score = torch.empty(n, device=dev)
        native.pull_dot(tab, ids, loc, score)
        prod = table1[il, :w] * loc.double()
        tol = (stride + 2) * EPS * prod.abs().sum(1)
        assert ((score.double() - prod.sum(1)).abs() <= MARGIN * tol).all(), w
    t.close()


@pytest.mark.parametrize("dim", [5, 64, 1028])
def test_nan_flag_tracks_non_finite_scaled_deltas(dim):
    """The flag is raised iff some ``scale * delta`` is non-finite (a finite delta can overflow under ``scale``).
    The wide-row kernel does not scan its deltas: a NaN it pushes leaves the flag alone."""
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    _sm()
    dev = torch.device("cuda", 0)
    stride = rows_ref.stride_of(dim)
    wide = rows_ref.use_wide(stride, stride, False)

    def push(value, scale, width, touch=False):
        t = ShardedTable(64, dim, init="zeros", track_touched=touch)
        delta = torch.zeros(40, width, device=dev)
        delta[17, width - 1] = value
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        native.push_add(t.table_c, torch.arange(40, device=dev), delta, scale=scale, touch=touch, nan_flag=flag)
        torch.cuda.synchronize()
        t.close()
        return int(flag)

    narrow_w = dim - 1 if dim % 4 == 0 else dim
    assert push(2.0e38, 1.0, narrow_w) == 0
    assert push(2.0e38, 2.0, narrow_w) == 1                # finite, overflows under scale
    assert push(float("nan"), 1.0, narrow_w) == 1
    assert push(float("inf"), 0.5, narrow_w) == 1
    assert push(1.0, float("inf"), narrow_w) == 1
    assert push(float("nan"), 1.0, stride) == (0 if wide else 1)
    assert push(float("nan"), 1.0, stride, touch=True) == 1   # touch keeps the scanning kernel


@pytest.mark.parametrize("dim", [1, 5, 64])
def test_push_add_fetch_returns_distinct_prefix_sums(dim):
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    sm = _sm()
    dev = torch.device("cuda", 0)
    threads = sm * rows_ref.CTAS_PER_SM * rows_ref.BLOCK
    m = 4096 if dim < 64 else 2048
    K = -(-3 * threads // (dim * m))
    n = K * m
    assert n * dim >= 3 * threads                              # several grid-stride rounds of the capped grid
    rng = np.random.default_rng(dim)
    t = ShardedTable(5 * K + 11, dim, init="zeros")
    t.local[:, :dim] = torch.from_numpy(_dyadic(rng, (t.local.shape[0], dim), 128, 2.0 ** -4)).to(dev)
    init = t.local.clone()
    keys = torch.from_numpy(rng.choice(5 * K + 11, K, replace=False)).to(dev)
    ids = keys.repeat_interleave(m)[torch.from_numpy(rng.permutation(n)).to(dev)]
    out = native.push_add_fetch(t.table_c, ids, torch.ones(n, dim, device=dev))
    order = torch.argsort(ids, stable=True)
    got = out[order].reshape(K, m, dim).sort(dim=1).values
    sk = ids[order].reshape(K, m)[:, 0]
    want = init[sk, :dim][:, None, :] + torch.arange(1, m + 1, device=dev, dtype=torch.float32)[None, :, None]
    assert torch.equal(got, want)
    final = init.clone()
    final[keys, :dim] += m
    assert torch.equal(t.local, final)
    t.close()


# ---- layouts ----------------------------------------------------------------------------------------------------
def _partitioner(n):
    return lambda i: (i * 7 + i // 5) % n


def _layout(num_shards, partition, dim, num_ids=NUM_IDS, **kw):
    """(table, pointer table, locate kwargs, usable ids).  ``range_clamp`` is a range table addressed with a divisor
    below ceil(num_ids / G), so the last shard takes the ids past ``G * div`` through the clamp."""
    from fps_b200.ops import native
    from fps_b200.store.multi_shard import MultiShardTable

    if partition == "lut":
        m = MultiShardTable(num_ids, dim, num_shards, partitioner=_partitioner(num_shards), devices=[0],
                            init="zeros", **kw)
        return m, m.table_c, dict(mode=rows_ref.LUT, num_shards=num_shards, div=m.div,
                                  lut=rows_ref.lut_from_partitioner(num_ids, num_shards,
                                                                    _partitioner(num_shards))), num_ids
    if partition == "range_clamp":
        m = MultiShardTable(1200, dim, num_shards, partition="range", devices=[0], init="zeros", **kw)
        tc = native.ShardTableC.from_buffer_copy(m.table_c)
        tc.div = num_ids // num_shards
        assert num_shards * tc.div < num_ids and num_ids - (num_shards - 1) * tc.div <= m.rows_per_shard
        return m, tc, dict(mode=rows_ref.RANGE, num_shards=num_shards, div=tc.div), num_ids
    m = MultiShardTable(num_ids, dim, num_shards, partition=partition, devices=[0], init="zeros", **kw)
    mode = rows_ref.HASH if partition == "hash" else rows_ref.RANGE
    return m, m.table_c, dict(mode=mode, num_shards=num_shards, div=m.div), num_ids


def _shards(m):
    torch.cuda.synchronize()
    return np.stack([s.cpu().numpy() for s in m.shards])


def _run_layout(num_shards, partition, dim, seed=0):
    """Assign with 32-bit ids, read back with 64-bit ones, push-add with 64-bit ids, read back with 32-bit ones.
    Returns (shards after the assign, values, locate kwargs, rows_per_shard, stride)."""
    from fps_b200.ops import native

    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(seed + 13 * num_shards + dim)
    m, tc, loc, nid = _layout(num_shards, partition, dim)
    stride = rows_ref.stride_of(dim)
    ids = rng.permutation(nid)
    cols = np.arange(dim, dtype=np.float32)
    vals = (ids[:, None].astype(np.float32) + cols[None, :] / 128).astype(np.float32)
    native.push_assign(tc, torch.from_numpy(ids).to(dev).int(), torch.from_numpy(vals).to(dev))
    assigned = _shards(m)
    order = rng.permutation(nid)
    out = torch.empty(nid, dim, device=dev)
    native.pull_gather(tc, torch.from_numpy(ids[order]).to(dev), out)
    assert np.array_equal(out.cpu().numpy(), vals[order])
    delta = (rng.integers(-64, 65, (nid, stride)) / 64.0).astype(np.float32)
    native.push_add(tc, torch.from_numpy(ids).to(dev), torch.from_numpy(delta).to(dev))
    native.pull_gather(tc, torch.from_numpy(ids[order]).to(dev).int(), out)
    want = vals.astype(np.float64) + delta[:, :dim]
    assert np.array_equal(out.cpu().numpy().astype(np.float64), want[order])
    m.close()
    return assigned, ids, vals, loc, m.rows_per_shard, stride


@pytest.mark.parametrize("dim", [3, 130])
@pytest.mark.parametrize("partition", ["hash", "range", "range_clamp", "lut"])
@pytest.mark.parametrize("num_shards", SHARDS)
def test_shard_layout_matches_host_locate(num_shards, partition, dim):
    _sm()
    assigned, ids, vals, loc, rps, stride = _run_layout(num_shards, partition, dim)
    owner, slot = rows_ref.locate(ids, **loc)
    want = rows_ref.place(ids, vals, owner, slot, num_shards, rps, stride)
    assert want is not None and np.array_equal(assigned, want)   # every row where locate says, nothing elsewhere


def test_broken_locates_fail():
    _sm()
    counts = {b: 0 for b in rows_ref.BREAKS}
    cases = 0
    for num_shards in (3, 4, 16):
        for partition in ("hash", "range_clamp", "lut"):
            assigned, ids, vals, loc, rps, stride = _run_layout(num_shards, partition, 3, seed=1)
            for b in rows_ref.BREAKS:
                owner, slot = rows_ref.locate(ids, **loc, breaks=b)
                want = rows_ref.place(ids, vals, owner, slot, num_shards, rps, stride)
                counts[b] += want is None or not np.array_equal(assigned, want)
            cases += 1
    print(f"\nLOCATE_SENSITIVITY failing cases of {cases}: {counts}")
    assert all(v > 0 for v in counts.values()), counts


@pytest.mark.parametrize("dim", [5, 64])
@pytest.mark.parametrize("partition", ["hash", "range"])
def test_init_rows_per_shard(partition, dim):
    from fps_b200.store.multi_shard import MultiShardTable

    _sm()
    for num_shards in SHARDS:
        m = MultiShardTable(NUM_IDS, dim, num_shards, partition=partition, devices=[0], init="uniform",
                            init_range=(-0.01, 0.01), seed=77)
        for s in range(num_shards):
            ref = init_rows_ref(m.shard_ids(s).cpu().numpy(), dim, 77, -0.01, 0.01)
            np.testing.assert_allclose(m.shards[s].cpu().numpy(), ref, rtol=0, atol=1e-9)
        m.close()


@pytest.mark.parametrize("multi", [False, True])
def test_touched_bitmap_is_the_set_of_touched_ids(multi):
    from fps_b200.store.multi_shard import MultiShardTable
    from fps_b200.store.sharded_table import ShardedTable

    _sm()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(5 + multi)
    dim = 9
    t = (MultiShardTable(NUM_IDS, dim, 3, devices=[0], track_touched=True) if multi
         else ShardedTable(NUM_IDS, dim, track_touched=True))
    a, b, c = (rng.choice(NUM_IDS, k, replace=True) for k in (150, 120, 90))
    t.pull(torch.from_numpy(a).to(dev))
    t.push(torch.from_numpy(b).to(dev).int(), torch.ones(b.size, dim, device=dev))
    t.load(torch.from_numpy(c).to(dev), torch.zeros(c.size, dim, device=dev))
    got, _ = t.dump_local(only_touched=True)
    assert sorted(got.tolist()) == sorted(set(a.tolist()) | set(b.tolist()) | set(c.tolist()))
    all_ids, _ = t.dump_local(only_touched=False)
    assert sorted(all_ids.tolist()) == list(range(NUM_IDS))
    t.close()


# ---- pull limiter -----------------------------------------------------------------------------------------------
@pytest.mark.timeout(120)
@pytest.mark.parametrize("limit", [1, 3, 64])
@pytest.mark.parametrize("dim", [4, 16, 128])          # LPR 1, 4, 32
def test_pull_limiter_is_bitwise_the_free_pull(dim, limit):
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    _sm()
    dev = torch.device("cuda", 0)
    assert rows_ref.pick_lpr(_nvec(dim)) in (1, 4, 32)
    t = ShardedTable(4999, dim, seed=4, init_range=(-1.0, 1.0))
    ids = torch.from_numpy(_ids(np.random.default_rng(dim + limit), 20000, 4999)).to(dev)
    free = t.pull(ids)
    lim = t.pull(ids, pull_limit=limit)
    assert torch.equal(lim, free)
    assert int(t._credits(limit, dev)[0]) == limit
    out = torch.empty_like(free)
    native.pull_gather(t.table_c, ids, out, max_inflight_rows=limit)     # the static limiter: a capped grid
    assert torch.equal(out, free)
    t.close()


# ---- alignment: refused before any launch -----------------------------------------------------------------------
@pytest.mark.parametrize("dim", [8, 1028])
def test_misaligned_row_buffers_are_refused(dim):
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    _sm()
    dev = torch.device("cuda", 0)
    n = 64
    t = ShardedTable(100, dim, seed=1)
    ids = torch.arange(n, device=dev)
    for off in (1, 2, 3):
        bad = torch.empty(off + dim * n, device=dev)[off:].view(n, dim)
        assert bad.is_contiguous() and bad.data_ptr() % 16 != 0
        before = native.launch_count()
        with pytest.raises(ValueError):
            t.pull(ids, out=bad)
        with pytest.raises(ValueError):
            native.pull_gather(t.table_c, ids, bad, max_inflight_rows=8)
        with pytest.raises(ValueError):
            t.push(ids, bad)
        with pytest.raises(ValueError):
            native.push_add(t.table_c, ids, bad, scale=2.0)
        assert native.launch_count() == before
    ok = torch.full((4 + dim * n,), 3.0, device=dev)[4:].view(n, dim)   # offset of 4 floats: aligned, accepted
    t.pull(ids, out=ok)
    assert torch.equal(ok, t.local[:n, :dim])
    t.close()
