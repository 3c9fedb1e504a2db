"""The pointwise MF step (``fps_mf_sgd_fused_kernel``, the TMA kernel ``fps_mf_sgd_tma_kernel`` and the fp64 kernel
``fps_mf_sgd_fused_f64_kernel``) against an fp64 replay of the same step (``tests/pointwise_ref.py``), at every
dispatch rung, with in-kernel negatives replayed by ``tests/philox_ref.py``.

Every case is built so that its result does not depend on the order the lane-groups run in: each row is read and
written by one record (or, for hot rows, only on coordinates that one record owns), so the replay applies the records
independently.  Every table is a slice of a larger tensor whose guard rows hold a sentinel; each case checks that the
guard rows, the padding columns and the rows outside the batch are bitwise unchanged."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests.philox_ref import init_rows_f64_ref, k5_negative, philox4x32
from tests.pointwise_ref import MARGIN, loss_bound, replay

pytestmark = pytest.mark.gpu

GUARD = 3                 # sentinel rows on each side of every table
SENTINEL = -4242.5
EPS = 2.0 ** -24          # fp32 unit roundoff

# dispatch_mf (csrc/fps_core.cu) for the SGD step: dim -> stride -> nvec = stride / 4 float4 per row -> <LPR, VPL, R>
# (lanes per row, float4 per lane, rows in flight per lane-group).  Every dim leaves lanes or columns empty.
#   dim  stride  nvec  <LPR, VPL, R>
#     3      4     1   < 1, 1, 2>
#     7      8     2   < 2, 1, 2>
#    13     16     4   < 4, 1, 2>
#    29     32     8   < 8, 1, 1>
#    61     64    16   <16, 1, 1>   reg variants 1 <16,1,4>, 3 <16,1,2>, 5 <16,1,2>, 9 <8,2,2>; l2_hints <16,1,1>
#   125    128    32   <32, 1, 1>
#   129    132    33   <32, 2, 1>   lane 0 holds 2 float4, the others 1
#   253    256    64   <32, 2, 1>
#   300    300    75   <32, 3, 1>
#   509    512   128   <32, 4, 1>
#  1021   1024   256   <32, 8, 1>
REG_LPR = {3: 1, 7: 2, 13: 4, 29: 8, 61: 16, 125: 32, 129: 32, 253: 32, 300: 32, 509: 32, 1021: 32}
VARIANT_LPR = {1: 16, 3: 16, 5: 16, 9: 8}
IDS = ("int32", "int64", "packed64")

# Each rung twice, with a different id form and error rule each time (every (id form, err_mode) pair occurs), the
# second time with the user rows read through a ShardTable (the user_sharded path).
RUNG_CASES = [(dim, IDS[(i + s) % 3], (i // 3 + s) % 3, s == 1) for i, dim in enumerate(REG_LPR) for s in (0, 1)]


def _stride(dim):
    return (dim + 3) // 4 * 4


def _tma_lpr(nvec):
    """dispatch_tma (csrc/fps_mf_tma.cu): one lane per float4 up to 32 lanes."""
    return min(32, 1 << max(0, nvec - 1).bit_length())


def _within(got, want, tol, what):
    bad = np.abs(got - want) > MARGIN * tol
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} elements off, worst "
                           f"{float(np.max(np.abs(got - want) - MARGIN * tol)):.3g} beyond the bound")


# ---- guarded tables -------------------------------------------------------------------------------------------

class Guarded:
    """``rows`` rows of ``width`` columns inside a tensor with GUARD sentinel rows on each side."""

    def __init__(self, rows, width, dtype, dev):
        self.big = torch.full((rows + 2 * GUARD, width), SENTINEL, dtype=dtype, device=dev)
        self.t = self.big[GUARD:GUARD + rows]
        self.dtype = dtype

    def check_guards(self):
        assert (self.big[:GUARD] == SENTINEL).all() and (self.big[-GUARD:] == SENTINEL).all(), "guard row written"


def _table(rows, dim, scale, gen, dev, dtype=torch.float32, width=None):
    g = Guarded(rows, width or _stride(dim), dtype, dev)
    g.t.zero_()
    g.t[:, :dim] = ((torch.rand(rows, dim, generator=gen, device=dev, dtype=torch.float64) * 2 - 1) * scale).to(dtype)
    return g


def _check_table(g, before, dim, touched, what):
    """Guards, padding columns and untouched rows bitwise unchanged."""
    g.check_guards()
    assert not g.t[:, dim:].any(), f"{what}: padding column written"
    keep = torch.ones(g.t.shape[0], dtype=torch.bool, device=g.t.device)
    keep[torch.as_tensor(np.asarray(touched, dtype=np.int64), device=g.t.device)] = False
    assert torch.equal(g.t[keep], before[keep]), f"{what}: a row outside the batch moved"


def _ratings(n, rng, err_mode):
    """fp16-representable ratings (packed64 records carry fp16): 0.5 to 4 in halves for the plain residual, 0/1
    labels for the two logistic rules."""
    if err_mode == 1:
        return rng.integers(1, 9, size=n).astype(np.float32) * np.float32(0.5)
    return rng.integers(0, 2, size=n).astype(np.float32)


def _ids(users, items, ratings, form, dev):
    """(users, items, ratings) arguments of native.mf_sgd_fused in one of the three id forms."""
    u = torch.from_numpy(np.asarray(users, dtype=np.int64))
    i = torch.from_numpy(np.asarray(items, dtype=np.int64))
    r = torch.from_numpy(np.asarray(ratings, dtype=np.float32))
    if form == "packed64":
        return native.pack_ratings(u, i, r).to(dev), None, None
    dt = torch.int32 if form == "int32" else torch.int64
    return u.to(dev, dt), i.to(dev, dt), r.to(dev)


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _pointwise(dev, dim, form, err_mode, *, lpr, n=3000, rows=3600, seed=0, lr=0.05, user_div=1,
               user_sharded=False, void_every=0, **kw):
    """One launch on a conflict-free batch: ``n`` records of distinct users and distinct items drawn from ``rows``
    rows, every ``void_every``-th record voided (user -1).  Checks the tables and stats against the replay and
    returns (user table, item table, user ids) after the launch."""
    gen = torch.Generator(device=dev).manual_seed(1000 * dim + seed)
    rng = np.random.default_rng(1000 * dim + seed)
    scale = dim ** -0.25
    U, V = _table(rows, dim, scale, gen, dev), _table(rows, dim, scale, gen, dev)
    U0, V0 = U.t.clone(), V.t.clone()
    slots = rng.permutation(rows)[:n]
    items = rng.permutation(rows)[:n]
    r = _ratings(n, rng, err_mode)
    users = slots * user_div + (user_div - 1)
    live = np.ones(n, dtype=bool)
    if void_every:
        live[::void_every] = False
        users = np.where(live, users, -1)
    stats = torch.zeros(2, device=dev)
    nan = torch.zeros(1, dtype=torch.int32, device=dev)
    a, b, c = _ids(users, items, r, form, dev)
    user_table = native.local_table(U.t, dim) if user_sharded else U.t
    native.mf_sgd_fused(a, b, c, user_table, user_div, native.local_table(V.t, dim), lr, err_mode=err_mode,
                        stats=stats, nan_flag=nan, **kw)
    torch.cuda.synchronize()
    s, it = slots[live], items[live]
    u0 = U0[torch.from_numpy(s).to(dev), :dim].double().cpu().numpy()
    v0 = V0[torch.from_numpy(it).to(dev), :dim].double().cpu().numpy()
    res = replay(u0, v0, r[live].astype(np.float64), lr, err_mode, lpr)
    _within(U.t[torch.from_numpy(s).to(dev), :dim].double().cpu().numpy(), res.u, res.tol_u, "user rows")
    _within(V.t[torch.from_numpy(it).to(dev), :dim].double().cpu().numpy(), res.v, res.tol_v, "item rows")
    _check_table(U, U0, dim, s, "user table")
    _check_table(V, V0, dim, it, "item table")
    st = stats.cpu().numpy().astype(np.float64)
    assert st[1] == live.sum()
    assert abs(st[0] - (res.resid * res.resid).sum()) <= MARGIN * loss_bound(res.resid, res.tol_resid)
    assert int(nan.item()) == 0
    return U, V, users


# ---- 1. every rung of dispatch_mf ------------------------------------------------------------------------------

def test_rung_cases_cover_the_ladder():
    assert len({REG_LPR[d] for d, _, _, _ in RUNG_CASES}) == 6
    assert {(f, m) for _, f, m, _ in RUNG_CASES} == {(f, m) for f in IDS for m in range(3)}
    assert sorted({(_stride(d) // 4 + REG_LPR[d] - 1) // REG_LPR[d] for d in REG_LPR}) == [1, 2, 3, 4, 8]


@pytest.mark.parametrize("dim,form,err_mode,user_sharded", RUNG_CASES)
def test_sgd_rung_matches_fp64_replay(dev, dim, form, err_mode, user_sharded):
    _pointwise(dev, dim, form, err_mode, lpr=REG_LPR[dim], user_sharded=user_sharded)


@pytest.mark.parametrize("variant", [1, 3, 5, 9])
@pytest.mark.parametrize("form", ["int32", "packed64"])
def test_reg_variants_match_fp64_replay(dev, monkeypatch, variant, form):
    monkeypatch.setenv("FPS_MF_REG_VARIANT", str(variant))
    try:
        _pointwise(dev, 61, form, variant % 3, lpr=VARIANT_LPR[variant])
    finally:
        native.lib().fps_set_mf_reg_variant(0)


@pytest.mark.parametrize("form", IDS)
def test_l2_hints_match_fp64_replay(dev, form):
    _pointwise(dev, 61, form, 0, lpr=16, l2_hints=True)


def test_user_div_not_a_power_of_two(dev):
    _pointwise(dev, 29, "int64", 1, lpr=8, user_div=3)


def test_dim_above_1024_is_refused(dev):
    U = torch.zeros(8, 1028, device=dev)
    V = torch.zeros(8, 1028, device=dev)
    ids = torch.arange(4, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError, match="-1000"):
        native.mf_sgd_fused(ids, ids, torch.ones(4, device=dev), U, 1, native.local_table(V, 1025), 0.1)
    torch.cuda.synchronize()
    assert not U.any() and not V.any()


# ---- 2. output stream, credit counter and TMA rungs ------------------------------------------------------------

SIDE_DIMS = [13, 29, 61, 125, 509]   # nvec 4, 8, 16, 32, 128: the rungs of the output-stream and credit dispatch


@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("dim", SIDE_DIMS)
def test_output_stream_stages_the_updated_user_rows(dev, dim, every):
    n, cap, start = 3000, 700, 5
    gen = torch.Generator(device=dev).manual_seed(dim)
    o_ids = torch.full((cap,), -7, dtype=torch.int64, device=dev)
    o_vecs = torch.full((cap, _stride(dim)), SENTINEL, device=dev)
    staged = torch.tensor([start], dtype=torch.int64, device=dev)
    U, V, users = _pointwise(dev, dim, "int32", 1, lpr=REG_LPR[dim], n=n,
                             output=(o_ids, o_vecs, staged, cap, every))
    idx = np.arange(0, n, every)
    slot = start + idx // every
    keep = slot < cap
    want_ids = np.full(cap, -7)
    want_ids[slot[keep]] = users[idx[keep]]
    assert np.array_equal(o_ids.cpu().numpy(), want_ids)
    assert (o_ids >= 0).sum().item() == min(cap - start, len(idx))
    # the staged vector is this update's u + g v, the row the table holds afterwards (distinct users: bitwise)
    got = o_vecs[torch.from_numpy(slot[keep]).to(dev)]
    assert torch.equal(got, U.t[torch.from_numpy(users[idx[keep]]).to(dev)])
    rest = torch.ones(cap, dtype=torch.bool, device=dev)
    rest[torch.from_numpy(slot[keep]).to(dev)] = False
    assert (o_vecs[rest] == SENTINEL).all()
    assert staged.item() == start


@pytest.mark.parametrize("limit", [32, 96])   # a warp takes a credit per lane-group at once: at most 32
@pytest.mark.parametrize("dim", SIDE_DIMS)
def test_credit_counter_returns_every_credit(dev, dim, limit):
    credits = torch.tensor([limit, 0], dtype=torch.int32, device=dev)
    U, V, _ = _pointwise(dev, dim, "int64", 0, lpr=REG_LPR[dim], credits=credits, max_inflight_rows=limit)
    assert credits[0].item() == limit and credits[1].item() >= 0
    U2, V2, _ = _pointwise(dev, dim, "int64", 0, lpr=REG_LPR[dim])    # same geometry without the counter
    assert torch.equal(U.t, U2.t) and torch.equal(V.t, V2.t)


TMA_DIMS = [3, 7, 13, 29, 61, 125, 300, 1021]   # LPR 1..32; 300 takes 3 float4 per lane; 1021 overflows the ring


@pytest.mark.parametrize("form", ["int32", "int64"])
@pytest.mark.parametrize("dim", TMA_DIMS)
def test_tma_rung_matches_fp64_replay(dev, dim, form):
    nvec = _stride(dim) // 4
    stage_bytes = 2 * 32 * _stride(dim) * 4 + 32 * 24 + 16
    fallback = (200 * 1024 // stage_bytes) < 2
    assert fallback == (dim == 1021)
    lpr = REG_LPR[dim] if fallback else _tma_lpr(nvec)
    _pointwise(dev, dim, form, dim % 3, lpr=lpr, kernel="tma", user_sharded=(form == "int64"))


# ---- 3. grid-stride rounds -------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim,variant,kernel", [(3, 0, "reg"), (7, 0, "reg"), (13, 0, "reg"), (61, 1, "reg"),
                                                (61, 9, "reg"), (1021, 0, "reg"), (61, 0, "tma"), (300, 0, "tma")])
def test_grid_stride_rounds_equal_the_default_grid(dev, monkeypatch, dim, variant, kernel):
    """A grid capped to one CTA by max_inflight_rows (every lane-group runs many rounds, with all R slots live) and
    to one CTA per SM by reserve_total (more records than that grid's lane-group slots) computes bitwise what the
    default grid does."""
    lpr = VARIANT_LPR[variant] if variant else (_tma_lpr(_stride(dim) // 4) if kernel == "tma" else REG_LPR[dim])
    r_slots = {1: 4, 3: 2, 5: 2, 9: 2}.get(variant, 2 if dim <= 13 and kernel == "reg" else 1)
    per_round = native.sm_count(0) * (256 // lpr) * r_slots
    n = per_round + per_round // 2 + 1 if kernel == "reg" else 20000
    rows = n + 500
    if variant:
        monkeypatch.setenv("FPS_MF_REG_VARIANT", str(variant))
    try:
        runs = [_pointwise(dev, dim, "int32", 1, lpr=lpr, n=n, rows=rows, kernel=kernel, **kw)
                for kw in ({}, {"max_inflight_rows": 1}, {"reserve_total": 1 << 20})]
    finally:
        native.lib().fps_set_mf_reg_variant(0)
    for U, V, _ in runs[1:]:
        assert torch.equal(U.t, runs[0][0].t) and torch.equal(V.t, runs[0][1].t)


# ---- 4. in-kernel negatives, replayed --------------------------------------------------------------------------

SEED = (7 << 32) + 12345    # both key words live
STEP = 5


def _negative_batch(n_pos, neg_rate, num_items, step, seed):
    """Positive items equal to their own j = 1 raw draw (so the rejection branch fires on every record), and the
    records whose items would meet another record's voided.  Returns (items, live, negatives [n_pos, neg_rate])."""
    pos = np.arange(n_pos)
    _, raw1 = k5_negative(pos, 1, np.full(n_pos, -1), num_items, step, seed)
    items = raw1
    negs = np.stack([k5_negative(pos, j, items, num_items, step, seed)[0] for j in range(1, neg_rate + 1)], 1)
    used, live = set(), np.zeros(n_pos, dtype=bool)
    for p in range(n_pos):
        rows = {int(items[p]), *map(int, negs[p])}
        if len(rows) == 1 + neg_rate and not rows & used:
            used |= rows
            live[p] = True
    return items, live, negs


@pytest.mark.parametrize("kernel,form,neg_rate", [("reg", "int32", 1), ("reg", "int64", 3), ("tma", "int32", 2),
                                                  ("tma", "int64", 1)])
def test_negatives_match_the_replayed_stream(dev, kernel, form, neg_rate):
    """Item table all zero: every pull reads zero, so each user row stays bitwise what it was and each drawn row
    becomes exactly lr * e * u, with e = r - sigmoid(0) = r - 1/2 (err_mode 2)."""
    dim, n_pos, num_items, lr = 29, 2000, 1 << 18, 0.25
    gen = torch.Generator(device=dev).manual_seed(3)
    U = _table(n_pos, dim, 0.5, gen, dev)
    V = Guarded(num_items, _stride(dim), torch.float32, dev)
    V.t.zero_()
    U0 = U.t.clone()
    items, live, negs = _negative_batch(n_pos, neg_rate, num_items, STEP, SEED)
    assert 0.9 * n_pos < live.sum() < n_pos                      # some records voided, most live
    users = np.where(live, np.random.default_rng(4).permutation(n_pos), -1)
    r = np.ones(n_pos, dtype=np.float32)
    stats = torch.zeros(2, device=dev)
    a, b, c = _ids(users, items, r, form, dev)
    native.mf_sgd_fused(a, b, c, U.t, 1, native.local_table(V.t, dim), lr, err_mode=2, neg_rate=neg_rate,
                        num_items=num_items, seed=SEED, step=STEP, stats=stats, kernel=kernel)
    torch.cuda.synchronize()
    U.check_guards()
    assert torch.equal(U.t, U0)
    lr32 = np.float32(lr)
    g_pos, g_neg = lr32 * (np.float32(1.0) - np.float32(0.5)), lr32 * (np.float32(0.0) - np.float32(0.5))
    want = np.zeros((num_items, _stride(dim)), dtype=np.float32)
    u = U0.cpu().numpy()
    for p in np.flatnonzero(live):
        want[items[p]] = g_pos * u[users[p]]
        want[negs[p]] = g_neg * u[users[p]]
    V.check_guards()
    assert np.array_equal(V.t.cpu().numpy(), want)
    assert np.all(negs[live, 0] != items[live])                   # the rejection branch moved every first draw
    assert stats[1].item() == live.sum() * (1 + neg_rate)


def _shift_covering_steps(want=7):
    """Steps whose first draw for record 0 takes every value of s.z % 7."""
    steps, seen = [], set()
    for step in range(1, 400):
        _, _, z, _ = philox4x32(0, 0, 1, step, SEED & 0xFFFFFFFF, SEED >> 32)
        if int(z) % 7 not in seen:
            seen.add(int(z) % 7)
            steps.append(step)
        if len(seen) == want:
            return steps
    raise AssertionError("no step covers every shift")


@pytest.mark.parametrize("kernel", ["reg", "tma"])
def test_small_catalogue_negative_is_never_the_positive(dev, kernel):
    """One record per launch whose positive is its own raw draw, over catalogues of 2..9 items and steps covering
    every shift: exactly the positive row and the replayed negative row move, and they are different rows."""
    dim, lr = 13, 0.25
    gen = torch.Generator(device=dev).manual_seed(5)
    U = _table(1, dim, 0.5, gen, dev)
    u = U.t.cpu().numpy()[0]
    for num_items in range(2, 10):
        for step in _shift_covering_steps():
            _, raw = k5_negative([0], 1, [-1], num_items, step, SEED)
            neg, _ = k5_negative([0], 1, raw, num_items, step, SEED)
            assert neg[0] != raw[0]
            V = Guarded(num_items, _stride(dim), torch.float32, dev)
            V.t.zero_()
            a, b, c = _ids([0], raw, [1.0], "int32", dev)
            native.mf_sgd_fused(a, b, c, U.t.clone(), 1, native.local_table(V.t, dim), lr, err_mode=2, neg_rate=1,
                                num_items=num_items, seed=SEED, step=step, kernel=kernel)
            torch.cuda.synchronize()
            V.check_guards()
            got = V.t.cpu().numpy()
            moved = set(np.flatnonzero(got.any(1)).tolist())
            assert moved == {int(raw[0]), int(neg[0])}, (num_items, step, moved)
            lr32 = np.float32(lr)
            assert np.array_equal(got[raw[0]], lr32 * np.float32(0.5) * u)
            assert np.array_equal(got[neg[0]], lr32 * np.float32(-0.5) * u)


def test_one_item_catalogue_with_negatives_is_refused(dev):
    ids = torch.zeros(1, dtype=torch.int32, device=dev)
    U, V = torch.zeros(1, 4, device=dev), torch.zeros(1, 4, device=dev)
    with pytest.raises(ValueError, match="num_items >= 2"):
        native.mf_sgd_fused(ids, ids, torch.ones(1, device=dev), U, 1, native.local_table(V, 4), 0.1, neg_rate=1,
                            num_items=1)
    with pytest.raises(ValueError, match="num_items >= 2"):
        native.mf_bpr_fused(ids, ids, torch.ones(1, device=dev), U, native.local_table(V, 4), 0.1, num_items=1)


# ---- 5. hot rows ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel,dim", [("reg", 13), ("reg", 61), ("reg", 300), ("tma", 61), ("tma", 125)])
def test_hot_items_are_schedule_free(dev, kernel, dim):
    """Hot item h has users i = 0..dim-1 whose rows are c_i e_i: record i reads and pushes only coordinate i of the
    item row, so d_i = c_i V0[h, i] and the item row ends bitwise at V0 + sum g_i c_i e_i.  User coordinate k != i
    is g_i times V0[h, k], or times V0[h, k] + g_k c_k if record k pushed first: one of the two, bitwise."""
    hot, lr = 6, 0.05
    gen = torch.Generator(device=dev).manual_seed(dim)
    rng = np.random.default_rng(dim)
    n_items = 40
    V = _table(n_items, dim, 0.5, gen, dev)
    V0 = V.t.clone()
    hot_items = rng.permutation(n_items)[:hot]
    n = hot * dim
    U = Guarded(n, _stride(dim), torch.float32, dev)
    U.t.zero_()
    c = (rng.random(n) * 0.9 + 0.1).astype(np.float32)
    coord = np.tile(np.arange(dim), hot)
    U.t[torch.arange(n, device=dev), torch.from_numpy(coord).to(dev)] = torch.from_numpy(c).to(dev)
    item_of = np.repeat(hot_items, dim)
    r = rng.integers(1, 9, size=n).astype(np.float32) * np.float32(0.5)
    order = rng.permutation(n)                                  # interleave the hot items
    users = np.arange(n)
    a, b, cc = _ids(users[order], item_of[order], r[order], "int32", dev)
    stats = torch.zeros(2, device=dev)
    native.mf_sgd_fused(a, b, cc, U.t, 1, native.local_table(V.t, dim), lr, err_mode=1, stats=stats, kernel=kernel)
    torch.cuda.synchronize()
    v0 = V0.cpu().numpy()
    lr32 = np.float32(lr)
    vi = v0[item_of, coord]
    d = c * vi
    g = lr32 * (r - d)
    want_v = v0.copy()
    want_v[item_of, coord] = vi + g * c
    V.check_guards()
    U.check_guards()
    assert np.array_equal(V.t.cpu().numpy(), want_v)
    got_u = U.t.cpu().numpy()
    want_own = c + g * vi
    assert np.array_equal(got_u[users, coord], want_own)
    for k in range(hot):
        blk = slice(k * dim, (k + 1) * dim)
        h = hot_items[k]
        before = g[blk, None] * v0[h][None, :dim]
        after = g[blk, None] * want_v[h][None, :dim]
        off = ~np.eye(dim, dtype=bool)
        uk = got_u[blk, :dim]
        assert np.all((uk == before) | (uk == after) | ~off)
    assert not got_u[:, dim:].any()
    assert stats[1].item() == n


# ---- 6. voided records ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel,form,neg_rate", [("reg", "int32", 0), ("reg", "int64", 2), ("tma", "int32", 0),
                                                  ("tma", "int64", 0), ("tma", "int32", 2)])
def test_voided_records_are_skipped(dev, kernel, form, neg_rate):
    """user -1 with user_div 1 addresses the row before the user table, a guard row here."""
    if neg_rate == 0:
        _pointwise(dev, 61, form, 1, lpr=16 if kernel == "reg" else _tma_lpr(16), void_every=3, kernel=kernel)
        return
    dim, n, num_items = 29, 1500, 1 << 20
    gen = torch.Generator(device=dev).manual_seed(9)
    U = _table(n, dim, 0.5, gen, dev)
    V = _table(num_items, dim, 0.5, gen, dev)
    U0, V0 = U.t.clone(), V.t.clone()
    users = np.full(n, -1)
    stats = torch.zeros(2, device=dev)
    a, b, c = _ids(users, np.arange(n), np.ones(n, dtype=np.float32), form, dev)
    native.mf_sgd_fused(a, b, c, U.t, 1, native.local_table(V.t, dim), 0.1, neg_rate=neg_rate, num_items=num_items,
                        seed=SEED, step=STEP, stats=stats, kernel=kernel)
    torch.cuda.synchronize()
    U.check_guards()
    V.check_guards()
    assert torch.equal(U.t, U0) and torch.equal(V.t, V0)
    assert stats.tolist() == [0.0, 0.0]


# ---- 7. the fp64 tier ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [5, 13, 61, 125])
@pytest.mark.parametrize("shard,num_shards", [(0, 1), (2, 3)])
def test_init_rows_f64_matches_replay(dev, dim, shard, num_shards):
    rows, seed = 777, (3 << 40) + 17
    kd = (dim + 1) // 2 * 2
    t = Guarded(rows, kd, torch.float64, dev)
    native.init_rows_f64(t.t, dim, shard, num_shards, native.PART_HASH, rows, seed, -0.3, 0.7)
    torch.cuda.synchronize()
    t.check_guards()
    ids = np.arange(rows) * num_shards + shard
    assert np.array_equal(t.t.cpu().numpy(), init_rows_f64_ref(ids, dim, seed, -0.3, 0.7))


# dispatch_f64 (csrc/fps_mf_f64.cu): k doubles -> row of (k + 1) // 2 * 2 doubles -> nvec double2 -> LPR
F64_RUNGS = {5: 4, 13: 8, 29: 16, 61: 32, 125: 32, 255: 32}
F64_CASES = [(k, IDS[i % 3], (i + 1) % 3) for i, k in enumerate(F64_RUNGS)] + [(61, "int64", 2), (13, "packed64", 0)]


def _f64_step(dev, k, form, err_mode, n, rows, void_every=0, seed=0):
    gen = torch.Generator(device=dev).manual_seed(k + seed)
    rng = np.random.default_rng(k + seed)
    kd = (k + 1) // 2 * 2
    scale = k ** -0.25
    U = _table(rows, k, scale, gen, dev, torch.float64, kd)
    V = _table(rows, k, scale, gen, dev, torch.float64, kd)
    U0, V0 = U.t.clone(), V.t.clone()
    slots, items = rng.permutation(rows)[:n], rng.permutation(rows)[:n]
    r = _ratings(n, rng, err_mode)
    live = np.ones(n, dtype=bool)
    if void_every:
        live[::void_every] = False
    users = np.where(live, slots, -1)
    stats = torch.zeros(2, device=dev)
    a, b, c = _ids(users, items, r, form, dev)
    lr = 0.05
    native.mf_sgd_fused_f64(a, b, c, U.t, 1, native.local_table(V.t.view(torch.float32), 2 * k), lr,
                            err_mode=err_mode, stats=stats)
    torch.cuda.synchronize()
    s, it = slots[live], items[live]
    u0 = U0.cpu().numpy()[s, :k]
    v0 = V0.cpu().numpy()[it, :k]
    rr = r[live].astype(np.float64)
    d = (u0 * v0).sum(1)
    resid = rr - d
    e = {0: lambda: 1 / (1 + np.exp(-resid)), 1: lambda: resid, 2: lambda: rr - 1 / (1 + np.exp(-d))}[err_mode]()
    g = float(np.float32(lr)) * e                                # lr travels as fp32
    for got, want, what in ((U.t.cpu().numpy()[s, :k], u0 + g[:, None] * v0, "user rows"),
                            (V.t.cpu().numpy()[it, :k], v0 + g[:, None] * u0, "item rows")):
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max(), err_msg=what)
    _check_table(U, U0, k, s, "user table")
    _check_table(V, V0, k, it, "item table")
    st = stats.cpu().numpy()
    assert st[1] == live.sum()
    # per-warp fp64 sums, each rounded to fp32 once, then added in fp32 in any order
    sq = (resid * resid).sum()
    assert abs(st[0] - sq) <= 2 * (len(resid) + 2) * EPS * sq
    return U, V


@pytest.mark.parametrize("k,form,err_mode", F64_CASES)
def test_f64_rung_matches_replay(dev, k, form, err_mode):
    _f64_step(dev, k, form, err_mode, n=3000, rows=3600, void_every=0 if form == "packed64" else 7)


def test_f64_multi_round_grid(dev):
    """150000 records: more than the 132 * 8 CTAs * 64 lane-groups of the largest grid for k = 5."""
    _f64_step(dev, 5, "int64", 1, n=150_000, rows=160_000, void_every=11)


def test_f64_k_above_256_is_refused(dev):
    U = torch.zeros(4, 258, dtype=torch.float64, device=dev)
    V = torch.zeros(4, 258, dtype=torch.float64, device=dev)
    ids = torch.arange(4, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError, match="-1000"):
        native.mf_sgd_fused_f64(ids, ids, torch.ones(4, device=dev), U, 1,
                                native.local_table(V.view(torch.float32), 514), 0.1)
    assert not U.any() and not V.any()
