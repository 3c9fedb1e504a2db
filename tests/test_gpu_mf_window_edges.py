"""The step-window drain (``fps_mf_window_kernel``) called through ``native.mf_window_drain`` on guarded tables,
against the fp64 replay of ``tests/window_ref.py``: every lane bucket and kernel variant, grid-stride rounds on capped
grids, the window partition and singletons, voided records, empty micro-batches, id edges and a non-finite rating.

Every case checks that the guard rows, the padding columns and the rows outside the micro-batches are bitwise
unchanged; that every table element is within MARGIN times the replay's bound; that the update counts are exact and
the sums within bound, per micro-batch and in total; that the slot table is back to -1 everywhere; that the drain
applied as many windows as the replay's partition has; and, where each micro-batch's result does not depend on the
order its records run in, that the tables equal one ``mf_sgd_fused`` launch per micro-batch, bitwise.

A self-conflicting micro-batch is made schedule-free by a no-op twin: a second record on an item (or of a user)
already in the micro-batch whose other row is all zero and whose rating makes ``e`` exactly 0 (err_mode 1: r = 0;
err_mode 2: r = 1/2), so it pushes zeros and every pull sees the same rows in any order."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests.test_gpu_mf_pointwise_edges import Guarded, _check_table, _ratings, _table
from tests.window_ref import MARGIN, lanes, partition, replay, stats_bound

pytestmark = pytest.mark.gpu

TWIN_RATING = {1: 0.0, 2: 0.5}    # e = 0 when d = 0


def _stride(k):
    return (k + 3) // 4 * 4


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _stage(batches, forms, dev):
    """The staging area as DeviceOnlineMF._stage fills it: slot j at j * slot_bytes, packed64 records or int32
    users | int32 items | fp32 ratings."""
    slot_bytes = max(256, -(-max(len(b[0]) * 12 for b in batches) // 256) * 256)
    stage = torch.zeros(len(batches) * slot_bytes, dtype=torch.uint8, device=dev)
    for j, ((u, i, r), packed) in enumerate(zip(batches, forms)):
        n = len(u)
        if n == 0:
            continue
        slot = stage[j * slot_bytes:(j + 1) * slot_bytes]
        ut, it, rt = (torch.from_numpy(np.asarray(a)) for a in (u, i, r))
        if packed:
            slot[:8 * n].view(torch.int64).copy_(native.pack_ratings(ut, it, rt.float()).to(dev))
        else:
            ids = slot[:12 * n].view(torch.int32)
            ids[:n].copy_(ut.to(dev, torch.int32))
            ids[n:2 * n].copy_(it.to(dev, torch.int32))
            ids[2 * n:].view(torch.float32).copy_(rt.to(dev, torch.float32))
    return stage, slot_bytes


def _per_launch(U, V, batches, forms, k, lr, err_mode):
    """One mf_sgd_fused launch per micro-batch on clones of the tables."""
    dev = U.device
    for (u, i, r), packed in zip(batches, forms):
        if len(u) == 0:
            continue
        ut, it, rt = (torch.from_numpy(np.asarray(a)) for a in (u, i, r))
        if packed:
            args = (native.pack_ratings(ut, it, rt.float()).to(dev), None, None)
        else:
            args = (ut.to(dev, torch.int32), it.to(dev, torch.int32), rt.to(dev, torch.float32))
        native.mf_sgd_fused(*args, U, 1, native.local_table(V, k), lr, err_mode=err_mode, kernel="reg")
    torch.cuda.synchronize()


def _rows(t, ids, k):
    return t[torch.from_numpy(np.asarray(ids, dtype=np.int64)).to(t.device), :k].double().cpu().numpy()


def _compact(batches, keep=None):
    """(live user ids, item ids, batches indexing them); ``keep(items)`` selects the records replayed."""
    sel = []
    for u, i, r in batches:
        m = np.ones(len(u), dtype=bool) if keep is None else keep(i)
        sel.append((np.asarray(u)[m], np.asarray(i)[m], np.asarray(r, dtype=np.float64)[m]))
    uid = np.unique(np.concatenate([u[u >= 0] for u, _, _ in sel]))
    iid = np.unique(np.concatenate([i[u >= 0] for u, i, _ in sel]))
    out = [(np.where(u >= 0, np.searchsorted(uid, u), -1), np.searchsorted(iid, np.where(u >= 0, i, iid[0])), r)
           for u, i, r in sel]
    return uid, iid, out


def _worst(err, tol):
    """Largest |error| / bound (an error where the bound is 0 counts as infinite)."""
    return float(np.where(err > 0, err / np.maximum(tol, 1e-300), 0.0).max(initial=0.0))


def run(dev, U, V, k, batches, forms, lr, err_mode, *, variant=0, num_sms=None, sample=None, nan=False):
    """Drain ``batches`` = [(users, items, ratings)] numpy arrays into the guarded tables ``U``, ``V`` and check
    everything the module docstring lists.  ``sample``: replay only the chains of these items (exact: the chains of
    different items are independent).  Returns the partition's groups."""
    n = len(batches)
    U0, V0 = U.t.clone(), V.t.clone()
    stage, slot_bytes = _stage(batches, forms, dev)
    rows = V.t.shape[0]
    slots = torch.full((n, rows), -1, dtype=torch.int64, device=dev)
    user_bits = torch.full((-(-U.t.shape[0] // 32),), -1, dtype=torch.int32, device=dev)   # the drain clears it
    ctl = torch.full((2 * native.WINDOW_MAX,), 7, dtype=torch.int32, device=dev)
    stats = torch.zeros(2, device=dev)
    slot_stats = torch.full((n, 2), 99.0, device=dev)
    nan_flag = torch.zeros(1, dtype=torch.int32, device=dev)
    phase_ns = torch.zeros(4, dtype=torch.int64, device=dev)
    native.lib().fps_set_mf_window_variant(variant)
    try:
        native.mf_window_drain(stage, slot_bytes, [len(b[0]) for b in batches], [int(f) for f in forms], U.t, V.t,
                               lr, err_mode, slots, user_bits, ctl, stats, slot_stats, nan_flag, phase_ns=phase_ns,
                               num_sms=num_sms)
    finally:
        native.lib().fps_set_mf_window_variant(0)
    torch.cuda.synchronize()

    groups, _ = partition([(u, i) for u, i, _ in batches])
    assert phase_ns[2].item() == len(groups), "windows applied"
    assert (slots == -1).all(), "a slot-table entry left behind"
    assert nan_flag.item() == int(nan)

    keep = None if sample is None else (lambda i: np.isin(i, sample))
    uid, iid, cb = _compact(batches, keep)
    lpr = lanes(_stride(k))
    rep = replay(_rows(U0, uid, k), _rows(V0, iid, k), cb, lr, err_mode, lpr, groups=groups)
    worst = 0.0
    for t, ids, want, tol, what in ((U.t, uid, rep["U"], rep["tU"], "user rows"),
                                    (V.t, iid, rep["V"], rep["tV"], "item rows")):
        got = _rows(t, ids, k)
        fin = np.isfinite(want).all(1)
        assert np.array_equal(fin, np.isfinite(got).all(1)), f"{what}: non-finite rows differ"
        # a non-finite g turns the padding of the rows it touches into inf * 0 = NaN too, as per launch; those rows
        # are checked to be non-finite above and left out of the padding check below
        t[torch.from_numpy(ids[~fin]).to(dev)] = 0.0
        err = np.abs(got[fin] - want[fin])
        bad = err > MARGIN * tol[fin]
        assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} beyond the bound"
        worst = max(worst, _worst(err, tol[fin]))
    print(f"[window-edges] k={k} lpr={lpr} variant={variant} worst |error|/bound {worst:.3f}")

    all_u = np.concatenate([u[u >= 0] for u, _, _ in batches])
    all_i = np.concatenate([i[u >= 0] for u, i, _ in batches])
    _check_table(U, U0, k, all_u, "user table")
    _check_table(V, V0, k, all_i, "item table")

    cnt = rep["cnt"] if sample is None else np.array([float((u >= 0).sum()) for u, _, _ in batches])
    ss = slot_stats.double().cpu().numpy()
    assert np.array_equal(ss[:, 1], cnt), "per-micro-batch update counts"
    assert stats[1].item() == cnt.sum()
    if sample is None and not nan:
        assert (np.abs(ss[:, 0] - rep["sq"]) <= MARGIN * rep["tol_sq"]).all(), "per-micro-batch sums"
        assert abs(stats[0].item() - rep["sq"].sum()) <= MARGIN * stats_bound(rep)
    if not nan:
        Uc, Vc = U0.clone(), V0.clone()
        _per_launch(Uc, Vc, batches, forms, k, lr, err_mode)
        assert torch.equal(U.t, Uc) and torch.equal(V.t, Vc), "not the per-launch tables"
    return groups


def _window(rng, n_users, n_items, slots, per, hot, err_mode, users=None, hot_items=None):
    """``slots`` micro-batches of ``per`` records with distinct users across all of them; ``hot`` items (or
    ``hot_items``) in every micro-batch (chains of ``slots`` links), the rest of each micro-batch's items distinct
    and drawn at random."""
    users = rng.permutation(n_users)[:slots * per] if users is None else users
    hot_items = rng.permutation(n_items)[:hot] if hot_items is None else np.asarray(hot_items)
    hot = len(hot_items)
    cold = np.setdiff1d(np.arange(n_items), hot_items)
    out = []
    for j in range(slots):
        items = np.concatenate([hot_items, rng.permutation(cold)[:per - hot]])
        order = rng.permutation(per)
        out.append((users[j * per:(j + 1) * per].astype(np.int64), items[order].astype(np.int64),
                    _ratings(per, rng, err_mode)))
    return out


def _tables(dev, n_users, n_items, k, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    scale = k ** -0.25
    return _table(n_users, k, scale, gen, dev), _table(n_items, k, scale, gen, dev)


def _twin(U, V, batch, err_mode, on, rng):
    """``batch`` with a no-op twin appended: a record on one of its items by the last user, whose row is zeroed
    (on="item"), or by one of its users on the last item, whose row is zeroed (on="user").  Neither last row may
    be in use."""
    u, i, r = batch
    if on == "item":
        user, item = U.t.shape[0] - 1, int(i[u >= 0][rng.integers((u >= 0).sum())])
        U.t[user].zero_()
    else:
        user, item = int(u[u >= 0][rng.integers((u >= 0).sum())]), V.t.shape[0] - 1
        V.t[item].zero_()
    assert user not in u or on == "user"
    assert item not in i or on == "item"
    return np.append(u, user), np.append(i, item), np.append(r, np.float32(TWIN_RATING[err_mode]))


# ---- 1. every bucket x variant ---------------------------------------------------------------------------------

DIMS = [3, 7, 13, 29, 61, 125, 36, 52]     # LPR 1, 2, 4, 8, 16, 32; 36 and 52 leave the 16-lane bucket's lanes uneven
BUCKET_CASES = [(k, v, bool(c % 2), (c // 2) % 3)
                for c, (k, v) in enumerate((k, v) for k in DIMS for v in (0, 1, 2))]


def test_bucket_cases_cover_every_bucket_variant_form_and_rule():
    assert {lanes(_stride(k)) for k, _, _, _ in BUCKET_CASES} == {1, 2, 4, 8, 16, 32}
    assert {(k, v) for k, v, _, _ in BUCKET_CASES} == {(k, v) for k in DIMS for v in (0, 1, 2)}
    assert {(f, m) for _, _, f, m in BUCKET_CASES} == {(f, m) for f in (False, True) for m in range(3)}


@pytest.mark.parametrize("k,variant,packed,err_mode", BUCKET_CASES)
def test_bucket_and_variant_match_the_replay(dev, k, variant, packed, err_mode):
    rng = np.random.default_rng(10 * k + variant)
    U, V = _tables(dev, 6_000, 1_500, k, 10 * k + variant)
    batches = _window(rng, 6_000, 1_500, 8, 400, 64, err_mode)
    groups = run(dev, U, V, k, batches, [packed] * 8, 0.05, err_mode, variant=variant)
    assert groups == [(0, 8, False)]


# ---- 2. grid-stride rounds -------------------------------------------------------------------------------------
# The chain and singleton loops stride by lane-groups (grid * 256 / G), the build by threads, the bitmap clear by
# 32-user words.  One SM holds at most 8 CTAs of 256 threads, so at num_sms = 1: 8000 rows and 6500 singleton records
# take >= 3 rounds at G = 1 (and more at larger G), 6500 records per micro-batch >= 3 build rounds, and 200,003
# users >= 3 bitmap-clear rounds.
GRID_USERS, GRID_ITEMS, GRID_PER = 200_003, 8_000, 6_500


def _grid_batches(rng, U, V, err_mode):
    """Two windowed micro-batches, a singleton (an item twice, by a no-op twin) of GRID_PER + 1 records, and one
    more windowed micro-batch; users distinct across all four."""
    users = rng.permutation(GRID_USERS - 1)[:4 * GRID_PER]
    batches = _window(rng, GRID_USERS, GRID_ITEMS, 4, GRID_PER, 16, err_mode, users=users)
    batches[2] = _twin(U, V, batches[2], err_mode, "item", rng)
    return batches


@pytest.mark.parametrize("k", [3, 7, 13, 29, 61, 125])
def test_capped_grid_equals_the_default_grid(dev, k):
    assert 3 * 8 * 256 < min(GRID_ITEMS, GRID_PER) and 3 * 32 * 8 * 256 < GRID_USERS
    res = []
    for num_sms in (None, 1):
        rng = np.random.default_rng(k)
        U, V = _tables(dev, GRID_USERS, GRID_ITEMS, k, k)
        batches = _grid_batches(rng, U, V, 1)
        groups = run(dev, U, V, k, batches, [False, True, False, True], 0.05, 1, num_sms=num_sms)
        assert groups == [(0, 2, False), (2, 3, True), (3, 4, False)]
        res.append((U.t, V.t))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


@pytest.mark.parametrize("sizes", [[838_861] * 5, [1_000_000] * 2], ids=["bench", "full"])
def test_bench_shape(dev, sizes):
    """bench.py's defaults: k = 64, 1M items, 10M users, packed64, a step of five micro-batches of 838,861 records
    (distinct users in the step, distinct items in a micro-batch); and micro-batches of exactly as many records as
    the table has rows.  Checked bitwise against the per-launch kernel and against the replay on 4,096 items."""
    k, n_users, n_items = 64, 10_000_000, 1_000_000
    g = torch.Generator().manual_seed(1000)
    users = torch.randperm(n_users, generator=g)[:sum(sizes)].split(sizes)
    batches = [(u.numpy().astype(np.int64), torch.randperm(n_items, generator=g)[:len(u)].numpy().astype(np.int64),
                torch.rand(len(u), generator=g).half().float().numpy()) for u in users]
    U, V = _tables(dev, n_users, n_items, k, 1234)
    sample = np.random.default_rng(1).permutation(n_items)[:4_096]
    groups = run(dev, U, V, k, batches, [True] * len(sizes), 0.01, 0, sample=sample)
    assert groups == [(0, len(sizes), False)]


# ---- 3. partition and singletons --------------------------------------------------------------------------------

def test_users_repeated_across_micro_batches_split_where_the_replay_says(dev):
    rng = np.random.default_rng(3)
    k = 29
    U, V = _tables(dev, 6_000, 1_500, k, 3)
    batches = _window(rng, 6_000, 1_500, 8, 300, 32, 1)
    for j, src in ((2, 0), (3, 2), (6, 4)):       # repeat one user of an earlier micro-batch
        batches[j][0][5] = batches[src][0][7]
    groups = run(dev, U, V, k, batches, [False, True] * 4, 0.05, 1)
    assert groups == [(0, 2, False), (2, 3, False), (3, 6, False), (6, 8, False)]


@pytest.mark.parametrize("where", [0, 4, 7])
@pytest.mark.parametrize("on", ["item", "user"])
def test_self_conflicting_micro_batch_is_a_singleton(dev, where, on):
    rng = np.random.default_rng(10 * where + (on == "user"))
    k, err_mode = 13, 2 if on == "user" else 1
    U, V = _tables(dev, 6_000, 1_500, k, where)
    batches = _window(rng, 5_999, 1_499, 8, 300, 32, err_mode)
    batches[where] = _twin(U, V, batches[where], err_mode, on, rng)
    groups = run(dev, U, V, k, batches, [bool(j % 2) for j in range(8)], 0.05, err_mode)
    want = ([(0, where, False)] if where else []) + [(where, where + 1, True)]
    assert groups == want + ([(where + 1, 8, False)] if where < 7 else [])


def test_worst_schedule_of_fifteen_attempts(dev):
    """One user in all eight micro-batches: eight windows of one, 15 scatter attempts (ctl has 16 flags)."""
    rng = np.random.default_rng(15)
    k = 61
    U, V = _tables(dev, 6_000, 1_500, k, 15)
    batches = _window(rng, 6_000, 1_500, 8, 200, 16, 0)
    for j in range(1, 8):
        batches[j][0][3] = batches[0][0][0]
    groups = run(dev, U, V, k, batches, [True] * 8, 0.05, 0)
    assert groups == [(j, j + 1, False) for j in range(8)]
    assert partition([(u, i) for u, i, _ in batches])[1] == 15


@pytest.mark.parametrize("k", [13, 61])
@pytest.mark.parametrize("mirror", [False, True], ids=["hot-item", "hot-user"])
def test_schedule_free_singletons(dev, k, mirror):
    """Hot item h of users c_i e_i (i < k): record i reads and pushes only coordinate i of h's row, so the item
    row ends bitwise at V0 + sum g_i c_i e_i, and user i's coordinate j != i is g_i times h's coordinate j before or
    after record j pushed.  The mirror: hot user of items c_i e_i, with the roles swapped."""
    lr = 0.05
    rng = np.random.default_rng(k + mirror)
    hot_rows, n_other = 6, 40
    n = hot_rows * k
    gen = torch.Generator(device=dev).manual_seed(k)
    Hot = _table(n_other, k, 0.5, gen, dev)                     # the dense side
    Cold = Guarded(n, _stride(k), torch.float32, dev)           # rows c_i e_i
    Cold.t.zero_()
    c = (rng.random(n) * 0.9 + 0.1).astype(np.float32)
    coord = np.tile(np.arange(k), hot_rows)
    Cold.t[torch.arange(n, device=dev), torch.from_numpy(coord).to(dev)] = torch.from_numpy(c).to(dev)
    hot_of = np.repeat(rng.permutation(n_other)[:hot_rows], k)
    r = (rng.integers(1, 9, size=n) * 0.5).astype(np.float32)
    order = rng.permutation(n)
    cold_ids = np.arange(n)
    users, items = (hot_of, cold_ids) if mirror else (cold_ids, hot_of)
    U, V = (Hot, Cold) if mirror else (Cold, Hot)
    H0 = Hot.t.clone()
    stats = torch.zeros(2, device=dev)
    ss = torch.zeros(1, 2, device=dev)
    stage, sb = _stage([(users[order], items[order], r[order])], [False], dev)
    slots = torch.full((1, V.t.shape[0]), -1, dtype=torch.int64, device=dev)
    phase = torch.zeros(4, dtype=torch.int64, device=dev)
    native.mf_window_drain(stage, sb, [n], [0], U.t, V.t, lr, 1, slots,
                           torch.zeros(-(-U.t.shape[0] // 32), dtype=torch.int32, device=dev),
                           torch.zeros(16, dtype=torch.int32, device=dev), stats, ss,
                           torch.zeros(1, dtype=torch.int32, device=dev), phase_ns=phase)
    torch.cuda.synchronize()
    assert phase[2].item() == 1 and (slots == -1).all()
    Hot.check_guards()
    Cold.check_guards()
    h0 = H0.cpu().numpy()
    hi = h0[hot_of, coord]
    g = np.float32(lr) * (r - c * hi)
    want_h = h0.copy()
    want_h[hot_of, coord] = hi + g * c
    assert np.array_equal(Hot.t.cpu().numpy(), want_h)
    got = Cold.t.cpu().numpy()
    assert np.array_equal(got[cold_ids, coord], c + g * hi)
    for b in range(hot_rows):
        blk = slice(b * k, (b + 1) * k)
        h = hot_of[b * k]
        off = ~np.eye(k, dtype=bool)
        ok = (got[blk, :k] == g[blk, None] * h0[h][None, :k]) | (got[blk, :k] == g[blk, None] * want_h[h][None, :k])
        assert np.all(ok | ~off)
    assert not got[:, k:].any()
    assert stats[1].item() == n and ss[0, 1].item() == n


# ---- 4. voids and empties ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [7, 61])
def test_voided_records_are_skipped_in_windows_and_singletons(dev, k):
    """int32 user -1 records (the row before the user table is a guard row) in windowed micro-batches and in a
    singleton; some voids repeat an item of their micro-batch, which is no conflict."""
    rng = np.random.default_rng(k)
    U, V = _tables(dev, 6_000, 1_500, k, k)
    batches = _window(rng, 5_999, 1_500, 6, 300, 32, 1)
    for u, i, _ in batches:
        u[::5] = -1
        i[::10] = i[1::10]                            # a void on a live record's item
    batches[3] = _twin(U, V, batches[3], 1, "item", rng)
    groups = run(dev, U, V, k, batches, [False] * 6, 0.05, 1)
    assert groups == [(0, 3, False), (3, 4, True), (4, 6, False)]


@pytest.mark.parametrize("empty", [[0], [3], [7], [0, 4, 7]], ids=["first", "middle", "last", "three"])
def test_empty_micro_batches(dev, empty):
    rng = np.random.default_rng(len(empty) + empty[0])
    k = 29
    U, V = _tables(dev, 6_000, 1_500, k, 5)
    batches = _window(rng, 6_000, 1_500, 8, 300, 32, 2)
    for j in empty:
        batches[j] = tuple(a[:0] for a in batches[j])
    groups = run(dev, U, V, k, batches, [bool(j % 2) for j in range(8)], 0.05, 2)
    assert groups == [(0, 8, False)]


@pytest.mark.parametrize("n_slots", [1, 8])
def test_window_of_one_and_eight_slots(dev, n_slots):
    rng = np.random.default_rng(n_slots)
    k = 125
    U, V = _tables(dev, 6_000, 1_500, k, n_slots)
    batches = _window(rng, 6_000, 1_500, n_slots, 700, 100, 0)
    assert run(dev, U, V, k, batches, [False] * n_slots, 0.05, 0) == [(0, n_slots, False)]


# ---- 5. id edges -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("packed", [False, True])
def test_first_and_last_rows(dev, packed):
    """Items 0 and rows - 1 (the first and last slot-table columns) and users 0 and n_users - 1 (the bitmap's last
    word, n_users % 32 != 0) in chains of eight."""
    rng = np.random.default_rng(21)
    k, n_users, n_items = 13, 6_001, 1_499
    assert n_users % 32
    U, V = _tables(dev, n_users, n_items, k, 21)
    users = np.concatenate([[0, n_users - 1], rng.permutation(np.arange(1, n_users - 1))[:8 * 200 - 2]])
    batches = _window(rng, n_users, n_items, 8, 200, 0, 1, users=users, hot_items=[0, n_items - 1])
    assert batches[0][0][0] == 0 and batches[0][0][1] == n_users - 1
    run(dev, U, V, k, batches, [packed] * 8, 0.05, 1)


def test_packed64_high_id_bits(dev):
    """users >= 2^25 and items >= 2^21: the top bits of the packed64 user:26 | item:22 decode, at k = 4."""
    rng = np.random.default_rng(25)
    k, n_users, n_items = 4, (1 << 25) + 37, (1 << 21) + 300
    U, V = _tables(dev, n_users, n_items, k, 25)
    per = 500
    users = np.concatenate([n_users - 1 - np.arange(8 * per // 2), rng.permutation(1 << 24)[:8 * per // 2]])
    users = rng.permutation(users)
    hi = n_items - 1 - np.arange(per // 2)
    batches = []
    for j in range(8):
        items = np.concatenate([hi, rng.permutation(1 << 20)[:per // 2]])
        batches.append((users[j * per:(j + 1) * per].astype(np.int64), rng.permutation(items).astype(np.int64),
                        _ratings(per, rng, 0)))
    assert users.max() >= 1 << 25 and hi.min() >= 1 << 21
    run(dev, U, V, k, batches, [True] * 8, 0.05, 0)


# ---- 6. a non-finite rating ------------------------------------------------------------------------------------

def test_inf_rating_mid_chain_sets_the_flag_and_spares_other_items(dev):
    rng = np.random.default_rng(6)
    k = 61
    U, V = _tables(dev, 6_000, 1_500, k, 6)
    batches = _window(rng, 6_000, 1_500, 8, 300, 32, 1)
    hot = sorted(set.intersection(*(set(i.tolist()) for _, i, _ in batches)))[0]     # in every micro-batch
    batches[4][2][batches[4][1] == hot] = np.inf
    run(dev, U, V, k, batches, [False] * 8, 0.05, 1, nan=True)
