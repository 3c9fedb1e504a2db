"""The step-window replay of ``tests/window_ref.py`` on the CPU: the drain's window partition on hand-built schedules,
a chain of length 1 equal to the pointwise replay, and a brute-force fp32 evaluation of the drain's arithmetic on
random chains within the replay's reported bound."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests.pointwise_ref import replay as pointwise_replay
from tests.window_ref import MARGIN, lanes, partition, replay, stats_bound

F = np.float32


def _mb(users, items=None):
    users = np.asarray(users, dtype=np.int64)
    items = np.arange(len(users)) if items is None else np.asarray(items, dtype=np.int64)
    return users, items


# ---- partition -----------------------------------------------------------------------------------------------

def test_lane_buckets():
    assert [lanes(s) for s in (4, 8, 12, 16, 20, 32, 36, 64, 68, 128)] == [1, 2, 4, 4, 8, 8, 16, 16, 32, 32]
    with pytest.raises(ValueError):
        lanes(132)


def test_conflict_free_schedule_is_one_window():
    groups, attempts = partition([_mb([4 * j, 4 * j + 1], [0, 1]) for j in range(8)])
    assert groups == [(0, 8, False)] and attempts == 8


def test_a_user_repeated_across_micro_batches_splits_the_window():
    groups, attempts = partition([_mb([0, 1]), _mb([2, 3]), _mb([4, 1]), _mb([5, 6]), _mb([0, 7])])
    assert groups == [(0, 2, False), (2, 5, False)]
    assert attempts == 3 + 3      # the clashing micro-batch is scattered again to open the next window


@pytest.mark.parametrize("where", [0, 3, 7])
@pytest.mark.parametrize("twice", ["item", "user"])
def test_a_self_conflicting_micro_batch_is_a_singleton(where, twice):
    batches = [_mb([3 * j, 3 * j + 1, 3 * j + 2]) for j in range(8)]
    u, i = batches[where]
    batches[where] = (u, np.array([5, 6, 5])) if twice == "item" else (np.array([u[0], u[1], u[0]]), i)
    groups, attempts = partition(batches)
    want = ([(0, where, False)] if where else []) + [(where, where + 1, True)]
    if where < 7:
        want.append((where + 1, 8, False))
    assert groups == want
    assert attempts == (where + 1 if where else 0) + 1 + (7 - where)


def test_voids_neither_conflict_nor_join():
    # void records repeat an item, a user (-1) and an earlier micro-batch's items: none of it is a conflict
    batches = [_mb([0, -1, -1], [7, 7, 8]), _mb([-1, 1], [7, 7]), _mb([-1, -1], [1, 1])]
    assert partition(batches) == ([(0, 3, False)], 3)


def test_empty_micro_batches_join_any_window():
    e = _mb([])
    assert partition([e, _mb([0]), e, _mb([1]), e]) == ([(0, 5, False)], 5)
    assert partition([e]) == ([(0, 1, False)], 1)
    assert partition([_mb([0]), e, _mb([0]), e]) == ([(0, 2, False), (2, 4, False)], 5)


def test_worst_schedule_takes_fifteen_attempts():
    """One user in every micro-batch: eight windows of one, each but the last scattered twice.  ``ctl`` holds
    2 * WIN_MAX = 16 conflict flags."""
    groups, attempts = partition([_mb([0], [j]) for j in range(8)])
    assert groups == [(j, j + 1, False) for j in range(8)]
    assert attempts == 15 < 2 * native.WINDOW_MAX
    singles, attempts = partition([_mb([j, j], [0, 1]) for j in range(8)])
    assert all(s for _, _, s in singles) and attempts == 8


# ---- replay --------------------------------------------------------------------------------------------------

def _rows(rng, shape, scale=0.5):
    return ((rng.random(shape) * 2 - 1) * scale).astype(F).astype(np.float64)



@pytest.mark.parametrize("err_mode", [0, 1, 2])
@pytest.mark.parametrize("k,stride", [(3, 4), (7, 8), (13, 16), (29, 32), (61, 64), (125, 128)])
def test_chain_of_one_is_the_pointwise_replay(err_mode, k, stride):
    rng = np.random.default_rng(k + 10 * err_mode)
    n = 50
    u0, v0 = _rows(rng, (n, k)), _rows(rng, (n, k))
    r = rng.integers(0, 2, size=n).astype(np.float64)
    items = rng.permutation(n)
    lpr = lanes(stride)
    rep = replay(u0, v0, [(np.arange(n), items, r)], 0.05, err_mode, lpr)
    one = pointwise_replay(u0, v0[items], r, 0.05, err_mode, lpr)
    assert np.array_equal(rep["U"], one.u) and np.array_equal(rep["tU"], one.tol_u)
    assert np.array_equal(rep["V"][items], one.v) and np.array_equal(rep["tV"][items], one.tol_v)
    assert rep["sq"][0] == (one.resid * one.resid).sum() and rep["cnt"][0] == n
    assert rep["groups"] == [(0, 1, False)] and rep["attempts"] == 1


# ---- the drain's fp32 arithmetic, evaluated one rounding at a time ---------------------------------------------

def _fma(a, b, c):
    return F(np.float64(a) * np.float64(b) + np.float64(c))


def _dot32(u, v, G, VPL):
    """win_dot: one fps_mf_dot4 per float4, lane l holding float4s l, l + G, ...; the in-lane tree, then the
    xor-shuffle tree over the G lanes."""
    lanes_ = []
    for lane in range(G):
        d = []
        for kk in range(VPL):
            x, y = u[4 * (lane + kk * G):][:4], v[4 * (lane + kk * G):][:4]
            t = F(x[1] * y[1])
            t = _fma(x[3], y[3], _fma(x[2], y[2], _fma(x[0], y[0], t)))
            d.append(F(F(0) + t))
        h = VPL // 2
        while h:
            d = [F(d[kk] + d[kk + h]) for kk in range(h)] + d[h:]
            h //= 2
        lanes_.append(d[0])
    o = G // 2
    while o:
        lanes_ = [F(lanes_[lane] + lanes_[lane ^ o]) for lane in range(G)]
        o //= 2
    return lanes_[0]


def _sig32(x):
    return F(F(1) / F(F(1) + F(np.exp(F(-x), dtype=F))))


def _chain32(v, users, r, lr, err_mode, G, VPL):
    """One item's chain in fp32: returns the item row and each link's new user row and residual."""
    lr32 = F(lr)
    out, res = [], []
    for u, rr in zip(users, r):
        d = _dot32(u, v, G, VPL)
        resid = F(rr - d)
        e = _sig32(resid) if err_mode == 0 else resid if err_mode == 1 else F(rr - _sig32(d))
        g = F(lr32 * e)
        u, v = (u + F(g) * v).astype(F), (v + F(g) * u).astype(F)
        out.append(u)
        res.append(resid)
    return v, out, res


# (k, stride, G, VPL): every bucket at one float4 per lane, and the default 16-lane geometry (4 float4 on 4 lanes)
GEOMS = [(3, 4, 1, 1), (7, 8, 2, 1), (13, 16, 4, 1), (29, 32, 8, 1), (52, 64, 4, 4), (61, 64, 16, 1),
         (125, 128, 32, 1)]


@pytest.mark.parametrize("err_mode", [0, 1, 2])
@pytest.mark.parametrize("k,stride,G,VPL", GEOMS)
def test_fp32_chains_stay_within_the_bound(err_mode, k, stride, G, VPL):
    """8 micro-batches over 6 items, each item once per micro-batch with a user of its own: chains of 8 links."""
    rng = np.random.default_rng(100 * k + err_mode)
    n_items, links, lr = 6, 8, 0.1
    scale = k ** -0.25
    V0 = _rows(rng, (n_items, k), scale)
    U0 = _rows(rng, (n_items * links, k), scale)
    r = (rng.integers(1, 9, size=(links, n_items)) * 0.5 if err_mode == 1
         else rng.integers(0, 2, size=(links, n_items))).astype(np.float64)
    batches = [(np.arange(n_items) + j * n_items, rng.permutation(n_items), r[j]) for j in range(links)]
    rep = replay(U0, V0, batches, lr, err_mode, G * VPL)
    assert rep["groups"] == [(0, links, False)]
    pad = np.zeros(stride, dtype=F)
    sq = np.zeros(links)
    for item in range(n_items):
        at = [int(np.flatnonzero(b[1] == item)[0]) for b in batches]
        users = [np.concatenate([U0[batches[j][0][a]].astype(F), pad])[:stride] for j, a in enumerate(at)]
        v0 = np.concatenate([V0[item].astype(F), pad])[:stride]
        v, us, res = _chain32(v0, users, [batches[j][2][a] for j, a in enumerate(at)], lr, err_mode, G, VPL)
        assert not v[k:].any()
        bad = np.abs(v[:k] - rep["V"][item]) > MARGIN * rep["tV"][item]
        assert not bad.any(), (item, np.abs(v[:k] - rep["V"][item]).max(), rep["tV"][item].max())
        for j, (a, u) in enumerate(zip(at, us)):
            row = batches[j][0][a]
            assert not (np.abs(u[:k] - rep["U"][row]) > MARGIN * rep["tU"][row]).any(), (item, j)
            sq[j] += float(res[j]) ** 2
    assert (np.abs(sq - rep["sq"]) <= MARGIN * rep["tol_sq"]).all()
    assert (rep["cnt"] == n_items).all()
    assert abs(sq.sum() - rep["sq"].sum()) <= MARGIN * stats_bound(rep)


def test_chain_bound_grows_with_every_link():
    """A chain's item-row bound after 8 links exceeds 8 independent single links' (the later dots see the
    earlier links' error), and applying the same links in reverse order gives another item row."""
    rng = np.random.default_rng(7)
    k, links = 61, 8
    V0, U0 = _rows(rng, (1, k)), _rows(rng, (links, k))
    r = rng.integers(1, 9, size=links) * 0.5
    batches = [(np.array([j]), np.array([0]), r[j:j + 1]) for j in range(links)]
    chain = replay(U0, V0, batches, 0.1, 1, 16)
    single = [replay(U0[j:j + 1], V0, [(np.array([0]), np.array([0]), r[j:j + 1])], 0.1, 1, 16) for j in range(links)]
    assert chain["tV"].sum() > 2 * max(s["tV"].sum() for s in single)
    rev = replay(U0, V0, batches[::-1], 0.1, 1, 16)
    assert np.abs(rev["V"] - chain["V"]).max() > 10 * MARGIN * chain["tV"].max()


def test_singleton_reductions_are_jacobi_within_their_race_bound():
    """A micro-batch with one hot item: every record pulls the rows as they were, and the item row is the sum of
    every record's push; the bound covers the other records' pushes a pull may already see."""
    rng = np.random.default_rng(8)
    k, n = 13, 6
    U0, V0 = _rows(rng, (n, k)), _rows(rng, (1, k))
    r = rng.integers(1, 9, size=n) * 0.5
    rep = replay(U0, V0, [(np.arange(n), np.zeros(n, dtype=np.int64), r)], 0.05, 1, 4)
    assert rep["groups"] == [(0, 1, True)]
    g = np.float32(0.05) * (r - U0 @ V0[0])
    assert np.allclose(rep["V"][0], V0[0] + (g[:, None] * U0).sum(0), rtol=0, atol=1e-15)
    # one record after another (each pull sees every earlier push) stays within the bound
    v, u = V0[0].copy(), U0.copy()
    for i in range(n):
        gi = np.float32(0.05) * (r[i] - u[i] @ v)
        u[i], v = u[i] + gi * v, v + gi * u[i]
    assert (np.abs(v - rep["V"][0]) <= MARGIN * rep["tV"][0]).all()
    assert (np.abs(u - rep["U"]) <= MARGIN * rep["tU"]).all()


def test_a_voided_record_is_neither_applied_nor_counted():
    rng = np.random.default_rng(9)
    U0, V0 = _rows(rng, (4, 7)), _rows(rng, (4, 7))
    users = np.array([0, -1, 2, -1])
    rep = replay(U0, V0, [(users, np.arange(4), np.ones(4))], 0.05, 1, 2)
    assert rep["cnt"][0] == 2
    assert np.array_equal(rep["V"][[1, 3]], V0[[1, 3]]) and not rep["tV"][[1, 3]].any()
    assert np.array_equal(rep["U"][[1, 3]], U0[[1, 3]])


def test_num_sms_below_one_is_refused():
    t = torch.zeros(4)
    with pytest.raises(ValueError, match="num_sms"):
        native.mf_window_drain(t, 16, [1], [0], t, t, 0.1, 0, t, t, t, t, t, t, num_sms=0)
