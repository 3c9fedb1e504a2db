"""The fp64 replays of ``tests/pairwise_ref.py`` and ``tests/pointwise_ref.py`` on the CPU: equal to the project's
numpy references (``models/mf/common.py``: ``bpr_delta``, ``warp_delta``, ``rowwise_adagrad``) on random small cases,
and within their own reported bound of a brute-force fp32 evaluation of the same expressions."""
import math

import numpy as np
import pytest

import fps_b200  # noqa: F401
from fps_b200.models.mf.common import bpr_delta, rowwise_adagrad, warp_delta
from tests.pairwise_ref import MARGIN, bpr_replay, f32, geometry, sampled_candidates, warp_replay
from tests.philox_ref import k5_negative
from tests.pointwise_ref import replay as pointwise_replay

F = np.float32


def _rows(rng, shape, scale=0.5):
    return ((rng.random(shape) * 2 - 1) * scale).astype(F).astype(np.float64)


def _case(seed, P=40, T=4, k=13, repeats=False):
    rng = np.random.default_rng(seed)
    u, vi = _rows(rng, (P, k)), _rows(rng, (P, k))
    negs = np.stack([rng.permutation(50)[:T] for _ in range(P)])
    negs[rng.random((P, T)) < 0.2] = -1
    if repeats:
        negs[:, T - 1] = negs[:, 0]
    table = _rows(rng, (50, k))
    vj = np.where(negs[..., None] >= 0, table[np.maximum(negs, 0)], 0.0)
    return rng, u, vi, vj, negs


def _close(a, b, what):
    np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-13, err_msg=what)


def _within(got, want, tol, what):
    bad = np.abs(np.asarray(got, dtype=np.float64) - want) > MARGIN * tol
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} beyond the bound"


def _sig32(x):
    return F(1) / (F(1) + np.exp(F(-x), dtype=F))


# ---- BPR -------------------------------------------------------------------------------------------------------

def _bpr_numpy(u, vi, vj, negs, lr, reg, ada=None):
    """bpr_delta per triple, summed for u and v_i; a repeated negative reads its row with the earlier push applied;
    AdaGrad by rowwise_adagrad on the summed (rate 1) deltas and on each negative's."""
    P, T, k = vj.shape
    U, VI, VJ = u.copy(), vi.copy(), vj.copy()
    Gu = Gi = Gj = None
    if ada is not None:
        Gu, Gi, Gj = (np.asarray(a, dtype=np.float64).copy() for a in ada[:3])
    for p in range(P):
        rows, acc = {}, {}
        du, di = np.zeros(k), np.zeros(k)
        n = 0
        for t in range(T):
            j = negs[p, t]
            if j < 0:
                continue
            n += 1
            r = rows.get(j, vj[p, t])
            a, b, c, _ = bpr_delta(u[p], vi[p], r, 1.0 if ada is not None else lr, reg)
            du += a
            di += b
            if ada is None:
                new = r + c
            else:
                G = acc.get(j, Gj[p, t])
                new, s = rowwise_adagrad(r, G, c, lr, k)
                acc[j] = G + s
                Gj[p, t] = G + s
            rows[j] = new
            VJ[p, t] = new
        if n:
            if ada is None:
                U[p], VI[p] = u[p] + du, vi[p] + di
            else:
                U[p], s = rowwise_adagrad(u[p], Gu[p], du, lr, k)
                Gu[p] += s
                VI[p], s = rowwise_adagrad(vi[p], Gi[p], di, lr, k)
                Gi[p] += s
    return U, VI, VJ, Gu, Gi, Gj


def _bpr_fp32(u, vi, vj, negs, lr, reg, ada=None):
    """The kernel's expressions in fp32, one positive at a time."""
    P, T, k = vj.shape
    lr, reg = F(lr), F(reg)
    decay = reg if ada is not None else lr * reg
    U, VI, VJ = u.astype(F), vi.astype(F), vj.astype(F).copy()
    Gu = Gi = Gj = None
    if ada is not None:
        Gu, Gi, Gj = (np.asarray(a, dtype=F).copy() for a in ada[:3])

    def step(G, d):
        s = F((d * d).sum(dtype=F) * (F(1) / F(k)))
        return lr / (np.sqrt(F(G + s)) + F(1e-8)), s

    for p in range(P):
        up, vp = u[p].astype(F), vi[p].astype(F)
        rows, acc = {}, {}
        du, gs, n = np.zeros(k, F), F(0), 0
        for t in range(T):
            j = negs[p, t]
            if j < 0:
                continue
            r = rows.get(j, vj[p, t].astype(F))
            diff = vp - r
            x = (up * diff).sum(dtype=F)
            g = F(1) / (F(1) + np.exp(x, dtype=F))
            g = g if ada is not None else lr * g
            d = -g * up - decay * r
            if ada is None:
                new = r + d
            else:
                G = acc.get(j, Gj[p, t])
                st, s = step(G, d)
                new = r + st * d
                acc[j] = Gj[p, t] = F(G + s)
            rows[j] = VJ[p, t] = new
            du, gs, n = du + g * diff, gs + g, n + 1
        if n:
            dec = decay * F(n)
            d_u, d_i = du - dec * up, gs * up - dec * vp
            if ada is None:
                U[p], VI[p] = up + d_u, vp + d_i
            else:
                st, s = step(Gu[p], d_u)
                U[p], Gu[p] = up + st * d_u, Gu[p] + s
                st, s = step(Gi[p], d_i)
                VI[p], Gi[p] = vp + st * d_i, Gi[p] + s
    return U, VI, VJ, Gu, Gi, Gj


@pytest.mark.parametrize("seed,k,stride,reg,repeats", [(0, 3, 4, 0.0, False), (1, 13, 16, 0.01, False),
                                                        (2, 61, 64, 0.01, True), (3, 300, 300, 0.0, True)])
@pytest.mark.parametrize("ada", [False, True])
def test_bpr_replay_matches_numpy_reference_and_fp32(seed, k, stride, reg, repeats, ada):
    rng, u, vi, vj, negs = _case(seed, k=k, repeats=repeats)
    lr = f32(0.05)
    acc = None
    if ada:
        P, T = negs.shape
        acc = (rng.random(P) * 0.5, np.zeros(P), rng.random((P, T)) * (rng.random((P, T)) < 0.5), k)
        acc = tuple(a.astype(F).astype(np.float64) if isinstance(a, np.ndarray) else a for a in acc)
    res = bpr_replay(u, vi, vj, negs, lr, reg, stride, acc)
    U, VI, VJ, Gu, Gi, Gj = _bpr_numpy(u, vi, vj, negs, lr, f32(reg), acc)
    live = negs >= 0
    _close(res.u, U, "u")
    _close(res.vi, VI, "v_i")
    _close(res.vj[live], VJ[live], "v_j")
    if ada:
        _close(res.Gu, Gu, "G_u")
        _close(res.Gi, Gi, "G_i")
        _close(res.Gj[live], Gj[live], "G_j")
        assert res.smooth
    loss = sum(bpr_delta(u[p], vi[p], vj[p, t], lr, 0.0)[3] for p, t in zip(*np.nonzero(live)) if not repeats)
    if not repeats:
        assert math.isclose(res.loss, loss, rel_tol=1e-12)
    assert res.count == live.sum()
    u32, vi32, vj32, Gu32, Gi32, Gj32 = _bpr_fp32(u, vi, vj, negs, lr, reg, acc)
    _within(u32, res.u, res.tol_u, "fp32 u")
    _within(vi32, res.vi, res.tol_vi, "fp32 v_i")
    _within(vj32[live], res.vj[live], res.tol_vj[live], "fp32 v_j")
    if ada:
        _within(Gu32, res.Gu, res.tol_Gu, "fp32 G_u")
        _within(Gj32[live], res.Gj[live], res.tol_Gj[live], "fp32 G_j")


def test_bpr_replay_sums_the_live_negatives_and_decays_by_n_live():
    """Two live negatives and a void: u and v_i move by the two triples' deltas, decayed by lr reg 2."""
    rng, u, vi, vj, negs = _case(9, P=1, T=3, k=7)
    negs[:] = [[4, -1, 9]]
    res = bpr_replay(u, vi, vj, negs, 0.25, 0.125, 8)
    d0 = bpr_delta(u[0], vi[0], vj[0, 0], 0.25, 0.125)
    d2 = bpr_delta(u[0], vi[0], vj[0, 2], 0.25, 0.125)
    _close(res.u[0], u[0] + d0[0] + d2[0], "u")
    assert res.n_live[0] == 2


# ---- WARP ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed,k,stride,margin,reg", [(0, 3, 4, 1.0, 0.0), (1, 13, 16, 0.1, 0.01),
                                                       (2, 125, 128, -0.05, 0.01), (3, 61, 64, 0.3, 0.0)])
def test_warp_replay_matches_numpy_reference_and_fp32(seed, k, stride, margin, reg):
    rng, u, vi, vj, negs = _case(seed, P=60, T=6, k=k)
    live = negs >= 0
    lr, rank_items = f32(0.05), 37
    res = warp_replay(u, vi, vj, live, lr, reg, margin, rank_items, stride)
    lr32, reg32, m32 = F(lr), F(reg), F(margin)
    for p in range(len(u)):
        du, dvi, ts, dvj, n, L, loss = warp_delta(u[p], vi[p], [vj[p, t] if live[p, t] else None for t in range(6)],
                                                  f32(margin), lr, f32(reg), rank_items)
        assert res.n[p] == n and res.hit[p] == (ts is not None)
        if ts is None:
            _close(res.u[p], u[p], "untouched u")
            continue
        assert res.tstar[p] == ts and math.isclose(res.L[p], L, rel_tol=1e-15)
        _close(res.u[p], u[p] + du, "u")
        _close(res.vi[p], vi[p] + dvi, "v_i")
        _close(res.vs[p], vj[p, ts] + dvj, "v_j")
        if res.decided[p]:   # fp32: the same violator, the deltas within the bound
            up, vp, vs = u[p].astype(F), vi[p].astype(F), vj[p, ts].astype(F)
            g = lr32 * F(math.log(max(1, (rank_items - 1) // n)))
            _within(up + (g * (vp - vs) - lr32 * reg32 * up), res.u[p], res.tol_u[p], "fp32 u")
            _within(vs + (-g * up - lr32 * reg32 * vs), res.vs[p], res.tol_vs[p], "fp32 v_j")
            xs = [(up * (vp - vj[p, t].astype(F))).sum(dtype=F) for t in range(6) if live[p, t]]
            assert next(i for i, x in enumerate(xs) if x < m32) + 1 == n
    assert res.updated == res.hit.sum() and res.examined == res.n.sum()


def test_warp_replay_rank_estimate_can_be_zero():
    """(N - 1) // n <= 1 gives L = 0: a decay-only update, still counted as updated."""
    rng, u, vi, vj, negs = _case(4, P=8, T=2, k=5)
    res = warp_replay(u, vi, vj, np.ones((8, 2), bool), 0.1, 0.01, 10.0, 2, 8)
    assert res.hit.all() and (res.L == 0).all() and res.updated == 8
    _close(res.u, u - f32(0.1) * f32(0.01) * u, "decay only")


# ---- pointwise, SGD and row-wise AdaGrad ------------------------------------------------------------------------

@pytest.mark.parametrize("ada", [False, True])
@pytest.mark.parametrize("err_mode", [0, 1, 2])
@pytest.mark.parametrize("k,stride", [(3, 4), (29, 32), (509, 512), (1021, 1024)])
def test_pointwise_replay_matches_numpy_reference_and_fp32(err_mode, k, stride, ada):
    rng = np.random.default_rng(k + err_mode)
    P = 50
    u0, v0 = _rows(rng, (P, k), k ** -0.25), _rows(rng, (P, k), k ** -0.25)
    r = rng.integers(0, 2, P).astype(np.float64) if err_mode != 1 else rng.integers(1, 9, P) * 0.5
    Gu = np.where(rng.random(P) < 0.5, rng.random(P), 0.0).astype(F).astype(np.float64)
    Gv = rng.random(P).astype(F).astype(np.float64)
    lr = f32(0.1)
    res = pointwise_replay(u0, v0, r, lr, err_mode, geometry(stride, 256)[0], acc=(Gu, Gv) if ada else None)
    d = (u0 * v0).sum(1)
    e = {0: 1 / (1 + np.exp(-(r - d))), 1: r - d, 2: r - 1 / (1 + np.exp(-d))}[err_mode]
    if ada:
        assert res.e_ok
        for p in range(P):
            nu, su = rowwise_adagrad(u0[p], Gu[p], e[p] * v0[p], lr, k)
            nv, sv = rowwise_adagrad(v0[p], Gv[p], e[p] * u0[p], lr, k)
            _close(res.u[p], nu, "u")
            _close(res.v[p], nv, "v")
            assert math.isclose(res.Gu[p], Gu[p] + su, rel_tol=1e-12)
            assert math.isclose(res.Gv[p], Gv[p] + sv, rel_tol=1e-12)
    else:
        assert res.Gu is None and res.Gv is None and res.tol_Gu is None and res.tol_Gv is None and res.e_ok is None
        _close(res.u, u0 + (lr * e)[:, None] * v0, "u")
        _close(res.v, v0 + (lr * e)[:, None] * u0, "v")
    # fp32
    U, V = u0.astype(F), v0.astype(F)
    d32 = (U * V).sum(1, dtype=F)
    rr = r.astype(F)
    e32 = {0: _sig32(rr - d32), 1: rr - d32, 2: rr - _sig32(d32)}[err_mode]
    if ada:
        ee = e32 * e32 / F(k)
        su, sv = ee * (V * V).sum(1, dtype=F), ee * (U * U).sum(1, dtype=F)
        gu = e32 * (F(lr) / (np.sqrt(Gu.astype(F) + su) + F(1e-8)))
        gv = e32 * (F(lr) / (np.sqrt(Gv.astype(F) + sv) + F(1e-8)))
    else:
        gu = gv = F(lr) * e32
    _within(U + gu[:, None] * V, res.u, res.tol_u, "fp32 u")
    _within(V + gv[:, None] * U, res.v, res.tol_v, "fp32 v")


# ---- the sampled candidates -------------------------------------------------------------------------------------

def test_sampled_candidates_are_k5_negative_t_plus_one():
    items = np.arange(30) % 7
    c = sampled_candidates(30, items, 3, 7, 5, (7 << 32) + 1)
    for t in range(3):
        assert np.array_equal(c[:, t], k5_negative(np.arange(30), t + 1, items, 7, 5, (7 << 32) + 1)[0])
    assert (c != items[:, None]).all()
