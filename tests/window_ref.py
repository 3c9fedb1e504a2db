"""fp64 replay of the step-window drain (``fps_mf_window_kernel``, ``ops/csrc/fps_mf_window.cu``): which windows and
singletons it forms from the staged micro-batches, and what it writes, with a first-order bound on every table
element and stat.  CPU only: the GPU suite feeds it the fp32 rows the drain starts from, as float64 arrays of the
logical ``k`` columns.

The drain splits the staged micro-batches greedily: micro-batch ``j`` joins the open window if, counting only its
live records (int32 ``user >= 0``), its items are distinct, its users are distinct and its users are disjoint from
the window's so far.  Every attempt to add one is a scatter pass.  A window's first micro-batch that fails is a
singleton, applied on its own with the per-launch update.

Inside a window every user row is read and written once and every item row once per micro-batch, so each item's
chain (its updates in micro-batch order) is the per-launch step applied micro-batch after micro-batch.  Where the
fp32 kernel rounds (unit roundoff EPS = 2^-24):
- ``win_dot`` reproduces ``fps_group_sum<LPR>``'s tree over one float4 dot per lane: a sum of depth ``5 + log2(LPR)``;
- ``__expf(x)`` is within ``(2 + 1.173 |x|)`` ulp (CUDA C Programming Guide); ``g = lr e`` rounds once;
- ``u + g v`` is a product and an add (``win_add``) per element.
An item row's error grows with every link of its chain: the next dot sees ``sum |u| tol_v`` on top of its own
rounding.  A singleton pulls rows that other records of its micro-batch may already have pushed to: its dots carry
those pushes' magnitudes as a further bound, and its reductions one rounding each.  Every bound is first order; the
suite compares with ``MARGIN`` times it."""
import numpy as np

from tests.pointwise_ref import dot_depth, grad

EPS = 2.0 ** -24          # fp32 unit roundoff
MARGIN = 2.0
WIN_MAX = 8               # micro-batches per drain (fps_mf_window.cu WIN_MAX)


def lanes(stride):
    """LPR bucket of ``fps_mf_window_drain`` for rows of ``stride`` floats: 1, 2, 4, 8, 16 or 32 lanes."""
    nvec = stride // 4
    if not 1 <= nvec <= 32:
        raise ValueError(f"no window bucket for {nvec} float4")
    return 1 << max(0, nvec - 1).bit_length()


def partition(batches):
    """The drain's windows from ``batches`` = [(users, items)] (int arrays, ``user < 0`` void).  Returns
    (groups, attempts): ``groups`` lists ``(start, end, singleton)`` in order, ``attempts`` the scatter passes."""
    live = []
    for u, i in batches:
        u, i = np.asarray(u, dtype=np.int64), np.asarray(i, dtype=np.int64)
        keep = u >= 0
        live.append((u[keep], i[keep]))
    groups, attempts, start = [], 0, 0
    while start < len(live):
        seen = np.zeros(0, dtype=np.int64)
        end = start
        while end < len(live):
            attempts += 1
            u, i = live[end]
            own = len(np.unique(u)) == len(u) and len(np.unique(i)) == len(i)
            if not own or np.isin(u, seen).any():
                break
            seen = np.concatenate([seen, u])
            end += 1
        if end > start:
            groups.append((start, end, False))
            start = end
        else:
            groups.append((start, start + 1, True))
            start += 1
    return groups, attempts


def replay(U0, V0, batches, lr, err_mode, lpr, groups=None):
    """The drain on ``U0`` [n_users, k] and ``V0`` [n_items, k] (float64 holding the fp32 rows) with ``batches`` =
    [(users, items, ratings)] indexing them (``user < 0`` void; ratings as the kernel reads them, so fp16-rounded
    for packed64 records).  ``groups``: the partition of the full micro-batches when ``batches`` keep only some of
    their records (default: the partition of ``batches``).

    Returns a dict: ``U``, ``V`` and their bounds ``tU``, ``tV``; per micro-batch ``sq``, ``cnt`` and ``tol_sq``
    (the slot_stats row and the bound on its sum); ``groups``, ``attempts``."""
    attempts = None
    if groups is None:
        groups, attempts = partition([(u, i) for u, i, _ in batches])
    U, V = np.array(U0, dtype=np.float64), np.array(V0, dtype=np.float64)
    tU, tV = np.zeros_like(U), np.zeros_like(V)
    depth = dot_depth(-(-U.shape[1] // 4) * 4, lpr)
    lr32 = float(np.float32(lr))
    n = len(batches)
    sq, cnt, tol_sq = np.zeros(n), np.zeros(n), np.zeros(n)
    with np.errstate(all="ignore"):      # a non-finite rating carries through as inf / nan
        for start, end, singleton in groups:
            for j in range(start, end):
                users, items, r = (np.asarray(a) for a in batches[j])
                keep = users >= 0
                users, items = users[keep].astype(np.int64), items[keep].astype(np.int64)
                r = r[keep].astype(np.float64)
                u0, v0, du0, dv0 = U[users], V[items], tU[users], tV[items]
                d = (u0 * v0).sum(1)
                dd = depth * EPS * np.abs(u0 * v0).sum(1) + (np.abs(u0) * dv0 + np.abs(v0) * du0).sum(1)
                if singleton:
                    # pushes of the other records to the rows this one pulls, to first order |g| times the row
                    g0 = grad(r, d, dd, lr32, err_mode)[2][:, None]
                    pu, pv = np.abs(g0 * v0), np.abs(g0 * u0)
                    su, sv = np.zeros_like(U), np.zeros_like(V)
                    np.add.at(su, users, pu)
                    np.add.at(sv, items, pv)
                    race_u, race_v = su[users] - pu, sv[items] - pv
                    dd = dd + (np.abs(u0) * race_v + np.abs(v0) * race_u).sum(1)
                resid, dres, g, dg = grad(r, d, dd, lr32, err_mode)
                g, dg = g[:, None], dg[:, None]
                du_new = np.abs(g) * dv0 + dg * np.abs(v0)
                dv_new = np.abs(g) * du0 + dg * np.abs(u0)
                if singleton:
                    # the pulled row in the push, with the same race; red.global.add of the product: one rounding
                    # for it, one for each reduction into the row
                    du_new = du_new + np.abs(g) * race_v
                    dv_new = dv_new + np.abs(g) * race_u
                    for T, tT, ids, delta, dnew in ((U, tU, users, g * v0, du_new), (V, tV, items, g * u0, dv_new)):
                        m, mag = np.zeros(len(T)), np.abs(T).copy()
                        np.add.at(m, ids, 1.0)
                        np.add.at(mag, ids, np.abs(delta))
                        np.add.at(tT, ids, dnew + EPS * np.abs(delta))
                        np.add.at(T, ids, delta)
                        touched = m > 0
                        tT[touched] += (m[touched, None] + 1) * EPS * mag[touched]
                else:
                    u1, v1 = u0 + g * v0, v0 + g * u0
                    U[users] = u1
                    V[items] = v1
                    tU[users] = du0 + du_new + 2 * EPS * (np.abs(g * v0) + np.abs(u1))
                    tV[items] = dv0 + dv_new + 2 * EPS * (np.abs(g * u0) + np.abs(v1))
                s = resid * resid
                sq[j], cnt[j] = s.sum(), len(s)
                tol_sq[j] = (2 * np.abs(resid) * dres + dres * dres).sum() + (len(s) + 1) * EPS * s.sum()
    return {"U": U, "V": V, "tU": tU, "tV": tV, "sq": sq, "cnt": cnt, "tol_sq": tol_sq, "groups": groups,
            "attempts": attempts}


def stats_bound(rep):
    """Bound on ``stats[0]``: the fp32 sum of the micro-batch sums, added in slot order onto a zero stats."""
    return rep["tol_sq"].sum() + (len(rep["sq"]) + 1) * EPS * rep["sq"].sum()
