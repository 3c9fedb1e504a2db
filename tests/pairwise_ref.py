"""fp64 replays of the pairwise MF steps (``fps_mf_bpr_kernel`` under SGD and row-wise AdaGrad,
``fps_mf_warp_kernel``), each with a first-order bound on every table element, accumulator and stat.  CPU only: the
GPU suites feed them the fp32 rows the kernel pulls, as float64 arrays of the logical ``k`` columns.

Where the fp32 kernels round (unit roundoff EPS = 2^-24, round to nearest; ``ops/build.py`` builds without
fast-math, so ``sqrtf`` and ``/`` are correctly rounded):
- a lane's part of a dot is an FMUL, three FFMAs and an add per float4, over ``VPL`` float4, then ``log2(LPR)``
  shuffle adds: a sum of depth ``5 VPL + log2(LPR)``; the pairwise ``v_i - v_j`` adds one rounding per term;
- ``__expf(x)`` within ``(2 + 1.173 |x|)`` ulp; ``logf`` and ``log1pf`` within 1 ulp, ``expf`` within 2 ulp (CUDA C
  Programming Guide); ``(float)((N - 1) / n)`` is exact below 2^24;
- one rounding per product, per add, per FMA and per reduction into a table.
A sum of depth ``n`` is within ``n EPS sum|terms|`` of the exact one.  Every bound is first order; the suites compare
with ``MARGIN`` times it, which covers the second-order terms.

Two discontinuities are conditions, not tolerances: the WARP violator (``x`` next to the margin), and the AdaGrad
step of a row whose ``G`` and delta are both near zero (``delta / |delta|`` keeps only the direction).  The replays
return whether their input stays clear of both, and the suites assert it."""
import math

import numpy as np

from tests.philox_ref import k5_negative

EPS = 2.0 ** -24          # fp32 unit roundoff
ULP = 2.0 ** -23          # one ulp, relative
MARGIN = 2.0
ADA_EPS = 1e-8


def f32(x):
    return float(np.float32(x))


def geometry(stride, max_nvec=128):
    """(LPR, VPL) of dispatch_bpr / dispatch_warp (max_nvec 128) and dispatch_mf's AdaGrad branch (256)."""
    nvec = stride // 4
    if nvec > max_nvec:
        raise ValueError(f"no rung for {nvec} float4")
    lpr = min(32, 1 << max(0, nvec - 1).bit_length())
    return lpr, -(-nvec // lpr)


def dot_depth(stride, lpr):
    """Depth of the kernels' fp32 dot over rows of ``stride`` floats on ``lpr`` lanes: each lane's running sum of
    ceil(nvec / lpr) float4 dots (an FMUL, three FFMAs and an add each), then log2(lpr) shuffle adds."""
    return 5 * -(-(stride // 4) // lpr) + int(math.log2(lpr))


def sampled_candidates(n_pos, items, T, num_items, step, seed):
    """Candidate ``t`` of positive ``pos`` as BPR and WARP draw it: K5 key ``(pos, t + 1, step, seed)``.  [n_pos, T]"""
    pos = np.arange(n_pos)
    return np.stack([k5_negative(pos, t + 1, items, num_items, step, seed)[0] for t in range(T)], 1)


def _sig(x):
    """sigmoid(x), overflow-free."""
    return 0.5 * (1.0 + np.tanh(0.5 * x))


def _expf_rel(x):
    return (2.0 + 1.173 * np.abs(x)) * ULP


def _dot(u, diff, depth, du=None):
    """x = u . diff and its bound: the sum's depth, the subtraction that formed diff, and diff's own error ``du``."""
    x = (u * diff).sum(-1)
    dx = (depth + 1) * EPS * np.abs(u * diff).sum(-1)
    if du is not None:
        dx = dx + (np.abs(u) * du).sum(-1)
    return x, dx


def _step(lr, G, dG, s, ds):
    """lr / (sqrt(G + s) + eps) and its bound (the add, sqrt, add and division round once each)."""
    Gs = G + s
    sq = np.sqrt(Gs)
    step = lr / (sq + ADA_EPS)
    dGs = dG + ds + EPS * Gs
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = np.where(Gs > 0, dGs / (2 * sq * (sq + ADA_EPS)), 0.0)
    return step, step * (rel + 4 * EPS), rel


def _norm2(delta, ddelta, k, depth):
    """s = |delta|^2 / k (the kernel's sum of squares of depth ``depth``, times a rounded 1 / k) and its bound."""
    s = (delta * delta).sum(-1) / k
    ds = 2 * (np.abs(delta) * ddelta).sum(-1) / k + (depth + 2) * EPS * s
    return s, ds


class Result(dict):
    __getattr__ = dict.__getitem__


# ---- BPR, SGD and row-wise AdaGrad -----------------------------------------------------------------------------

def bpr_replay(u, vi, vj, negs, lr, reg, stride, ada=None):
    """One BPR launch over independent positives.  ``u``, ``vi`` ``[P, k]`` and ``vj`` ``[P, T, k]``: the rows as
    pulled; ``negs`` ``[P, T]``: candidate ids as the kernel resolves them (``-1`` = void; the caller voids a negative
    equal to its positive).  A negative repeated in one positive's list is read with the earlier triples' pushes
    applied (and, under AdaGrad, with their ``G += s``): sequential in the list.

    ``ada``: ``None`` for SGD, else ``(Gu [P], Gi [P], Gj [P, T], k)``, the accumulators as pulled.

    Returns a :class:`Result`: ``u``, ``vi`` and ``vj`` ``[P, T, k]`` (the row after triple ``t``'s push) with
    ``tol_*``; under AdaGrad ``Gu``, ``Gi``, ``Gj`` with ``tol_G*``; ``n_live``; the stats ``loss``, ``tol_loss``,
    ``count``, ``xpos_lo`` / ``xpos_hi`` (the ``x > 0`` count, the bound admitting either side at ``x`` near 0); and
    ``smooth`` (every AdaGrad step's relative bound below 1e-3)."""
    P, T, k = vj.shape
    depth = dot_depth(stride, geometry(stride)[0])
    lr32, reg32 = f32(lr), f32(reg)
    rate, decay = (1.0, reg32) if ada is not None else (lr32, lr32 * reg32)
    d_decay = 0.0 if ada is not None else EPS * decay          # lr * reg rounded once
    live = negs >= 0
    n_live = live.sum(1)
    worst_rel = np.zeros(P)
    out_vj, tol_vj = vj.copy(), np.zeros_like(vj)
    Gj_out, tol_Gj = None, None
    if ada is not None:
        Gu, Gi, Gj, kk = ada
        assert kk == k
        Gj_out, tol_Gj = Gj.astype(np.float64).copy(), np.zeros(Gj.shape)
    du_acc, ddu_acc, dterm_sum = np.zeros((P, k)), np.zeros((P, k)), np.zeros((P, k))
    g_sum, dg_sum, g_abs = np.zeros(P), np.zeros(P), np.zeros(P)
    loss = dloss = 0.0
    xs, dxs = [], []
    for t in range(T):
        # the row this triple reads: the originally pulled one, or the one the latest earlier repeat pushed to
        r, dr = vj[:, t].copy(), np.zeros((P, k))
        G_r = dG_r = None
        if ada is not None:
            G_r, dG_r = Gj[:, t].astype(np.float64).copy(), np.zeros(P)
        for t2 in range(t):
            rep = live[:, t] & (negs[:, t2] == negs[:, t])
            r[rep], dr[rep] = out_vj[rep, t2], tol_vj[rep, t2]
            if ada is not None:
                G_r[rep], dG_r[rep] = Gj_out[rep, t2], tol_Gj[rep, t2]
        lv = live[:, t]
        diff = vi - r
        x, dx = _dot(u, diff, depth, dr)
        sp = _sig(x)                                              # sigmoid(x); g = rate * sigmoid(-x)
        g = rate * _sig(-x)
        dg = g * (sp * (_expf_rel(x) + dx) + 2 * EPS)
        # v_j's delta: -g u - decay v_j (an FMA over a product)
        dj = -g[:, None] * u - decay * r
        ddj = np.abs(u) * dg[:, None] + 2 * EPS * (np.abs(g[:, None] * u) + np.abs(decay * r)) \
            + decay * dr + d_decay * np.abs(r)
        if ada is None:
            new = r + dj
            dnew = dr + ddj + EPS * np.abs(new)
        else:
            s, ds = _norm2(dj, ddj, k, depth)
            st, dst, rel = _step(lr32, G_r, dG_r, s, ds)
            worst_rel = np.where(lv, np.maximum(worst_rel, rel), worst_rel)
            upd = st[:, None] * dj
            new = r + upd
            dnew = dr + np.abs(dj) * dst[:, None] + st[:, None] * ddj + EPS * np.abs(upd) + EPS * np.abs(new)
            Gn = G_r + s
            Gj_out[lv, t], tol_Gj[lv, t] = Gn[lv], (dG_r + ds + EPS * Gn)[lv]
        out_vj[lv, t], tol_vj[lv, t] = new[lv], dnew[lv]
        # the summed anchor delta and g, from the live triples
        m = lv[:, None]
        du_acc += np.where(m, g[:, None] * diff, 0.0)
        gd = np.abs(g[:, None] * diff)
        ddu_acc += np.where(m, np.abs(diff) * dg[:, None] + EPS * gd + np.abs(g[:, None]) * dr, 0.0)
        dterm_sum += np.where(m, gd, 0.0)
        g_sum += np.where(lv, g, 0.0)
        dg_sum += np.where(lv, dg, 0.0)
        g_abs += np.where(lv, np.abs(g), 0.0)
        # stats: softplus(-x) = max(-x, 0) + log1p(exp(-|x|))
        lt = np.maximum(-x, 0.0) + np.log1p(np.exp(-np.abs(x)))
        loss += lt[lv].sum()
        dloss += (_sig(-x) * dx + 11 * EPS * lt)[lv].sum()
        xs.append(x[lv])
        dxs.append(dx[lv])
    ddu_acc += n_live[:, None] * EPS * dterm_sum                  # one FMA rounding per accumulated triple
    dg_sum += n_live * EPS * g_abs
    dec = decay * n_live
    d_dec = 2 * EPS * dec if ada is None else EPS * dec           # (lr * reg) * n_live, or reg * n_live
    du = du_acc - dec[:, None] * u
    d_du = ddu_acc + d_dec[:, None] * np.abs(u) + EPS * (np.abs(du_acc) + np.abs(dec[:, None] * u))
    di = g_sum[:, None] * u - dec[:, None] * vi
    d_di = np.abs(u) * dg_sum[:, None] + d_dec[:, None] * np.abs(vi) \
        + 2 * EPS * (np.abs(g_sum[:, None] * u) + np.abs(dec[:, None] * vi))
    res = Result(n_live=n_live, vj=out_vj, tol_vj=tol_vj)
    wrote = (n_live > 0)[:, None]
    if ada is None:
        u1, vi1 = u + du, vi + di
        res.update(u=np.where(wrote, u1, u), tol_u=np.where(wrote, d_du + EPS * np.abs(u1), 0.0),
                   vi=np.where(wrote, vi1, vi), tol_vi=np.where(wrote, d_di + EPS * np.abs(vi1), 0.0))
    else:
        for name, row, G, delta, dd in (("u", u, Gu, du, d_du), ("vi", vi, Gi, di, d_di)):
            s, ds = _norm2(delta, dd, k, depth)
            G = G.astype(np.float64)
            st, dst, rel = _step(lr32, G, 0.0, s, ds)
            worst_rel = np.where(n_live > 0, np.maximum(worst_rel, rel), worst_rel)
            upd = st[:, None] * delta
            new = row + upd
            dnew = np.abs(delta) * dst[:, None] + st[:, None] * dd + EPS * np.abs(upd) + EPS * np.abs(new)
            key = "Gu" if name == "u" else "Gi"
            res[name] = np.where(wrote, new, row)
            res["tol_" + name] = np.where(wrote, dnew, 0.0)
            res[key] = np.where(n_live > 0, G + s, G)
            res["tol_" + key] = np.where(n_live > 0, ds + EPS * (G + s), 0.0)
        res.update(Gj=Gj_out, tol_Gj=tol_Gj)
    x_all, dx_all = np.concatenate(xs), np.concatenate(dxs)
    count = int(n_live.sum())
    res.update(loss=loss, tol_loss=dloss + (count + 1) * EPS * loss, count=count,
               xpos_lo=int((x_all - MARGIN * dx_all > 0).sum()), xpos_hi=int((x_all + MARGIN * dx_all > 0).sum()),
               smooth=bool((worst_rel < 1e-3).all()))
    return res


# ---- WARP ------------------------------------------------------------------------------------------------------

def warp_replay(u, vi, vj, live, lr, reg, margin, rank_items, stride):
    """One WARP launch over independent positives: candidate rows ``vj`` ``[P, T, k]`` in draw order, ``live``
    ``[P, T]`` (void candidates are skipped and not counted).  The first live ``x_t < margin`` violates; ``n`` counts
    the live candidates examined up to it; ``L = ln(max(1, (rank_items - 1) // n))``.

    Returns a :class:`Result`: ``hit`` [P], ``tstar`` [P] (-1 without a violator), ``n`` [P], ``L``, the rows ``u``,
    ``vi``, ``vs`` (the violator's row, pushed) with ``tol_*``; the stats ``loss``, ``tol_loss``, ``updated``,
    ``examined``; and ``decided`` [P]: every examined ``x`` is farther from the margin than MARGIN times its bound,
    so the violator is the same in any fp32 evaluation."""
    P, T, k = vj.shape
    depth = dot_depth(stride, geometry(stride)[0])
    lr32, m32 = f32(lr), f32(margin)
    decay = lr32 * f32(reg)
    active = np.ones(P, dtype=bool)
    hit = np.zeros(P, dtype=bool)
    tstar = np.full(P, -1)
    n = np.zeros(P, dtype=np.int64)
    decided = np.ones(P, dtype=bool)
    xstar, dxstar = np.zeros(P), np.zeros(P)
    for t in range(T):
        x, dx = _dot(u, vi - vj[:, t], depth)
        ex = active & live[:, t]
        n += ex
        decided &= ~ex | (np.abs(x - m32) > MARGIN * dx)
        v = ex & (x < m32)
        hit |= v
        tstar[v], xstar[v], dxstar[v] = t, x[v], dx[v]
        active &= ~v
    ratio = (int(rank_items) - 1) // np.maximum(n, 1)
    L = np.where(hit, np.log(np.maximum(1, ratio).astype(np.float64)), 0.0)
    dL = ULP * np.abs(L)
    g = lr32 * L
    dg = lr32 * dL + EPS * np.abs(g)
    vs = vj[np.arange(P), np.maximum(tstar, 0)]
    diff = vi - vs
    G, gd = g[:, None], dg[:, None]
    upd_u = G * diff - decay * u
    upd_i = G * u - decay * vi
    upd_j = -G * u - decay * vs

    def tol(upd, a, b, bx, row):
        # |a| dg + the diff's rounding + the two products' roundings + the decay's rounding + the reduction's
        new = row + upd
        return new, np.abs(a) * gd + 2 * EPS * (np.abs(G * a) + np.abs(decay * b)) + EPS * decay * np.abs(b) \
            + bx + EPS * np.abs(new)

    h = hit[:, None]
    u1, tu = tol(upd_u, diff, u, EPS * np.abs(G * diff), u)
    vi1, ti = tol(upd_i, u, vi, 0.0, vi)
    vs1, tj = tol(upd_j, u, vs, 0.0, vs)
    lt = L * (m32 - xstar)
    dlt = np.abs(m32 - xstar) * dL + L * dxstar + 2 * EPS * np.abs(lt)
    loss = lt[hit].sum()
    return Result(hit=hit, tstar=tstar, n=n, L=L, decided=decided,
                  u=np.where(h, u1, u), tol_u=np.where(h, tu, 0.0), vi=np.where(h, vi1, vi),
                  tol_vi=np.where(h, ti, 0.0), vs=np.where(h, vs1, vs), tol_vs=np.where(h, tj, 0.0),
                  loss=loss, tol_loss=dlt[hit].sum() + (P + 1) * EPS * loss, updated=int(hit.sum()),
                  examined=int(n.sum()))
