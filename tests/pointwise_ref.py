"""fp64 replay of the pointwise MF step (``fps_mf_sgd_fused_kernel``, SGD and row-wise AdaGrad) with a first-order
bound on every table element, accumulator and loss term, and the error model of ``fps_mf_grad`` that the step-window
replay (``tests/window_ref.py``) shares.  CPU only: the GPU suites feed it the fp32 rows the kernel pulls, as float64
arrays of the logical ``k`` columns.

The kernel computes, per record, in fp32: ``d = u.v`` (``dot_depth`` roundings deep); ``resid = r - d``; ``e`` from
``resid`` or ``d``; ``__expf(x)`` is within ``(2 + 1.173 |x|)`` ulp (CUDA C Programming Guide, intrinsic functions),
and the sigmoid ``1 / (1 + E)`` moves by at most a quarter of E's relative error, plus its add and division.
- SGD: ``g = lr e``; ``u += g v`` and ``v += g u`` by one product and one reduction each.
- Row-wise AdaGrad: ``e`` at rate 1, ``delta_u = e v``, ``delta_v = e u``, and per row ``s = |delta|^2 / k``,
  ``row += lr delta / (sqrt(G + s) + 1e-8)``, ``G += s``.
Every bound is first order; the suites compare with ``MARGIN`` times it, which covers the second-order terms."""
import numpy as np

from tests.pairwise_ref import EPS, MARGIN, ULP, Result, _sig, _step, dot_depth, f32


def sigmoid_err(x):
    """Relative error of the kernel's 1 / (1 + __expf(-x)): a quarter of __expf's, plus the add and the division."""
    return 0.25 * (2.0 + 1.173 * np.abs(x)) * ULP + 2 * EPS


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _error(r, d, dd, err_mode, sig=_sigmoid):
    """(resid, dres, e, de): fps_mf_grad's error at rate 1 and its bound, from d and its bound.  ``sig``: the fp64
    sigmoid; either form is exact to fp64 rounding, far inside the bound."""
    resid = r - d
    dres = dd + EPS * np.abs(resid)
    if err_mode == 0:
        e = sig(resid)
        de = 0.25 * dres + sigmoid_err(resid)
    elif err_mode == 1:
        e, de = resid, dres
    else:
        e = r - sig(d)
        de = 0.25 * dd + sigmoid_err(d) + EPS * np.abs(e)
    return resid, dres, e, de


def grad(r, d, dd, lr32, err_mode):
    """(resid, dres, g, dg) of fps_mf_grad from d and its bound: g = lr e, rounded once."""
    resid, dres, e, de = _error(r, d, dd, err_mode)
    g = lr32 * e
    return resid, dres, g, lr32 * de + EPS * np.abs(g)


def loss_bound(resid, dres):
    """The loss stat, an fp32 sum of the squared residuals in any order: each square is off by 2 |resid| dres (+ its
    rounding), and a sum of n terms in any order by n * EPS * sum."""
    sq = resid * resid
    return (2 * np.abs(resid) * dres + dres * dres).sum() + (len(resid) + 1) * EPS * sq.sum()


def replay(u0, v0, r, lr, err_mode, lpr, acc=None):
    """One launch over independent records: ``u0``, ``v0`` ``[n, k]`` the rows each record pulls, ``r`` the ratings
    as the kernel reads them, ``lpr`` the lanes per row of the geometry that runs.  ``acc``: ``None`` for SGD, else
    ``(Gu, Gv)``, the accumulators as pulled.

    Returns a :class:`Result` with ``u``, ``v`` and their ``tol_*``, ``resid`` / ``tol_resid`` (the loss stat's
    terms), and under AdaGrad ``Gu``, ``Gv`` with ``tol_G*`` and ``e_ok``: ``|e|`` above MARGIN times its bound, so
    the step's direction is settled where ``G`` is 0.  These five are ``None`` under SGD."""
    k = u0.shape[1]
    depth = dot_depth(-(-k // 4) * 4, lpr)
    lr32 = f32(lr)
    d = (u0 * v0).sum(1)
    dd = depth * EPS * np.abs(u0 * v0).sum(1)
    res = Result(Gu=None, Gv=None, tol_Gu=None, tol_Gv=None, e_ok=None)
    if acc is None:
        resid, dres, g, dg = grad(r, d, dd, lr32, err_mode)
        u1 = u0 + g[:, None] * v0
        v1 = v0 + g[:, None] * u0
        res.update(u=u1, v=v1, resid=resid, tol_resid=dres,
                   tol_u=dg[:, None] * np.abs(v0) + 2 * EPS * (np.abs(g[:, None] * v0) + np.abs(u1)),
                   tol_v=dg[:, None] * np.abs(u0) + 2 * EPS * (np.abs(g[:, None] * u0) + np.abs(v1)))
        return res
    resid, dres, e, de = _error(r, d, dd, err_mode, _sig)     # the overflow-free form of the pairwise replays
    nu, nv = (u0 * u0).sum(1), (v0 * v0).sum(1)
    dnu, dnv = depth * EPS * nu, depth * EPS * nv
    ee = e * e / k                                                # g * g / (float)dim: two roundings
    dee = 2 * np.abs(e) * de / k + 2 * EPS * ee
    res.update(resid=resid, tol_resid=dres, e_ok=bool((np.abs(e) > MARGIN * de).all()))
    for name, row, other, G, nrm, dnrm in (("u", u0, v0, acc[0], nv, dnv), ("v", v0, u0, acc[1], nu, dnu)):
        s = ee * nrm
        ds = dee * nrm + ee * dnrm + EPS * s
        G = G.astype(np.float64)
        st, dst, _ = _step(lr32, G, 0.0, s, ds)
        gr = e * st
        dgr = np.abs(e) * dst + st * de + EPS * np.abs(gr)
        upd = gr[:, None] * other
        new = row + upd
        res[name] = new
        res["tol_" + name] = np.abs(other) * dgr[:, None] + EPS * np.abs(upd) + EPS * np.abs(new)
        key = "G" + name
        res[key] = G + s
        res["tol_" + key] = ds + EPS * (G + s)
    return res
