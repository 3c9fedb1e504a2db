"""fp64 replay of one ``fps_pa_step`` launch (ops/csrc/fps_pa.cu, both the warp and the block kernel) with a
first-order bound on every table element.  CPU only: the GPU suite feeds it the fp32 table as the kernel reads it.

Semantics mirrored from the kernels:
- Examples run in CSR order, each reading the table as the earlier examples left it.  (The kernel races the
  examples of one launch; with disjoint feature sets per example that race has this one result.)
- Predictions use the parameters from before the example's own update.  Binary predicts ``d > 0``; multiclass
  takes the first maximum (``np.argmax``: ties go to the lower class, NaN ranks first).  An all-zero decision
  vector is computed exactly, so it predicts 0 exactly and is not a tie within tolerance.
- No update unless the example is labelled, has an entry, and ``||x||^2 > 0`` in fp32 (a NaN norm does not
  update either).  The host algorithms would divide by zero there instead.
- Entries are used in CSR order.  A feature repeated within one example contributes once per entry to ``d``,
  to ``||x||^2`` and to the pushes, like ``SparseVector`` (which sorts but does not merge repeats).
- ``loss`` is written only for an example that updates, and then only when ``L == 1`` (the hinge), or for PB /
  ML when ``q != label`` (``d_q - d_label + sqrt(c)``).  Everywhere else the output is NaN: untouched.
- PB's ``q`` is the prediction; ML's ``q`` is the first maximum of ``d_i - d_label + sqrt(c(label, i))``.
  Without a cost matrix the cost is 0 on the diagonal and 1 elsewhere.
- A push adds ``x * mult`` to the row one 4-column chunk at a time, and skips a chunk whose four products are
  all zero.  ``red.add.f32`` (SASS ``REDG.E.ADD.F32[x4].FTZ.RN``) flushes subnormal inputs and results to zero,
  on every column of a pushed chunk.
- The non-finite flag is raised by a pushed chunk whose ``|d.x| + |d.y| + |d.z| + |d.w|`` is not ``<= 3e38``.

Error model (first order, EPS = 2^-24, round to nearest; ``ops/build.py`` builds without fast-math, so ``/`` and
``sqrtf`` round once).  Every bound holds for any summation order, because the block kernel reduces through
shared-memory atomics in no fixed order:
- ``d_i`` and ``||x||^2``: ``(k - 1) EPS sum|terms|`` over the ``k`` nonzero terms (adding a zero is exact), plus
  one rounding per inexact product, plus ``sum |x| tol(w)`` carried from earlier pushes in the same launch;
- the hinge, PA-I's ``min`` and the arg-max inputs carry their error through, plus one rounding per ``-`` / ``+``;
- one rounding per ``/`` and per product; ``1.f / (2.f * C)`` and ``sqrtf(cost)`` are replayed exactly in fp32;
- one rounding per push into the table, so ``k`` roundings for a feature repeated ``k`` times.
An operation on exact inputs whose result is an fp32 number adds no rounding, which keeps exact ties exact.

``fp32=False`` switches the fp32 model off (no overflow to inf, no flush to zero, C and the cost used as given):
the replay is then the host algorithms of ``models/pa/algorithms.py`` evaluated in fp64."""
import numpy as np

EPS = 2.0 ** -24
MARGIN = 2.0
FLT_MIN = 2.0 ** -126
FLAG_LIMIT = 3.0e38
UNLABELLED = -(2 ** 31)
MAX_LABELS = 1024
ALGOS = ("PA", "PAI", "PAII", "PB", "ML")


def geometry(L, variant=0):
    """(kernel, LPR, VPL) that ``dispatch_pa`` launches for ``L`` labels; ``variant`` 1 forces the block kernel."""
    if not 1 <= L <= MAX_LABELS:
        raise ValueError(f"no kernel for {L} labels")
    nvec = -(-L // 4)
    lpr = min(32, 1 << max(0, nvec - 1).bit_length())
    if variant == 0 and nvec <= 32 and L <= 128:
        return "warp", lpr, 1
    return "block", lpr, (8 if lpr == 32 else 1)


def dispatch_table():
    """Every (kernel, LPR, VPL) rung of ``dispatch_pa``."""
    return sorted({geometry(L, v) for L in range(1, MAX_LABELS + 1) for v in (0, 1)})


def cap(kernel, sms):
    """Examples one launch covers before its grid-stride loop takes a second round."""
    return sms * (32 if kernel == "warp" else 16)


class Result(dict):
    __getattr__ = dict.__getitem__


def _rnd(r, t_in):
    """One rounding of result ``r`` whose inputs carry ``t_in``; none when they are exact and ``r`` is an fp32."""
    with np.errstate(over="ignore", invalid="ignore"):
        inexact = (np.asarray(t_in) > 0) | (np.float32(r) != r)
        return t_in + np.where(inexact & np.isfinite(r), EPS * np.abs(r), 0.0)


def _div(a, ta, b, tb):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = a / b
        t = np.where(np.isfinite(q), np.abs(q) * tb / np.abs(b) + ta / np.abs(b), 0.0)
    return q, _rnd(q, t)


def first_argmax(v, t, same=None):
    """(np.argmax of ``v``, whether the choice is clear of the bounds ``t``): every rival is either behind by more
    than ``MARGIN`` times the two bounds, or equal with both exact, or computed from the same inputs as the winner
    (``same``): an exact tie, decided by index."""
    k = int(np.argmax(v))
    if np.isnan(v[k]):
        return k, bool(t[k] == 0) and not np.isnan(v[:k]).any()
    with np.errstate(invalid="ignore"):
        gap = v[k] - v
        tt = t[k] + t
        ok = (gap > MARGIN * tt) | ((v == v[k]) & (tt == 0))
        if same is not None and same[k]:
            ok |= same
    ok[k] = True
    return k, bool(ok.all())


def replay(table, row_ptr, cols, vals, labels, *, algo, binary, C=0.0, cost=None, tol=None, fp32=True):
    """Replay one launch.  ``table`` ``[F, L]``: the rows as the kernel reads them (float64 copies of the fp32
    table; ``tol`` their bounds, default 0).  ``row_ptr``, ``cols``, ``vals``, ``labels``: the CSR batch
    (``labels`` +-1 for binary, a class index, or ``UNLABELLED``).  ``cost`` ``[L, L]`` or ``None``.

    Returns a :class:`Result`: ``table`` and ``tol`` after the launch; ``pred``; ``loss`` and ``tol_loss`` (NaN
    where the kernel leaves the output untouched); ``bad`` (the example raises the non-finite flag); ``decided``
    (its binary sign, prediction and ML ``q`` are clear of their bounds); ``updated``."""
    W = np.array(table, dtype=np.float64)
    L = W.shape[1]
    T = np.zeros_like(W) if tol is None else np.array(tol, dtype=np.float64)
    if binary and L != 1:
        raise ValueError("a binary model has one column")
    if algo not in ALGOS:
        raise ValueError(f"unknown algorithm {algo!r}")
    vals = np.asarray(vals, dtype=np.float64)
    cols = np.asarray(cols, dtype=np.int64)
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    n = len(labels)
    if fp32:
        C = float(np.float32(C))
        cost = None if cost is None else np.asarray(cost, dtype=np.float32).astype(np.float64)
    cm = np.where(np.eye(L, dtype=bool), 0.0, 1.0) if cost is None else np.asarray(cost, dtype=np.float64)
    sq = np.float32(np.sqrt(cm)).astype(np.float64) if fp32 else np.sqrt(cm)
    if algo == "PAII":
        r = float(np.float32(1) / (np.float32(2) * np.float32(C))) if fp32 else 1.0 / (2.0 * C)
    pred = np.zeros(n, dtype=np.int64)
    loss = np.full(n, np.nan)
    tol_loss = np.full(n, np.nan)
    bad = np.zeros(n, dtype=bool)
    clear = np.ones(n, dtype=bool)
    updated = np.zeros(n, dtype=bool)

    def ov(v):  # fp32 overflow
        if not fp32:
            return v
        with np.errstate(over="ignore", invalid="ignore"):
            f = np.float32(v).astype(np.float64)
        return np.where(np.isinf(f) & np.isfinite(v), f, v)

    def ftz(v):
        return np.where(np.abs(v) < FLT_MIN, 0.0, v) if fp32 else v

    def dsum(terms, x, tw):
        """column sums of ``terms`` [k, m] and their bound (any order)"""
        with np.errstate(invalid="ignore", over="ignore"):
            s = ov(terms.sum(0))
            fin = np.isfinite(terms)
            a = np.where(fin, np.abs(terms), 0.0)
            k = ((terms != 0) & fin).sum(0)
            inexact = fin & (np.float32(terms) != terms)
            t = (np.maximum(k - 1, 0) * EPS * a.sum(0) + EPS * np.where(inexact, a, 0.0).sum(0)
                 + (np.abs(x)[:, None] * tw).sum(0))
        return s, np.where(np.isfinite(t), t, 0.0)

    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for ex in range(n):
            b, e = int(row_ptr[ex]), int(row_ptr[ex + 1])
            idx, x = cols[b:e], vals[b:e]
            label = int(labels[ex])
            d, td = dsum(x[:, None] * W[idx], x, T[idx])
            sqx = (np.float32(x) * np.float32(x)).astype(np.float64) if fp32 else x * x
            n2, tn2 = dsum(sqx[:, None], x * 0, np.zeros((e - b, 1)))
            n2, tn2 = float(n2[0]), float(tn2[0])
            if binary:
                pred[ex] = int(d[0] > 0)
                clear[ex] = bool(td[0] == 0 or abs(d[0]) > MARGIN * td[0])
            else:
                pred[ex], clear[ex] = first_argmax(d, td)
            if label == UNLABELLED or e == b or not n2 > 0:
                continue
            updated[ex] = True
            if binary or algo in ("PA", "PAI", "PAII"):
                y = np.full(L, float(label)) if binary else np.where(np.arange(L) == label, 1.0, -1.0)
                h = ov(1.0 - y * d)
                th = _rnd(h, td)
                l = np.maximum(0.0, h)
                tl = np.where(h > -th, th, 0.0)
                if algo == "PA":
                    tau, ttau = _div(l, tl, n2, tn2)
                elif algo == "PAI":
                    qt, tq = _div(l, tl, n2, tn2)
                    tau = np.minimum(C, qt)
                    ttau = np.where(qt - tq < C, tq, 0.0)
                else:
                    den = n2 + r
                    tau, ttau = _div(l, tl, den, _rnd(den, tn2))
                mult, tmult = tau * y, ttau
                if L == 1:
                    loss[ex], tol_loss[ex] = l[0], tl[0]
            else:
                if algo == "ML":
                    # every v_i subtracts the same d_label, so its error cancels between rivals: the bound of
                    # a comparison keeps td_i and the roundings, and identical (d_i, s_i) tie exactly
                    fin = lambda a: np.where(np.isfinite(a), np.abs(a), 0.0)
                    t1 = ov(d - d[label])
                    tt1 = _rnd(t1, td) if td[label] == 0 else td + EPS * fin(t1)
                    tt1[label] = 0.0                      # d_label - d_label is exactly 0 (or NaN)
                    v = ov(t1 + sq[label])
                    tv = _rnd(v, tt1) if td[label] == 0 else tt1 + EPS * fin(v)
                    tv[label] = _rnd(v[label], 0.0)       # 0 + sqrt(c(label, label))
                    k = int(np.argmax(v))
                    q, ok = first_argmax(v, tv, same=(d == d[k]) & (td == 0) & (sq[label] == sq[label, k]))
                    clear[ex] &= ok
                else:
                    q = int(pred[ex])
                if q == label:
                    continue
                t1 = ov(d[q] - d[label])
                tt1 = _rnd(t1, td[q] + td[label])
                lq = ov(t1 + sq[label, q])
                tlq = _rnd(lq, tt1)
                loss[ex], tol_loss[ex] = lq, tlq
                tau, ttau = _div(lq, tlq, 2.0 * n2, 2.0 * tn2)
                mult, tmult = np.zeros(L), np.zeros(L)
                mult[label], mult[q] = tau, -tau
                tmult[label] = tmult[q] = ttau
            chunk = np.arange(L) // 4
            for j in range(b, e):
                f, xj = int(cols[j]), vals[j]
                p = ov(xj * mult)
                tp = _rnd(p, np.abs(xj) * tmult)
                nz = (np.float32(p) != 0) if fp32 else (p != 0)
                live = np.bincount(chunk, weights=nz, minlength=chunk[-1] + 1) > 0
                mag = np.bincount(chunk, weights=np.abs(p), minlength=chunk[-1] + 1)
                if (live & ~(mag <= FLAG_LIMIT)).any():
                    bad[ex] = True
                s = live[chunk]                            # every column of a pushed chunk
                w = ftz(ov(W[f, s] + ftz(p[s])))
                T[f, s] = _rnd(w, T[f, s] + tp[s])
                W[f, s] = w
    T = np.where(np.isfinite(T), T, 0.0)
    return Result(table=W, tol=T, pred=pred, loss=loss, tol_loss=tol_loss, bad=bad, decided=clear, updated=updated)
