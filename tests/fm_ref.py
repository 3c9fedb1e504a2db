"""fp64 replay of one ``fps_fm_step`` launch (ops/csrc/fps_fm.cu, DESIGN §2.15) with a first-order bound on every
table element.  CPU only: the GPU suite feeds it the fp32 table as the kernel reads it.

Semantics mirrored from the kernel:
- Examples run in CSR order, each reading the feature rows as the earlier examples of the launch left them.  (The
  kernel races the examples of one launch; with no feature shared between two entries that race has this one
  result.)  Every example reads ``w0`` as it was before the launch.
- An example's end is clamped to ``nnz``; an entry whose id is outside ``[0, num_features)`` is skipped and sets
  ``bad_id``.  ``vals=None`` is one-hot (every x = 1).
- ``pred`` is ``yhat`` from before the example's own update.  A NaN label (or ``predict_only``) pushes nothing and
  is not counted.
- Each entry's delta uses the row as the example pulled it; the entries of an example push in CSR order.  Every
  16-byte chunk of the row is pushed (padding with 0), and ``red.add.f32`` flushes subnormal inputs and results
  to zero on every column of a pushed chunk, as tests/pa_ref.py models it.
- After the launch, ``w0 += fl(-lr * fl(sum g / n_labelled))`` when ``bias`` and at least one example was
  labelled.

Error model (first order, EPS = 2^-24, FMA contraction allowed, any summation order): a sum of ``N`` terms is off
by at most ``N EPS sum|terms|``; ``yhat`` counts the per-lane sums (``4 VPL`` columns per entry) and the group
reduction; sigmoid and softplus add ``4 EPS``; each product, difference and push adds one rounding of its
magnitude.  ``breaks`` switches one rule off (the sensitivity checks of the GPU suite): ``"no_xv"`` drops the
``- x v`` term, ``"no_half"`` the 1/2, ``"w0_per_example"`` steps ``w0`` after every example, ``"col0_factor"``
treats column 0 as one more factor, ``"reg_sign"`` flips the regularisation's sign in the delta.

AdaGrad (DESIGN §2.17): ``acc`` holds ``H = G - 1`` per element in the table's layout; ``acc=None`` is plain SGD.
Every element an entry updates takes ``gam`` (the bracket the SGD delta scales by ``-lr``), its ``H`` as the example
pulled it, and ``theta += -lr gam / sqrt(1 + H + gam^2)``, ``H += gam^2``, both pushes flushing subnormals like the
table's.  The kernel's ``sqrtf`` and division are IEEE round-to-nearest (0.5 ulp each, one ``EPS`` of their
results), and the bound carries ``H``'s own ``acc_tol`` through them.  ``ADAGRAD_BREAKS`` (apart from ``BREAKS``,
which the SGD suites run, and refused without ``acc``): ``"acc_after"`` divides by ``sqrt(1 + H)``, ``"no_init"`` by
``sqrt(H + gam^2)``, ``"acc_abs"`` adds ``|gam|`` to ``H``, ``"acc_unregularised"`` adds the square of the loss term
of ``gam`` only."""
import math

import numpy as np

EPS = 2.0 ** -24
MARGIN = 2.0
FLT_MIN = 2.0 ** -126
FLAG_LIMIT = 3.0e38
MAX_DIM = 512
BREAKS = ("no_xv", "no_half", "w0_per_example", "col0_factor", "reg_sign")
ADAGRAD_BREAKS = ("acc_after", "no_init", "acc_abs", "acc_unregularised")


def geometry(stride):
    """(LPR, VPL, TB) that ``fm_dispatch`` launches for rows of ``stride`` floats."""
    nvec = stride // 4
    if stride % 4 or nvec < 1 or stride > MAX_DIM:
        raise ValueError(f"no kernel for stride {stride}")
    if nvec <= 32:
        return 1 << (nvec - 1).bit_length(), 1, 8
    return 32, -(-nvec // 32), 4


def rungs():
    """Every (LPR, VPL) rung of the dispatch ladder, with the k at and just above each boundary."""
    return sorted({geometry(4 * -(-(1 + k) // 4))[:2] for k in range(MAX_DIM)})


class Result(dict):
    __getattr__ = dict.__getitem__


def adagrad(gam, tgam, H, tH, lr, breaks=None, gam_loss=None):
    """libffm's AdaGrad step of every element with bracket ``gam`` (bound ``tgam``) and accumulator ``H`` (bound
    ``tH``): ``(delta, tol_delta, dH, tol_dH)``.  Elements with ``gam == 0`` (padding) take exact zeros.
    ``gam_loss``: the loss term of ``gam``, for the ``"acc_unregularised"`` break."""
    gam, tgam, H, tH = (np.asarray(v, dtype=np.float64) for v in (gam, tgam, H, tH))
    gg = gam * gam
    tgg = 2 * np.abs(gam) * tgam + EPS * gg
    if breaks == "no_init":
        S = H + gg
    elif breaks == "acc_after":
        S = 1.0 + H
    else:
        S = 1.0 + H + gg
    tS = tH + tgg + 2 * EPS * np.abs(S)
    zero = gam == 0
    with np.errstate(divide="ignore", invalid="ignore"):
        sq = np.sqrt(np.where(zero, 1.0, S))
        num = lr * gam
        D = np.where(zero, 0.0, -num / sq)
        tsq = tS / (2 * sq) + EPS * sq                  # sqrtf: the carried bound, then one rounding
        tD = np.where(zero, 0.0, (lr * tgam + EPS * np.abs(num)) / sq + np.abs(num) * tsq / (sq * sq)
                      + EPS * np.abs(D))                # the product, the carried bounds, the division's rounding
    if breaks == "acc_abs":
        dH = np.abs(gam)
    elif breaks == "acc_unregularised":
        dH = np.asarray(gam_loss, dtype=np.float64) ** 2
    else:
        dH = gg
    return D, tD, dH, tgg


def replay(table, row_ptr, cols, vals, labels, *, num_features, dim, loss="logistic", lr=0.05, reg_linear=0.0,
           reg_factors=0.0, bias=True, predict_only=False, tol=None, fp32=True, breaks=None, stale=False, acc=None,
           acc_tol=None, repull=False):
    """Replay one launch.  ``table`` ``[num_features + 1, stride]``: the rows as the kernel reads them (float64
    copies of the fp32 table; ``tol`` their bounds, default 0).  Returns a :class:`Result` with ``table`` and
    ``tol`` after the launch, ``pred`` / ``tol_pred``, ``g``, ``loss_sum``, ``labelled``, ``w0_delta`` and
    ``bad_id``.  ``stale=True`` lets every example read the rows as they were before the launch (all examples
    at once, the other end of the race from CSR order).  ``acc``: AdaGrad's ``H`` as the kernel reads it (same shape
    as ``table``; ``acc_tol`` its bounds); the result's ``acc`` / ``tol_acc`` are ``H`` after the launch (``None``
    without ``acc``: plain SGD).  ``repull=True`` is the end of the race inside one example: an entry whose feature
    an earlier entry of the example pushed reads that row (and its ``H``) as the push left it, as the kernel's pass
    2 may when the two entries fall in different row blocks."""
    if breaks is not None and breaks not in BREAKS + (ADAGRAD_BREAKS if acc is not None else ()):
        raise ValueError(f"unknown break {breaks!r}")
    W = np.array(table, dtype=np.float64)
    T = np.zeros_like(W) if tol is None else np.array(tol, dtype=np.float64)
    R, RT = (W.copy(), T.copy()) if stale else (W, T)   # the rows each example reads
    ada = acc is not None
    if ada:
        Hm = np.array(acc, dtype=np.float64)
        TH = np.zeros_like(Hm) if acc_tol is None else np.array(acc_tol, dtype=np.float64)
        RH, RTH = (Hm.copy(), TH.copy()) if stale else (Hm, TH)
    nf, stride = int(num_features), W.shape[1]
    _, vpl, _ = geometry(stride)
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    cols = np.asarray(cols, dtype=np.int64)
    nnz = len(cols)
    vals = np.ones(nnz) if vals is None else np.asarray(vals, dtype=np.float64)
    n = len(row_ptr) - 1
    labels = np.full(n, np.nan) if labels is None else np.asarray(labels, dtype=np.float64)
    lr, rl, rv = (float(np.float32(v)) for v in (lr, reg_linear, reg_factors)) if fp32 else (lr, reg_linear,
                                                                                            reg_factors)
    if breaks == "reg_sign":
        rl, rv = -rl, -rv
    f0 = 0 if breaks == "col0_factor" else 1           # first factor column
    half = 1.0 if breaks == "no_half" else 0.5
    w0 = W[nf, 0] if bias else 0.0
    tw0 = T[nf, 0] if bias else 0.0
    pred = np.zeros(n)
    tol_pred = np.zeros(n)
    gs = np.full(n, np.nan)
    bad_id = False
    loss_sum, labelled, sum_g, sum_tg = 0.0, 0, 0.0, 0.0

    def ftz(v):
        return np.where(np.abs(v) < FLT_MIN, 0.0, v) if fp32 else v

    with np.errstate(over="ignore", invalid="ignore"):
        for ex in range(n):
            e = min(int(row_ptr[ex + 1]), nnz)
            b = min(max(int(row_ptr[ex]), 0), e)
            idx, x = cols[b:e], vals[b:e]
            ok = (idx >= 0) & (idx < nf)
            bad_id |= not ok.all()
            idx, x = idx[ok], x[ok]
            m = len(idx)
            w, tw = R[idx, 0], RT[idx, 0]
            V, tV = R[idx, f0:dim], RT[idx, f0:dim]
            xv = x[:, None] * V
            s = xv.sum(0)
            ts = m * EPS * np.abs(xv).sum(0) + (np.abs(x)[:, None] * tV).sum(0)
            sq = (xv * xv).sum()
            lin = (x * w).sum()
            yhat = w0 + lin + half * ((s * s).sum() - sq)
            A = abs(w0) + np.abs(x * w).sum() + half * ((s * s).sum() + sq)
            N = m * 4 * vpl + 4 * vpl + 16
            ty = (tw0 + (np.abs(x) * tw).sum() + N * EPS * A + (2 * np.abs(s) * ts).sum()
                  + (2 * np.abs(xv) * np.abs(x)[:, None] * tV).sum())
            pred[ex], tol_pred[ex] = yhat, ty
            y = labels[ex]
            if predict_only or y != y:
                continue
            if loss == "logistic":
                g = 1.0 / (1.0 + math.exp(-yhat)) - y if yhat > -700 else -y
                tg = 0.25 * ty + 4 * EPS
                loss_sum += max(yhat, 0.0) + math.log1p(math.exp(-abs(yhat))) - y * yhat
            else:
                g = yhat - y
                tg = ty + EPS * (abs(yhat) + abs(y))
                loss_sum += g * g
            gs[ex] = g
            labelled += 1
            sum_g += g
            sum_tg += tg
            # every entry's delta from the rows as the example pulled them
            gx = g * x
            D = np.zeros((m, stride))
            TD = np.zeros((m, stride))
            if breaks != "col0_factor":
                D[:, 0] = -lr * (gx + rl * w)
                TD[:, 0] = (lr * (np.abs(x) * tg + abs(rl) * tw) + 3 * EPS * lr * (np.abs(gx) + np.abs(rl * w))
                            + EPS * np.abs(D[:, 0]))
            t1 = s[None, :] - (0.0 if breaks == "no_xv" else xv)
            tt1 = ts[None, :] + np.abs(x)[:, None] * tV + EPS * (np.abs(xv) + np.abs(t1))
            dv = -lr * (gx[:, None] * t1 + rv * V)
            D[:, f0:dim] = dv
            TD[:, f0:dim] = (lr * (np.abs(x)[:, None] * tg * np.abs(t1) + np.abs(gx)[:, None] * tt1 + abs(rv) * tV)
                             + 3 * EPS * lr * (np.abs(gx[:, None] * t1) + np.abs(rv * V)) + EPS * np.abs(dv))
            if ada:
                # the same brackets without -lr, and H as the example pulled it
                gam, tgam, gl = np.zeros((m, stride)), np.zeros((m, stride)), np.zeros((m, stride))
                if breaks != "col0_factor":
                    gam[:, 0], gl[:, 0] = gx + rl * w, gx
                    tgam[:, 0] = np.abs(x) * tg + abs(rl) * tw + 2 * EPS * (np.abs(gx) + np.abs(rl * w))
                gam[:, f0:dim], gl[:, f0:dim] = gx[:, None] * t1 + rv * V, gx[:, None] * t1
                tgam[:, f0:dim] = (np.abs(x)[:, None] * tg * np.abs(t1) + np.abs(gx)[:, None] * tt1 + abs(rv) * tV
                                   + 2 * EPS * (np.abs(gx[:, None] * t1) + np.abs(rv * V)))
                D, TD, DH, TDH = adagrad(gam, tgam, RH[idx], RTH[idx], lr, breaks, gl)
            if len(np.unique(idx)) == m:
                new = ftz(W[idx] + ftz(D))
                T[idx] = T[idx] + TD + EPS * np.abs(new)
                W[idx] = new
                if ada:
                    new = ftz(Hm[idx] + ftz(DH))
                    TH[idx] = TH[idx] + TDH + EPS * np.abs(new)
                    Hm[idx] = new
            else:
                for j in range(m):   # a repeated feature: its pushes land in CSR order
                    i = int(idx[j])
                    if repull and i in idx[:j]:
                        v = W[i, f0:dim]
                        bracket, loss_part = np.zeros(stride), np.zeros(stride)
                        if breaks != "col0_factor":
                            loss_part[0] = gx[j]
                            bracket[0] = gx[j] + rl * W[i, 0]
                        loss_part[f0:dim] = gx[j] * (s - (0.0 if breaks == "no_xv" else x[j] * v))
                        bracket[f0:dim] = loss_part[f0:dim] + rv * v
                        if ada:
                            D[j], TD[j], DH[j], TDH[j] = adagrad(bracket, tgam[j], Hm[i], TH[i], lr, breaks,
                                                                 loss_part)
                        else:
                            D[j] = -lr * bracket
                    new = ftz(W[i] + ftz(D[j]))
                    T[i] = T[i] + TD[j] + EPS * np.abs(new)
                    W[i] = new
                    if ada:
                        new = ftz(Hm[i] + ftz(DH[j]))
                        TH[i] = TH[i] + TDH[j] + EPS * np.abs(new)
                        Hm[i] = new
            if breaks == "w0_per_example" and bias:
                w0 = float(ftz(w0 + ftz(-lr * g)))
                tw0 = tw0 + lr * tg + 2 * EPS * abs(w0)
    w0_delta = 0.0
    if bias and labelled:
        if breaks == "w0_per_example":
            w0_delta = w0 - W[nf, 0]
            W[nf, 0], T[nf, 0] = w0, tw0
        else:
            mean = sum_g / labelled
            w0_delta = float(np.float32(-lr * float(np.float32(mean)))) if fp32 else -lr * mean
            new = float(ftz(W[nf, 0] + ftz(w0_delta)))
            T[nf, 0] = T[nf, 0] + lr * sum_tg / labelled + 2 * EPS * abs(w0_delta) + EPS * abs(new)
            W[nf, 0] = new
    T = np.where(np.isfinite(T), T, 0.0)
    if ada:
        TH = np.where(np.isfinite(TH), TH, 0.0)
    return Result(table=W, tol=T, pred=pred, tol_pred=tol_pred, g=gs, loss_sum=loss_sum, labelled=labelled,
                  w0_delta=w0_delta, bad_id=bad_id, acc=Hm if ada else None, tol_acc=TH if ada else None)


def objective(table, cols, vals, y, *, num_features, dim, loss, reg_linear=0.0, reg_factors=0.0, bias=True, xp=np):
    """The loss of one example plus the lazy L2 of the rows its entries touch (once per entry):
    ``l(yhat, y) + sum_j (reg_linear / 2 w_j^2 + reg_factors / 2 |v_j|^2)``.  One example's update in
    :func:`replay` (``fp32=False``) is ``-lr`` times this function's gradient.  ``xp``: numpy or torch."""
    nf = int(num_features)
    idx = cols
    w = table[idx, 0]
    V = table[idx, 1:dim]
    xv = vals[:, None] * V
    s = xv.sum(0)
    w0 = table[nf, 0] if bias else 0.0
    yhat = w0 + (vals * w).sum() + 0.5 * ((s * s).sum() - (xv * xv).sum())
    if loss == "logistic":
        l = xp.log1p(xp.exp(-xp.abs(yhat))) + xp.maximum(yhat, yhat * 0) - y * yhat
    else:
        l = 0.5 * (yhat - y) ** 2
    return l + 0.5 * reg_linear * (w * w).sum() + 0.5 * reg_factors * (V * V).sum()
