"""fp64 replay of one ``fps_ffm_step`` launch (ops/csrc/fps_ffm.cu, DESIGN §2.16) with a first-order bound on every
table element.  CPU only: the GPU suite feeds it the fp32 table as the kernel reads it.

Row ``i`` of the table is ``[w_i | 0 0 0 | V_i,0 | .. | V_i,F-1]``, slab ``f`` at columns ``4 + f kp .. + k``,
``kp = round_up(k, 4)``; columns ``[k, kp)`` of a slab are padding.  Semantics mirrored from the kernel:
- Examples run in CSR order, each reading the rows as the earlier examples of the launch left them.  (The kernel
  races the examples of one launch; with no slab and no ``w`` pushed twice that race has this one result.)  Every
  example reads ``w0`` as it was before the launch.  ``stale=True`` lets every example read the rows as they were
  before the launch, the other end of the race; ``repull=True`` is the end of the race inside one example.
- An example's end is clamped to ``nnz``; an entry whose feature is outside ``[0, num_features)`` or whose field is
  outside ``[0, num_fields)`` is skipped and sets ``bad_id``.  ``vals=None`` is one-hot.
- The pairs of an example are its kept entries ``a < b`` in CSR order; ``pred`` is ``yhat`` from before the
  example's own update.  A NaN label (or ``predict_only``) pushes nothing and is not counted.
- Every delta uses the slabs as the example pulled them.  ``w`` takes a scalar ``red.add.f32``, each slab a
  ``red.add.v4.f32`` (padding receives 0); both flush subnormal inputs and results to zero.
- After the launch, ``w0 += fl(-lr * fl(sum g / n_labelled))`` when ``bias`` and at least one example was labelled.

Error model (first order, EPS = 2^-24, FMA contraction allowed, any summation order): a sum of ``N`` terms is off by
at most ``N EPS sum|terms|``; ``yhat`` counts every pair and entry of the example and the warp reduction; sigmoid and
softplus add ``4 EPS``; each product, difference and push adds one rounding of its magnitude.  ``breaks`` switches one
rule off (the sensitivity checks of the GPU suite): ``"field_unaware"`` pairs ``V[i_a, f_a]`` with ``V[i_b, f_b]``,
``"self_pairs"`` takes ``a <= b``, ``"no_xx"`` drops ``x_a x_b`` from the slab deltas, ``"w0_per_example"`` steps
``w0`` after every example, ``"reg_sign"`` flips the regularisation's sign in the deltas.

AdaGrad (DESIGN §2.17): ``acc`` / ``acc_tol`` are ``H`` and its bounds, as in tests/fm_ref.py, whose rule, error
model and ``ADAGRAD_BREAKS`` apply to ``w`` and to both slabs of every pair; ``acc=None`` is plain SGD.  ``stale``
and ``repull`` apply to ``H`` as to the slabs: a slab pushed twice inside one example reads an ``H`` that may or may
not hold the earlier pair's ``gam^2`` (PTX orders a reduction only before the same thread's own later loads)."""
import math

import numpy as np

from tests.fm_ref import ADAGRAD_BREAKS, adagrad

EPS = 2.0 ** -24
MARGIN = 2.0
FLT_MIN = 2.0 ** -126
BREAKS = ("field_unaware", "self_pairs", "no_xx", "w0_per_example", "reg_sign")


def kpad(k):
    return 4 * -(-int(k) // 4)


def stride(num_fields, k):
    return 4 + int(num_fields) * kpad(k)


def lanes(k):
    """Q, the lanes per pair ``ffm_dispatch`` launches for ``k`` factors: kp / 4 rounded up to a power of two."""
    return 1 << (kpad(k) // 4 - 1).bit_length()


class Result(dict):
    __getattr__ = dict.__getitem__


def _pairs(m, breaks):
    a, b = np.triu_indices(m, 0 if breaks == "self_pairs" else 1)
    return a, b


def _slab_cols(f, k, kp):
    return 4 + np.asarray(f)[:, None] * kp + np.arange(k)[None, :]


def replay(table, row_ptr, cols, fields, vals, labels, *, num_features, num_fields, k, loss="logistic", lr=0.05,
           reg_linear=0.0, reg_factors=0.0, bias=True, predict_only=False, tol=None, fp32=True, breaks=None,
           stale=False, repull=False, acc=None, acc_tol=None):
    """Replay one launch.  ``table`` ``[num_features + 1, stride]``: the rows as the kernel reads them (float64
    copies of the fp32 table; ``tol`` their bounds, default 0).  Returns a :class:`Result` with ``table`` and
    ``tol`` after the launch, ``pred`` / ``tol_pred``, ``g``, ``loss_sum``, ``labelled``, ``w0_delta`` and
    ``bad_id``.  ``repull=True`` computes every push of an example from the rows as its earlier pushes left them
    (the kernel's pass 2 re-pulls; with a slab pushed twice in one example it lies between the two ends).  ``acc``
    / ``acc_tol``: AdaGrad's ``H`` and its bounds, as in tests/fm_ref.py; the result's ``acc`` / ``tol_acc`` are
    ``None`` without them."""
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
    nf, F, k = int(num_features), int(num_fields), int(k)
    kp = kpad(k)
    if W.shape[1] != stride(F, k):
        raise ValueError(f"rows of {W.shape[1]} floats, want {stride(F, k)}")
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    cols = np.asarray(cols, dtype=np.int64)
    fields = np.asarray(fields, dtype=np.int64)
    nnz = len(cols)
    vals = np.ones(nnz) if vals is None else np.asarray(vals, dtype=np.float64)
    n = len(row_ptr) - 1
    labels = np.full(n, np.nan) if labels is None else np.asarray(labels, dtype=np.float64)
    lr, rl, rv = (float(np.float32(v)) for v in (lr, reg_linear, reg_factors)) if fp32 else (lr, reg_linear,
                                                                                            reg_factors)
    if breaks == "reg_sign":
        rl, rv = -rl, -rv
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
            idx, fld, x = cols[b:e], fields[b:e], vals[b:e]
            ok = (idx >= 0) & (idx < nf) & (fld >= 0) & (fld < F)
            bad_id |= not ok.all()
            idx, fld, x = idx[ok], fld[ok], x[ok]
            m = len(idx)
            pa, pb = _pairs(m, breaks)
            ra, rb = idx[pa], idx[pb]
            # the slab each side of a pair reads and pushes: V[i_a, f_b] and V[i_b, f_a]
            fa, fb = (fld[pa], fld[pb]) if breaks == "field_unaware" else (fld[pb], fld[pa])
            ca, cb = _slab_cols(fa, k, kp), _slab_cols(fb, k, kp)
            VA, tVA = R[ra[:, None], ca], RT[ra[:, None], ca]
            VB, tVB = R[rb[:, None], cb], RT[rb[:, None], cb]
            w, tw = R[idx, 0], RT[idx, 0]
            xx = x[pa] * x[pb]
            dots = (VA * VB).sum(1)
            yhat = w0 + (x * w).sum() + (xx * dots).sum()
            A = abs(w0) + np.abs(x * w).sum() + (np.abs(xx) * (np.abs(VA) * np.abs(VB)).sum(1)).sum()
            N = len(pa) + m + kp + 16
            ty = (tw0 + (np.abs(x) * tw).sum() + N * EPS * A
                  + (np.abs(xx)[:, None] * (np.abs(VB) * tVA + np.abs(VA) * tVB)).sum())
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
            # every delta from the rows as the example pulled them
            gx = g * x
            dw = -lr * (gx + rl * w)
            tdw = (lr * (np.abs(x) * tg + abs(rl) * tw) + 3 * EPS * lr * (np.abs(gx) + np.abs(rl * w))
                   + EPS * np.abs(dw))
            c = np.full(len(pa), g) if breaks == "no_xx" else g * xx
            tc = (np.zeros(len(pa)) if breaks == "no_xx" else np.abs(xx)) * tg + 2 * EPS * np.abs(c)
            dA = -lr * (c[:, None] * VB + rv * VA)
            dB = -lr * (c[:, None] * VA + rv * VB)
            tdA = (lr * (tc[:, None] * np.abs(VB) + np.abs(c)[:, None] * tVB + abs(rv) * tVA)
                   + 3 * EPS * lr * (np.abs(c[:, None] * VB) + np.abs(rv * VA)) + EPS * np.abs(dA))
            tdB = (lr * (tc[:, None] * np.abs(VA) + np.abs(c)[:, None] * tVA + abs(rv) * tVB)
                   + 3 * EPS * lr * (np.abs(c[:, None] * VA) + np.abs(rv * VB)) + EPS * np.abs(dB))
            rows = np.concatenate([ra, rb])
            scol = np.concatenate([ca, cb])
            D, TD = np.concatenate([dA, dB]), np.concatenate([tdA, tdB])
            keys = rows * (F + 1) + (scol[:, 0] - 4) // kp if len(rows) else rows
            if ada:
                # the brackets without -lr, each with H as the example pulled it
                gw = gx + rl * w
                tgw = np.abs(x) * tg + abs(rl) * tw + 2 * EPS * (np.abs(gx) + np.abs(rl * w))
                dw, tdw, dHw, tdHw = adagrad(gw, tgw, RH[idx, 0], RTH[idx, 0], lr, breaks, gx)
                gA, gB = c[:, None] * VB + rv * VA, c[:, None] * VA + rv * VB
                tgA = (tc[:, None] * np.abs(VB) + np.abs(c)[:, None] * tVB + abs(rv) * tVA
                       + 2 * EPS * (np.abs(c[:, None] * VB) + np.abs(rv * VA)))
                tgB = (tc[:, None] * np.abs(VA) + np.abs(c)[:, None] * tVA + abs(rv) * tVB
                       + 2 * EPS * (np.abs(c[:, None] * VA) + np.abs(rv * VB)))
                G_, TG = np.concatenate([gA, gB]), np.concatenate([tgA, tgB])
                GL = np.concatenate([c[:, None] * VB, c[:, None] * VA])
                D, TD, DH, TDH = adagrad(G_, TG, RH[rows[:, None], scol], RTH[rows[:, None], scol], lr, breaks, GL)

            def push(Wt, Tt, i, cc, d, td):
                new = ftz(Wt[i, cc] + ftz(d))
                Tt[i, cc] = Tt[i, cc] + td + EPS * np.abs(new)
                Wt[i, cc] = new

            if repull:
                # the other end of the race inside the example: each entry and pair reads its rows (and H) as the
                # pushes before it left them
                for j in range(m):
                    i = int(idx[j])
                    if ada:
                        d, td, dh, tdh = adagrad(gx[j] + rl * W[i, 0], tgw[j], Hm[i, 0], TH[i, 0], lr, breaks, gx[j])
                        push(W, T, i, 0, float(d), float(td))
                        push(Hm, TH, i, 0, float(dh), float(tdh))
                    else:
                        push(W, T, i, 0, -lr * (gx[j] + rl * W[i, 0]), tdw[j])
                for j in range(len(pa)):
                    va, vb = W[ra[j], ca[j]], W[rb[j], cb[j]]
                    if ada:
                        for i, cc, gm, tgm, gl in ((ra[j], ca[j], c[j] * vb + rv * va, tgA[j], c[j] * vb),
                                                   (rb[j], cb[j], c[j] * va + rv * vb, tgB[j], c[j] * va)):
                            d, td, dh, tdh = adagrad(gm, tgm, Hm[i, cc], TH[i, cc], lr, breaks, gl)
                            push(W, T, i, cc, d, td)
                            push(Hm, TH, i, cc, dh, tdh)
                    else:
                        for i, cc, d, td in ((ra[j], ca[j], -lr * (c[j] * vb + rv * va), tdA[j]),
                                             (rb[j], cb[j], -lr * (c[j] * va + rv * vb), tdB[j])):
                            push(W, T, i, cc, d, td)
            elif len(np.unique(idx)) == m and len(np.unique(keys)) == len(keys):
                push(W, T, idx, 0, dw, tdw)
                push(W, T, rows[:, None], scol, D, TD)
                if ada:
                    push(Hm, TH, idx, 0, dHw, tdHw)
                    push(Hm, TH, rows[:, None], scol, DH, TDH)
            else:
                for j in range(m):   # a repeated feature or slab: its pushes land one after the other
                    push(W, T, int(idx[j]), 0, dw[j], tdw[j])
                    if ada:
                        push(Hm, TH, int(idx[j]), 0, dHw[j], tdHw[j])
                for j in range(len(rows)):
                    push(W, T, int(rows[j]), scol[j], D[j], TD[j])
                    if ada:
                        push(Hm, TH, int(rows[j]), scol[j], DH[j], TDH[j])
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


def objective(table, cols, fields, vals, y, *, num_features, num_fields, k, loss, reg_linear=0.0, reg_factors=0.0,
              bias=True, xp=np):
    """The loss of one example plus the lazy L2 of what it touches: ``l(yhat, y) + sum_a reg_linear / 2 w_a^2 +
    sum_{a<b} reg_factors / 2 (|V[i_a, f_b]|^2 + |V[i_b, f_a]|^2)``.  One example's update in :func:`replay`
    (``fp32=False``) is ``-lr`` times this function's gradient.  ``xp``: numpy or torch."""
    nf, kp = int(num_features), kpad(k)
    cols_n, fields_n = np.asarray(cols), np.asarray(fields)
    pa, pb = np.triu_indices(len(cols_n), 1)
    ra, rb = cols_n[pa], cols_n[pb]
    ca, cb = _slab_cols(fields_n[pb], k, kp), _slab_cols(fields_n[pa], k, kp)
    if xp is not np:
        pa, pb, ra, rb, ca, cb, cols_n = (xp.as_tensor(v) for v in (pa, pb, ra, rb, ca, cb, cols_n))
    VA, VB = table[ra[:, None], ca], table[rb[:, None], cb]
    w = table[cols_n, 0]
    xx = vals[pa] * vals[pb]
    w0 = table[nf, 0] if bias else 0.0
    yhat = w0 + (vals * w).sum() + (xx * (VA * VB).sum(1)).sum()
    if loss == "logistic":
        l = xp.log1p(xp.exp(-xp.abs(yhat))) + xp.maximum(yhat, yhat * 0) - y * yhat
    else:
        l = 0.5 * (yhat - y) ** 2
    return l + 0.5 * reg_linear * (w * w).sum() + 0.5 * reg_factors * ((VA * VA).sum() + (VB * VB).sum())
