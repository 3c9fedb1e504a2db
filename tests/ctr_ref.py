"""fp64 replay of one ``fps_ctr_step`` launch (ops/csrc/fps_ctr.cu: the fused wide-&-deep tower and its apply
kernel) with a first-order bound on every value it returns.  CPU only: the GPU suite feeds it the fp32 state the
kernel reads.

Semantics mirrored from the kernel, for ``B`` examples of ``F`` pulled rows each (``E`` embedding floats, then the
wide weight in column ``E``, then padding up to the row stride):
- ``x_e`` is the ``F * E`` embedding floats of example ``e``; ``pre = b1 + W1^T x``, ``h = relu(pre)``,
  ``logit = w2 . h + b2 + sum_f wide_f``, ``p = sigmoid(logit)``, loss ``max(z, 0) - z y + log1p(exp(-|z|))``.
- Backward with ``d = p - y``: ``dh = d w2`` where ``pre > 0`` and exactly 0 elsewhere (ReLU'(0) = 0);
  ``gW1 = sum_e x dh``, ``gb1 = sum_e dh``, ``gw2 = sum_e d h``, ``gb2 = sum_e d``; the pushed row gradients are
  ``-lr W1 dh`` on the embedding columns, ``-lr d`` on the wide column and exactly 0 on the padding columns.
- The apply step is SGD with the mean gradient: ``theta -= fl32(lr / B) * g`` for ``W1, b1, w2, b2``, ``W1T``
  rewritten as the transpose of the new ``W1`` and every gradient buffer zeroed.  ``train=False`` computes ``prob``
  and the loss only and writes nothing else.

Error model (first order, EPS = 2^-24, any summation order unless said): a sum of ``N`` terms is off by at most
``N EPS sum|terms|``.  The one exception is ``pre``: each hidden unit runs one fused multiply-add chain over the
inputs in index order starting from ``b1``, so its error is at most ``EPS`` times the sum of the chain's partial sums,
bounded here by ``EPS (IN |b1| + sum_k |S_k|)`` with ``S_k`` the prefix sums of ``x W1``.  That bound is tight
enough for ``make_b1`` to keep every pre-activation of a test batch more than 100 bounds away from 0, so the kernel
and the replay agree on every ReLU.  ``sigmoid`` and the loss use ``__expf`` (at most ``2 + 1.17 |z|`` ulp) and
``log1pf`` (1 ulp).

``BREAKS`` (the sensitivity checks of the GPU suite) each switch one rule off: ``"dense_sum_not_mean"`` steps the
dense weights by ``lr`` times the summed gradient, ``"no_wide_grad"`` pushes nothing into the wide column,
``"relu_grad_at_zero_one"`` takes ReLU'(0) = 1, ``"w1t_stale"`` leaves ``W1T`` as it was, ``"row_grad_unscaled"``
pushes ``-dLoss/drow`` without ``lr``, ``"bias_grad_from_padding_examples"`` lets the zero-filled examples of a
partial last tile (label 0) add to ``gb1``, ``gw2`` and ``gb2``."""
import math

import numpy as np

EPS = 2.0 ** -24
MARGIN = 2.0
H = 256
TB = 32
RELU_MARGIN = 100.0
BREAKS = ("dense_sum_not_mean", "no_wide_grad", "relu_grad_at_zero_one", "w1t_stale", "row_grad_unscaled",
          "bias_grad_from_padding_examples")


class Result(dict):
    __getattr__ = dict.__getitem__


def _f64(a):
    return np.asarray(a, dtype=np.float64)


def split_rows(rows, F, E):
    """(x [B, F E], wide [B, F]) of the pulled rows ``[B F, stride]``."""
    rows = _f64(rows)
    B = rows.shape[0] // F
    return rows[:, :E].reshape(B, F * E), rows[:, E].reshape(B, F)


def pre_activations(x, W1, b1):
    """(pre [B, H], tol_pre [B, H]) with the bound of the kernel's in-order FMA chain (module docstring)."""
    x, W1, b1 = _f64(x), _f64(W1), _f64(b1)
    B, IN = x.shape
    pre = np.empty((B, W1.shape[1]))
    abs_partials = np.empty_like(pre)
    for e0 in range(0, B, 64):
        terms = x[e0:e0 + 64, :, None] * W1[None, :, :]          # [b, IN, H]
        S = np.cumsum(terms, axis=1)
        pre[e0:e0 + 64] = b1[None, :] + S[:, -1, :]
        abs_partials[e0:e0 + 64] = np.abs(S).sum(axis=1)
    return pre, EPS * (IN * np.abs(b1)[None, :] + abs_partials)


def make_b1(rng, x, W1, scale=0.3, fixed_zero=(), tries=4096):
    """Draw ``b1`` so that every pre-activation of the batch ``x`` lies more than ``RELU_MARGIN`` bounds away from 0.
    Columns in ``fixed_zero`` keep ``b1 = 0`` (the caller makes their pre-activations safe some other way)."""
    x, W1 = _f64(x), _f64(W1)
    B, IN = x.shape
    _, tpre0 = pre_activations(x, W1, np.zeros(W1.shape[1]))
    S = x @ W1                                                   # [B, H]
    b1 = np.zeros(W1.shape[1], dtype=np.float32)
    for j in range(W1.shape[1]):
        if j in fixed_zero:
            continue
        for _ in range(tries // 64):
            cand = (rng.normal(0.0, scale, 64)).astype(np.float32).astype(np.float64)
            pre = cand[:, None] + S[None, :, j]
            tol = EPS * IN * np.abs(cand)[:, None] + tpre0[None, :, j]
            ok = (np.abs(pre) > RELU_MARGIN * tol).all(axis=1)
            if ok.any():
                b1[j] = cand[np.argmax(ok)]
                break
        else:
            raise RuntimeError(f"no b1[{j}] keeps the batch's pre-activations away from 0")
    return b1


def relu_margin(pre, tpre, exact_zero=None):
    """min |pre| / tol over the pre-activations that are not deliberately exactly 0."""
    r = np.abs(pre) / np.maximum(tpre, 1e-300)
    if exact_zero is not None:
        r = np.where(exact_zero, np.inf, r)
    return float(r.min())


def _sigmoid(z):
    return np.where(z >= 0, 1.0 / (1.0 + np.exp(-np.abs(z))), np.exp(-np.abs(z)) / (1.0 + np.exp(-np.abs(z))))


def replay(rows, labels, F, E, W1, b1, w2, b2, lr, train=True, breaks=None):
    """Every output of one ``native.ctr_step`` launch, in fp64, each with its bound ``tol_<name>``."""
    if breaks is not None and breaks not in BREAKS:
        raise ValueError(f"unknown break {breaks!r}")
    rows = _f64(rows)
    y = _f64(labels)
    W1, b1, w2 = _f64(W1), _f64(b1), _f64(w2)
    b2 = float(np.asarray(b2, dtype=np.float64).reshape(-1)[0])
    lr32 = float(np.float32(lr))
    B = y.shape[0]
    IN = F * E
    stride = rows.shape[1]
    x, wide = split_rows(rows, F, E)

    pre, tpre = pre_activations(x, W1, b1)
    on = pre > 0
    h = np.where(on, pre, 0.0)
    th = np.where(on, tpre, 0.0)
    hw = h * w2[None, :]
    nlog = H + F + 1
    logit = hw.sum(1) + b2 + wide.sum(1)
    tlogit = (np.abs(w2)[None, :] * th).sum(1) + (nlog + 1) * EPS * (
        np.abs(hw).sum(1) + abs(b2) + np.abs(wide).sum(1))
    p = _sigmoid(logit)
    q = np.exp(-np.abs(logit))
    r_exp = (3.0 + 1.2 * np.abs(logit)) * 2 * EPS                 # __expf, relative
    pq = p * (1 - p)
    tp = pq * (tlogit + r_exp) + 3 * EPS * p
    l1p = np.log1p(q)
    loss_e = np.maximum(logit, 0) - logit * y + l1p
    tloss_e = np.abs(p - y) * tlogit + q * r_exp + 3 * EPS * (np.abs(np.maximum(logit, 0)) + np.abs(logit * y) + l1p)
    out = Result(prob=p, tol_prob=tp, loss_sum=loss_e.sum(),
                 tol_loss_sum=B * EPS * np.abs(loss_e).sum() + tloss_e.sum(), count=B, pre=pre, tol_pre=tpre)
    if not train:
        return out

    d = p - y
    td = tp + EPS * np.abs(d)
    act = pre >= 0 if breaks == "relu_grad_at_zero_one" else on
    dh = np.where(act, d[:, None] * w2[None, :], 0.0)
    tdh = np.where(act, np.abs(w2)[None, :] * td[:, None] + EPS * np.abs(dh), 0.0)
    gW1 = x.T @ dh
    tgW1 = B * EPS * (np.abs(x).T @ np.abs(dh)) + np.abs(x).T @ tdh
    gb1, tgb1 = dh.sum(0), B * EPS * np.abs(dh).sum(0) + tdh.sum(0)
    gw2 = (d[:, None] * h).sum(0)
    tgw2 = B * EPS * np.abs(d[:, None] * h).sum(0) + (np.abs(h) * td[:, None] + np.abs(d)[:, None] * th).sum(0)
    gb2, tgb2 = d.sum(), B * EPS * np.abs(d).sum() + td.sum()
    if breaks == "bias_grad_from_padding_examples" and B % TB:
        npad = TB - B % TB                           # zero inputs, label 0: pre = b1, logit = w2 . relu(b1) + b2
        hp = np.maximum(b1, 0.0)
        dp = _sigmoid(np.array([hp @ w2 + b2]))[0]
        gb1 = gb1 + npad * np.where(b1 > 0, dp * w2, 0.0)
        gw2 = gw2 + npad * dp * hp
        gb2 = gb2 + npad * dp

    dx = dh @ W1.T                                               # [B, IN]
    tdx = H * EPS * (np.abs(dh) @ np.abs(W1).T) + tdh @ np.abs(W1).T
    rlr = 1.0 if breaks == "row_grad_unscaled" else lr32
    d_rows = np.zeros((B * F, stride))
    td_rows = np.zeros_like(d_rows)
    d_rows[:, :E] = (-rlr * dx).reshape(B * F, E)
    td_rows[:, :E] = (rlr * tdx + EPS * rlr * np.abs(dx)).reshape(B * F, E)
    if breaks != "no_wide_grad":
        d_rows[:, E] = np.repeat(-rlr * d, F)
        td_rows[:, E] = np.repeat(rlr * td + EPS * rlr * np.abs(d), F)

    scale = lr32 if breaks == "dense_sum_not_mean" else float(np.float32(np.float32(lr32) / np.float32(B)))

    def step(theta, g, tg):
        new = theta - scale * g
        return new, scale * tg + 2 * EPS * (np.abs(new) + np.abs(scale * g))

    W1n, tW1n = step(W1, gW1, tgW1)
    b1n, tb1n = step(b1, gb1, tgb1)
    w2n, tw2n = step(w2, gw2, tgw2)
    b2n, tb2n = step(np.array([b2]), np.array([gb2]), np.array([tgb2]))
    W1Tn, tW1Tn = (W1.T.copy(), np.zeros_like(W1.T)) if breaks == "w1t_stale" else (W1n.T.copy(), tW1n.T.copy())
    out.update(d_rows=d_rows, tol_d_rows=td_rows, W1=W1n, tol_W1=tW1n, W1T=W1Tn, tol_W1T=tW1Tn, b1=b1n,
               tol_b1=tb1n, w2=w2n, tol_w2=tw2n, b2=b2n, tol_b2=tb2n)
    return out


FIELDS = ("prob", "loss_sum", "d_rows", "W1", "W1T", "b1", "w2", "b2")


def violations(ref, got, fields=FIELDS, margin=MARGIN):
    """{field: number of elements of ``got`` outside ``margin`` times the replay's bound} (only nonzero counts)."""
    bad = {}
    for k in fields:
        if k not in ref or k not in got:
            continue
        want = np.asarray(ref[k], dtype=np.float64)
        have = np.asarray(got[k], dtype=np.float64).reshape(want.shape)
        n = int((~(np.abs(have - want) <= margin * np.asarray(ref["tol_" + k]))).sum())
        if n:
            bad[k] = n
    return bad


def padding_examples(B):
    """Examples the last tile carries past ``B`` (zero inputs)."""
    return (-B) % TB


def n_tiles(B):
    return math.ceil(B / TB)
