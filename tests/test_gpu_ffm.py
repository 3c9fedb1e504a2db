"""Field-aware FM kernel (ops/csrc/fps_ffm.cu) against the fp64 replay of tests/ffm_ref.py, launch by launch, and the
public DeviceFieldAwareFM on a planted model.

Every replay case reads the table, runs one ``native.ffm_step`` launch, reads the table back and compares it with the
replay fed the pre-launch table: every element within ``MARGIN`` times its bound, so rows no entry touches (row 0 and
row NF - 1 are sentinels no batch uses), the padding of every slab, columns 1..3 and the bias row's other columns
must come back bit for bit.  Unless a case says otherwise no feature is shared by two entries of a launch and no
example has a field twice among three or more entries, so no slab and no ``w`` takes two pushes and the launch has
one correct result however the kernel races its examples."""
import numpy as np
import pytest
import torch

from tests import ffm_ref
from tests.test_ffm_host import (AUC_FFM, AUC_MARGIN_FM, AUC_MARGIN_LINEAR, QUALITY, QUALITY_K, QUALITY_LR,
                                 QUALITY_SEED, planted)

pytestmark = pytest.mark.gpu

MARGIN = ffm_ref.MARGIN
EPS = ffm_ref.EPS
KS = [1, 4, 5, 8, 9, 16, 17, 32, 33, 64]
FS = [1, 2, 39, 256]


def _nf(F, k):
    """Features of a case's table: 4096, fewer when the rows are wide."""
    return 4096 if ffm_ref.stride(F, k) <= 1100 else 1024


def _model(k, F, loss="logistic", bias=True, partition="hash", reg=(0.0, 0.0), lr=0.05, nf=None):
    from fps_b200.models.fm import DeviceFieldAwareFM

    nf = _nf(F, k) if nf is None else nf
    torch.cuda.set_device(0)
    m = DeviceFieldAwareFM(nf, F, k, loss=loss, learning_rate=lr, reg_linear=reg[0], reg_factors=reg[1],
                           init_range=(-0.3, 0.3), bias=bias, partition=partition, seed=11)
    g = torch.Generator(device="cuda").manual_seed(k + F)
    m.table.local[:nf, 0] = torch.randn(nf, generator=g, device="cuda") * 0.3   # a non-trivial linear term
    if bias:
        m.table.local[nf, 0] = 0.2
    return m


def _table(m):
    torch.cuda.synchronize()
    return m.table.local.cpu().numpy().astype(np.float64)


def _fields(rng, F, k):
    """Fields of an example of k entries with no slab pushed twice: distinct, or any two."""
    if k <= 2:
        return list(rng.integers(0, F, k))
    return list(rng.choice(F, k, replace=False))


def _batch(rng, n, F, nf, nnz=(0, 6), loss="logistic", onehot=False, nan_every=0, lo=1, hi=None):
    """CSR batch over disjoint features drawn from [lo, hi)."""
    hi = nf - 1 if hi is None else hi
    perm = rng.permutation(np.arange(lo, hi))
    pos = 0
    rp, cols, fields, vals, labels = [0], [], [], [], []
    for ex in range(n):
        k = int(rng.integers(nnz[0], min(nnz[1], max(F, 2)) + 1))
        cols += list(perm[pos:pos + k])
        pos += k
        fields += _fields(rng, F, k)
        vals += list(np.ones(k) if onehot else rng.normal(0, 1.0, k))
        rp.append(len(cols))
        if nan_every and ex % nan_every == 0:
            labels.append(np.nan)
        else:
            labels.append(float(rng.integers(0, 2)) if loss == "logistic" else float(rng.normal(0.5, 1.0)))
    assert pos <= hi - lo
    return (np.array(rp, np.int64), np.array(cols, np.int64), np.array(fields, np.int32),
            None if onehot else np.array(vals, np.float32), np.array(labels, np.float32))


def _launch(m, batch, id64=False, max_ctas=0, predict_only=False):
    from fps_b200.ops import native

    rp, cols, fields, vals, labels = batch
    dev = m.dev
    n = len(rp) - 1
    pred = torch.full((n,), float("nan"), dtype=torch.float32, device=dev)
    m._flags.zero_()
    m._stats.zero_()
    t = lambda a: torch.from_numpy(a).to(dev)
    native.ffm_step(m.table.table_c, t(rp), t(cols.astype(np.int64 if id64 else np.int32)), t(fields),
                    None if vals is None else t(vals), None if predict_only else t(labels), pred,
                    num_features=m.num_features, num_fields=m.num_fields, num_factors=m.k, loss=m.loss, lr=m.lr,
                    reg_linear=m.reg_linear, reg_factors=m.reg_factors, bias=m.bias, bias_state=m._bias_state,
                    predict_only=predict_only, stats=m._stats, nan_flag=m._flags[0:1], bad_id=m._flags[1:2],
                    max_ctas=max_ctas, acc=m._acc_c)
    torch.cuda.synchronize()
    return pred.cpu().numpy().astype(np.float64), m._flags.cpu().numpy(), m._stats.cpu().numpy()


def _replay(m, W, batch, breaks=None, predict_only=False, **kw):
    rp, cols, fields, vals, labels = batch
    return ffm_ref.replay(W, rp, cols, fields, vals, labels, num_features=m.num_features, num_fields=m.num_fields,
                          k=m.k, loss=m.loss, lr=m.lr, reg_linear=m.reg_linear, reg_factors=m.reg_factors,
                          bias=m.bias, breaks=breaks, predict_only=predict_only, **kw)


def _violations(r, W_after, pred):
    """Elements of the table and predictions outside the replay's bounds."""
    bad = int((np.abs(W_after - r.table) > MARGIN * r.tol).sum())
    bad += int((np.abs(pred - r.pred) > MARGIN * r.tol_pred + EPS * np.abs(r.pred)).sum())
    return bad


def _padding_ok(m, W, W2):
    kp = ffm_ref.kpad(m.k)
    pad = np.zeros(W.shape[1], bool)
    pad[1:4] = True
    for f in range(m.num_fields):
        pad[4 + f * kp + m.k: 4 + (f + 1) * kp] = True
    return (W2[:, pad] == 0).all() and (W2[m.num_features, 1:] == W[m.num_features, 1:]).all()


def _step(m, batch, **kw):
    W = _table(m)
    pred, flags, stats = _launch(m, batch, **kw)
    W2 = _table(m)
    r = _replay(m, W, batch, predict_only=kw.get("predict_only", False))
    assert _violations(r, W2, pred) == 0, (np.abs(W2 - r.table) / np.maximum(r.tol, 1e-30)).max()
    assert _padding_ok(m, W, W2)
    assert int(flags[0]) == 0 and int(flags[1]) == int(r.bad_id)
    if not kw.get("predict_only"):
        assert stats[1] == r.labelled
        assert abs(stats[0] - r.loss_sum) <= 1e-4 * (1 + abs(r.loss_sum))
    return r, W, W2, pred


def _config(i):
    """The i-th combination of id width, partition, one-hot, regularisation, bias and loss."""
    return dict(id64=bool(i & 1), partition="range" if i & 2 else "hash", onehot=bool(i & 4),
                reg=(0.02, 0.05) if i % 3 == 1 else (0.0, 0.0), bias=i % 5 != 3,
                loss="squared" if (i // 8) % 2 else "logistic")


@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("k", KS)
def test_rung_against_replay(k, F):
    i = KS.index(k) * len(FS) + FS.index(F)
    c = _config(i)
    m = _model(k, F, c["loss"], bias=c["bias"], partition=c["partition"], reg=c["reg"])
    rng = np.random.default_rng(100 + i)
    n = 200 if m.num_features > 2000 else 120
    for _ in range(2):
        _step(m, _batch(rng, n, F, m.num_features, loss=c["loss"], onehot=c["onehot"], nan_every=9),
              id64=c["id64"])
    m.close()


@pytest.mark.parametrize("k, F", [(1, 39), (5, 2), (17, 39), (64, 7)])
def test_grid_stride_rounds_and_one_cta_are_bitwise_equal(k, F):
    rng = np.random.default_rng(k + F)
    n = 600
    batch = _batch(rng, n, F, 4096, nnz=(0, 6), nan_every=13)
    tables, preds = [], []
    for max_ctas in (0, 1, 3):
        m = _model(k, F, reg=(0.01, 0.01), nf=4096)
        if max_ctas == 0:
            r, _, W2, pred = _step(m, batch)
        else:
            pred, _, _ = _launch(m, batch, max_ctas=max_ctas)
            W2 = _table(m)
        tables.append(W2)
        preds.append(pred)
        m.close()
    assert n > 3 * 8        # the capped grids take several grid-stride rounds (8 warps per CTA)
    for W2, pred in zip(tables[1:], preds[1:]):
        assert (pred == preds[0]).all()
        assert (W2[:4096] == tables[0][:4096]).all()
        assert abs(W2[4096, 0] - tables[0][4096, 0]) <= EPS * abs(tables[0][4096, 0])


def test_edges_empty_one_entry_long_bad_entries_nan_and_short_cols():
    k, F, nf = 4, 256, 4096
    m = _model(k, F, reg=(0.01, 0.02), nf=nf)
    rng = np.random.default_rng(7)
    rp, cols, fields, vals, labels = _batch(rng, 60, F, nf, nnz=(0, 4), nan_every=5, hi=1500)
    rp = np.concatenate([rp, [rp[-1], rp[-1] + 1]])            # an empty example and a one-entry example
    cols = np.concatenate([cols, [1600]])
    fields = np.concatenate([fields, [3]]).astype(np.int32)
    vals = np.concatenate([vals, [0.7]])
    labels = np.concatenate([labels, [1.0, 0.0]])
    # one example of 320 entries over five metadata chunks: 256 kept, every field once, and 64 skipped entries
    # (ids NF and -1, fields F and -1) spread through it
    ids = np.arange(2000, 2256)
    lf = rng.permutation(F)
    bad = [(nf, 0), (-1, 1), (2300, F), (2301, -1)] * 16
    at = np.sort(rng.choice(320, 64, replace=False))
    lc, lfs, j, q = [], [], 0, 0
    for pos in range(320):
        if q < 64 and at[q] == pos:
            lc.append(bad[q][0]); lfs.append(bad[q][1]); q += 1
        else:
            lc.append(ids[j]); lfs.append(lf[j]); j += 1
    rp = np.concatenate([rp, [rp[-1] + 320]])
    cols = np.concatenate([cols, lc])
    fields = np.concatenate([fields, lfs]).astype(np.int32)
    vals = np.concatenate([vals, rng.normal(0, 0.2, 320)]).astype(np.float32)
    labels = np.concatenate([labels, [1.0]])
    rp = np.concatenate([rp, [len(cols) + 5]])                 # ends past nnz: clamped to an empty example
    labels = np.concatenate([labels, [1.0]]).astype(np.float32)
    batch = (rp, cols, fields, vals, labels)
    w0 = _table(m)[nf, 0]
    r, W, W2, pred = _step(m, batch)
    assert r.bad_id
    with pytest.raises(IndexError):
        m.check()
    assert W2[nf, 0] != w0 and np.isclose(W2[nf, 0] - w0, r.w0_delta, rtol=1e-5, atol=1e-9)
    assert pred[-1] == pytest.approx(w0) and pred[60] == pytest.approx(w0)   # empty examples predict w0
    assert (W2[ids, 4:] != W[ids, 4:]).sum() >= 255 * k                  # the long example's slabs moved
    m.close()


@pytest.mark.parametrize("kind", ["multi_hot", "shared", "zipf"])
def test_shared_slabs(kind):
    k, F, nf = 8, 5, 4096
    m = _model(k, F, reg=(0.01, 0.01), lr=0.01, nf=nf)
    rng = np.random.default_rng(21)
    n = 300
    sizes = rng.integers(1, 6, n)
    rp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    nnz = int(rp[-1])
    fields = rng.integers(0, F, nnz).astype(np.int32)                # multi-hot: fields repeat inside examples
    if kind == "multi_hot":
        cols = rng.permutation(np.arange(1, nf - 1))[:nnz]
    elif kind == "shared":
        cols = rng.permutation(np.arange(1, nf - 1))[:nnz]
        cols[1::7] = cols[0::7][: len(cols[1::7])]                 # repeats inside and across examples
    else:
        cols = np.minimum(rng.zipf(1.3, nnz), nf - 2)
    cols = cols.astype(np.int64)
    vals = rng.normal(0, 1.0, nnz).astype(np.float32)
    labels = rng.integers(0, 2, n).astype(np.float32)
    batch = (rp, cols, fields, vals, labels)
    W = _table(m)
    pred, flags, _ = _launch(m, batch)
    W2 = _table(m)
    fwd = _replay(m, W, batch)
    order = np.arange(n)[::-1]
    rrp = np.concatenate([[0], np.cumsum(np.diff(rp)[order])]).astype(np.int64)
    seg = lambda a: np.concatenate([a[rp[i]:rp[i + 1]] for i in order])
    rev = _replay(m, W, (rrp, seg(cols), seg(fields), seg(vals), labels[order]))
    stale = _replay(m, W, batch, stale=True)
    live = _replay(m, W, batch, repull=True)
    # the kernel races its examples and, in pass 2, the pairs of one example: each push lies somewhere between
    # CSR order, reverse order, every example reading the pre-launch rows and every push reading the rows before
    # it.  An example pulls in pass 1 and re-pulls in pass 2 at two moments of that race, so the pushes a row takes
    # can each sit at a different end: the envelope grows with the entries that push the row
    spread = np.maximum.reduce([np.abs(fwd.table - o.table) for o in (rev, stale, live)])
    pushes = np.bincount(cols, minlength=nf + 1)[:, None]
    bound = 2 * np.maximum(pushes, 1) * spread + MARGIN * (fwd.tol + rev.tol + stale.tol + live.tol) + 1e-7
    err = np.abs(W2 - fwd.table)
    if kind == "multi_hot":
        assert (err <= bound).all(), (err / bound).max()
    else:
        # with shared features a row's deltas read partner slabs that other examples push at the same time, at
        # moments no replay order reproduces, and the per-element envelope does not hold; the launch's update as a
        # whole must lie within twice the replays' own spread of it
        upd = np.linalg.norm(fwd.table - W)
        rel = np.linalg.norm(W2 - fwd.table) / upd
        spread_rel = max(np.linalg.norm(fwd.table - o.table) / upd for o in (rev, stale, live))
        print(f"\nFFM_SHARED {kind}: |kernel - replay| / |update| = {rel:.2e}, replays' spread {spread_rel:.2e}, "
              f"element envelope ratio {(err / bound).max():.2f}")
        assert rel <= 2 * spread_rel + 1e-6
    untouched = ~np.isin(np.arange(nf + 1), cols)
    untouched[nf] = False
    assert np.isfinite(W2).all() and (W2[untouched] == W[untouched]).all()
    assert _padding_ok(m, W, W2) and int(flags[0]) == 0
    m.close()


@pytest.mark.parametrize("loss", ["logistic", "squared"])
def test_w0_is_read_before_the_launch_and_steps_by_the_mean(loss):
    m = _model(5, 3, loss)
    nf = m.num_features
    rng = np.random.default_rng(4)
    rp = np.zeros(201, np.int64)                   # 200 empty examples: every prediction is w0
    labels = (rng.integers(0, 2, 200) if loss == "logistic" else rng.normal(0, 1, 200)).astype(np.float32)
    labels[::10] = np.nan
    w0 = _table(m)[nf, 0]
    r, _, W2, pred = _step(m, (rp, np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32), labels))
    assert (pred == np.float32(w0)).all()
    g = np.float32(w0) - labels if loss == "squared" else 1 / (1 + np.exp(-np.float64(np.float32(w0)))) - labels
    mean = np.nanmean(g.astype(np.float64))
    assert abs((W2[nf, 0] - w0) - (-m.lr * mean)) <= 8 * EPS * (abs(w0) + m.lr)
    assert m._bias_state[0][0].item() == 0 and m._bias_state[0][1].item() == 0 and m._bias_state[1].item() == 0
    m.close()


def test_predictions_equal_predict_before_the_step():
    m = _model(12, 39, "logistic", reg=(0.01, 0.0))
    rng = np.random.default_rng(8)
    rp, cols, fields, vals, labels = _batch(rng, 400, 39, m.num_features)
    t = lambda a: torch.from_numpy(a).to(m.dev)
    before = _table(m)
    p0 = m.predict_csr(t(rp), t(cols), t(fields), t(vals))
    assert (_table(m) == before).all() and m.stats.sum().item() == 0
    p1 = m.step_csr(t(rp), t(cols), t(fields), t(vals), t(labels))
    torch.cuda.synchronize()
    assert torch.equal(p0, p1)
    assert (_table(m) != before).any()
    m.close()


def test_no_host_sync_and_one_launch_per_step():
    from fps_b200.ops import native

    m = _model(15, 39)
    rng = np.random.default_rng(2)
    rp, cols, fields, vals, labels = _batch(rng, 256, 39, m.num_features)
    args = [torch.from_numpy(a).to(m.dev) for a in (rp, cols.astype(np.int32), fields, vals, labels)]
    m.step_csr(*args)
    torch.cuda.synchronize()
    before = native.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(4):
            m.step_csr(*args)
        m.predict_csr(*args[:4])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert native.launch_count() - before == 5
    torch.cuda.synchronize()
    m.check()
    m.close()


def _sensitivity_counts():
    counts = {b: 0 for b in ffm_ref.BREAKS}
    cases = 0
    for i, k in enumerate(KS):
        for loss in ("logistic", "squared"):
            F = FS[(i + (loss == "squared")) % len(FS)]
            m = _model(k, F, loss, reg=(0.05, 0.05))
            rng = np.random.default_rng(300 + i)
            batch = _batch(rng, 100, F, m.num_features, nnz=(1, 6), loss=loss)
            W = _table(m)
            pred, _, _ = _launch(m, batch)
            W2 = _table(m)
            assert _violations(_replay(m, W, batch), W2, pred) == 0
            for b in ffm_ref.BREAKS:
                counts[b] += _violations(_replay(m, W, batch, breaks=b), W2, pred) > 0
            cases += 1
            m.close()
    return counts, cases


def test_broken_replays_fail():
    counts, cases = _sensitivity_counts()
    print(f"\nFFM_SENSITIVITY failing cases of {cases}: {counts}")
    for b in ffm_ref.BREAKS:
        assert counts[b] > cases // 2, (b, counts[b], cases)


def _fit_device(kind):
    from fps_b200.models.fm import DeviceFactorizationMachine, DeviceFieldAwareFM, roc_auc

    q = QUALITY
    torch.cuda.set_device(0)
    if kind == "ffm":
        m = DeviceFieldAwareFM(q["num_features"], q["fields"], QUALITY_K, learning_rate=QUALITY_LR,
                               init_range=(-0.1, 0.1), seed=QUALITY_SEED)
    else:
        m = DeviceFactorizationMachine(q["num_features"], QUALITY_K if kind == "fm" else 0,
                                       learning_rate=QUALITY_LR, init_range=(-0.1, 0.1), seed=QUALITY_SEED)
    rp, c, f, l = planted()
    n, B = q["n_train"], q["batch"]
    d = m.dev
    c_d, f_d, l_d = (torch.from_numpy(a).to(d) for a in (c, f, l))
    for _ in range(q["epochs"]):
        for b0 in range(0, n, B):
            b1 = min(b0 + B, n)
            rp_d = torch.from_numpy(rp[b0:b1 + 1] - rp[b0]).to(d)
            s = slice(rp[b0], rp[b1])
            if kind == "ffm":
                m.step_csr(rp_d, c_d[s], f_d[s], None, l_d[b0:b1])
            else:
                m.step_csr(rp_d, c_d[s], None, l_d[b0:b1])
    rp_t = torch.from_numpy(rp[n:] - rp[n]).to(d)
    pred = (m.predict_csr(rp_t, c_d[rp[n]:], f_d[rp[n]:]) if kind == "ffm" else
            m.predict_csr(rp_t, c_d[rp[n]:])).cpu().numpy()
    m.check()
    m.close()
    return roc_auc(pred, l[n:])


def test_quality_gate_through_the_public_model():
    ffm, fm, lin = _fit_device("ffm"), _fit_device("fm"), _fit_device("linear")
    print(f"\nFFM_QUALITY device held-out AUC: FFM k={QUALITY_K} {ffm:.4f}  FM k={QUALITY_K} {fm:.4f}  "
          f"linear {lin:.4f}")
    assert ffm >= AUC_FFM - 0.01
    assert ffm > fm + AUC_MARGIN_FM and ffm > lin + AUC_MARGIN_LINEAR


def test_host_step_and_model_round_trip():
    m = _model(6, 3, reg=(0.0, 0.0), nf=64)
    ex = [[(0, 5, 1.0), (1, 9, 0.5), (2, 11, 2.0)], [(2, 7, 1.0)], []]
    before = {i: (w, V) for i, w, V in m.model(only_nonzero=False)}
    pred = m.step(ex, [1.0, None, 0.0])
    assert len(pred) == 3 and pred[2] == pytest.approx(0.2)
    after = {i: (w, V) for i, w, V in m.model(only_nonzero=False)}
    assert after[5][1].shape == (3, 6)
    assert not np.array_equal(after[5][1], before[5][1]) and np.array_equal(after[7][1], before[7][1])
    m.load_model([(5, 0.5, np.full((3, 6), 0.25))])
    got = {i: (w, V) for i, w, V in m.model(only_nonzero=False)}
    assert got[5][0] == 0.5 and (got[5][1] == 0.25).all()
    assert _padding_ok(m, _table(m), _table(m))
    m.check()
    m.close()


def test_multi_rank_ffm():
    from tests.test_gpu_multi import _run

    _run("mp_ffm_check.py", 2, 29653, "MP_FFM_CHECK_OK")
