"""Factorization-machine kernel (ops/csrc/fps_fm.cu) against the fp64 replay of tests/fm_ref.py, launch by launch,
and the public DeviceFactorizationMachine on a planted model.

Every replay case reads the table, runs one ``native.fm_step`` launch, reads the table back and compares it with the
replay fed the pre-launch table: every element within ``MARGIN`` times its bound, so rows no entry touches (row 0,
row NF - 1 and the bias row's factor columns are sentinels no batch uses) and the padding columns must come back
bit for bit.  Unless a case says otherwise no feature is shared by two entries of a launch, so the launch has one
correct result however the kernel races its examples."""
import numpy as np
import pytest
import torch

from tests import fm_ref
from tests.test_fm_host import AUC_K4, QUALITY, QUALITY_LR, QUALITY_SEED, RMSE_K4, planted

pytestmark = pytest.mark.gpu

NF = 4096
MARGIN = fm_ref.MARGIN
EPS = fm_ref.EPS
KS = [0, 3, 4, 7, 8, 15, 16, 31, 32, 63, 64, 127, 128, 255, 256, 383, 384, 511]


def _model(k, loss="logistic", bias=True, partition="hash", reg=(0.0, 0.0), lr=0.05, nf=NF):
    from fps_b200.models.fm import DeviceFactorizationMachine

    torch.cuda.set_device(0)
    m = DeviceFactorizationMachine(nf, k, loss=loss, learning_rate=lr, reg_linear=reg[0], reg_factors=reg[1],
                                   init_range=(-0.3, 0.3), bias=bias, partition=partition, seed=11)
    g = torch.Generator(device="cuda").manual_seed(k + 1)
    m.table.local[:nf, 0] = torch.randn(nf, generator=g, device="cuda") * 0.3   # a non-trivial linear term
    if bias:
        m.table.local[nf, 0] = 0.2
    return m


def _table(m):
    torch.cuda.synchronize()
    return m.table.local.cpu().numpy().astype(np.float64)


def _batch(rng, n, nnz=(0, 6), loss="logistic", onehot=False, nan_every=0, lo=1, hi=NF - 1, zero_every=0):
    """CSR batch over disjoint features drawn from [lo, hi)."""
    perm = rng.permutation(np.arange(lo, hi))
    pos = 0
    rp, cols, vals, labels = [0], [], [], []
    for ex in range(n):
        k = int(rng.integers(nnz[0], nnz[1] + 1))
        cols += list(perm[pos:pos + k])
        pos += k
        x = np.ones(k) if onehot else rng.normal(0, 1.0, k)
        if zero_every and ex % zero_every == 1:
            x = np.zeros(k)
        vals += list(x)
        rp.append(len(cols))
        if nan_every and ex % nan_every == 0:
            labels.append(np.nan)
        else:
            labels.append(float(rng.integers(0, 2)) if loss == "logistic" else float(rng.normal(0.5, 1.0)))
    assert pos <= hi - lo
    return (np.array(rp, np.int64), np.array(cols, np.int64), None if onehot else np.array(vals, np.float32),
            np.array(labels, np.float32))


def _launch(m, batch, id64=False, max_ctas=0, predict_only=False):
    from fps_b200.ops import native

    rp, cols, vals, labels = batch
    dev = m.dev
    n = len(rp) - 1
    pred = torch.full((n,), float("nan"), dtype=torch.float32, device=dev)
    m._flags.zero_()
    m._stats.zero_()
    native.fm_step(m.table.table_c, torch.from_numpy(rp).to(dev),
                   torch.from_numpy(cols.astype(np.int64 if id64 else np.int32)).to(dev),
                   None if vals is None else torch.from_numpy(vals).to(dev),
                   None if predict_only else torch.from_numpy(labels).to(dev), pred,
                   num_features=m.num_features, loss=m.loss, lr=m.lr, reg_linear=m.reg_linear,
                   reg_factors=m.reg_factors, bias=m.bias, bias_state=m._bias_state, predict_only=predict_only,
                   stats=m._stats, nan_flag=m._flags[0:1], bad_id=m._flags[1:2], max_ctas=max_ctas,
                   acc=m._acc_c)
    torch.cuda.synchronize()
    return pred.cpu().numpy().astype(np.float64), m._flags.cpu().numpy(), m._stats.cpu().numpy()


def _replay(m, W, batch, breaks=None, predict_only=False):
    rp, cols, vals, labels = batch
    return fm_ref.replay(W, rp, cols, vals, labels, num_features=m.num_features, dim=1 + m.k, loss=m.loss, lr=m.lr,
                         reg_linear=m.reg_linear, reg_factors=m.reg_factors, bias=m.bias, breaks=breaks,
                         predict_only=predict_only)


def _violations(r, W_after, pred):
    """Elements of the table and predictions outside the replay's bounds."""
    bad = int((np.abs(W_after - r.table) > MARGIN * r.tol).sum())
    bad += int((np.abs(pred - r.pred) > MARGIN * r.tol_pred + EPS * np.abs(r.pred)).sum())
    return bad


def _step(m, batch, **kw):
    W = _table(m)
    pred, flags, stats = _launch(m, batch, **kw)
    W2 = _table(m)
    r = _replay(m, W, batch, predict_only=kw.get("predict_only", False))
    assert _violations(r, W2, pred) == 0, (np.abs(W2 - r.table) / np.maximum(r.tol, 1e-30)).max()
    assert (W2[:, 1 + m.k:] == 0).all()                                    # padding
    assert (W2[m.num_features, 1:] == W[m.num_features, 1:]).all()       # the bias row's other columns
    assert int(flags[0]) == 0 and int(flags[1]) == int(r.bad_id)
    if not kw.get("predict_only"):
        assert stats[1] == r.labelled
        assert abs(stats[0] - r.loss_sum) <= 1e-4 * (1 + abs(r.loss_sum))
    return r, W, W2, pred


def _config(i):
    """The i-th combination of id width, partition, one-hot, regularisation and bias."""
    return dict(id64=bool(i & 1), partition="range" if i & 2 else "hash", onehot=bool(i & 4),
                reg=(0.02, 0.05) if i % 3 == 1 else (0.0, 0.0), bias=i % 5 != 3)


@pytest.mark.parametrize("loss", ["logistic", "squared"])
@pytest.mark.parametrize("k", KS)
def test_rung_against_replay(k, loss):
    i = KS.index(k) + (7 if loss == "squared" else 0)
    c = _config(i)
    m = _model(k, loss, bias=c["bias"], partition=c["partition"], reg=c["reg"])
    rng = np.random.default_rng(100 + i)
    for _ in range(2):
        _step(m, _batch(rng, 300, loss=loss, onehot=c["onehot"], nan_every=9), id64=c["id64"])
    m.close()


@pytest.mark.parametrize("k", [0, 7, 31, 64, 383])
def test_grid_stride_rounds_and_one_cta_are_bitwise_equal(k):
    rng = np.random.default_rng(k)
    batch = _batch(rng, 1500, nnz=(0, 2), nan_every=13)
    tables, preds = [], []
    for max_ctas in (0, 1, 3):
        m = _model(k, reg=(0.01, 0.01))
        if max_ctas == 0:
            r, _, W2, pred = _step(m, batch)
        else:
            pred, _, _ = _launch(m, batch, max_ctas=max_ctas)
            W2 = _table(m)
        tables.append(W2)
        preds.append(pred)
        m.close()
    lpr = fm_ref.geometry(4 * -(-(1 + k) // 4))[0]
    assert 1500 > 3 * 256 // lpr        # the capped grids take several grid-stride rounds
    for W2, pred in zip(tables[1:], preds[1:]):
        assert (pred == preds[0]).all()
        assert (W2[:NF] == tables[0][:NF]).all()
        assert abs(W2[NF, 0] - tables[0][NF, 0]) <= EPS * abs(tables[0][NF, 0])


def test_edges_empty_zero_nan_long_bad_ids_short_cols():
    k = 20
    m = _model(k, reg=(0.01, 0.02))
    rng = np.random.default_rng(7)
    rp, cols, vals, labels = _batch(rng, 60, nnz=(0, 4), nan_every=5, zero_every=4, hi=1900)
    # one example of about 1000 entries (many TB blocks), then entries with ids NF and -1, then a short cols
    long_ids = np.arange(2000, 2999)
    rp = np.concatenate([rp, [rp[-1] + len(long_ids), rp[-1] + len(long_ids) + 3]])
    cols = np.concatenate([cols, long_ids, [NF, 3000, -1]])
    vals = np.concatenate([vals, rng.normal(0, 0.1, len(long_ids)), [1.0, 0.5, 1.0]]).astype(np.float32)
    labels = np.concatenate([labels, [1.0, 0.0]]).astype(np.float32)
    rp = np.concatenate([rp, [len(cols) + 5]])      # ends past nnz: clamped
    labels = np.concatenate([labels, [1.0]]).astype(np.float32)
    batch = (rp, cols, vals, labels)
    w0 = _table(m)[NF, 0]
    r, W, W2, pred = _step(m, batch)
    assert r.bad_id
    with pytest.raises(IndexError):
        m.check()
    assert W2[NF, 0] != w0 and np.isclose(W2[NF, 0] - w0, r.w0_delta, rtol=1e-5, atol=1e-9)
    assert pred[-1] == pytest.approx(w0)            # an empty (clamped) example predicts w0
    m.close()


@pytest.mark.parametrize("kind", ["repeated", "zipf"])
def test_shared_rows_within_forward_reverse_bound(kind):
    k = 16
    m = _model(k, reg=(0.01, 0.01), lr=0.01)
    rng = np.random.default_rng(21)
    n = 400
    if kind == "repeated":
        rp, cols, vals, labels = _batch(rng, n, nnz=(1, 5))
        cols = cols.copy()
        cols[1::7] = cols[0::7][: len(cols[1::7])]   # repeats inside and across examples
    else:
        sizes = rng.integers(1, 6, n)
        rp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        cols = np.minimum(rng.zipf(1.3, rp[-1]), NF - 2).astype(np.int64)
        vals = rng.normal(0, 1.0, rp[-1]).astype(np.float32)
        labels = rng.integers(0, 2, n).astype(np.float32)
    batch = (rp, cols, vals, labels)
    W = _table(m)
    pred, flags, _ = _launch(m, batch)
    W2 = _table(m)
    fwd = _replay(m, W, batch)
    order = np.arange(n)[::-1]
    rrp = np.concatenate([[0], np.cumsum(np.diff(rp)[order])]).astype(np.int64)
    rcols = np.concatenate([cols[rp[i]:rp[i + 1]] for i in order])
    rvals = np.concatenate([vals[rp[i]:rp[i + 1]] for i in order])
    rev = _replay(m, W, (rrp, rcols, rvals, labels[order]))
    rp_, cols_, vals_, labels_ = batch
    stale = fm_ref.replay(W, rp_, cols_, vals_, labels_, num_features=NF, dim=1 + k, loss=m.loss, lr=m.lr,
                          reg_linear=m.reg_linear, reg_factors=m.reg_factors, stale=True)
    # the kernel races its examples: somewhere between CSR order, reverse order and every example reading the
    # pre-launch rows
    spread = np.maximum(np.abs(fwd.table - rev.table), np.abs(fwd.table - stale.table))
    bound = 2 * spread + MARGIN * (fwd.tol + rev.tol + stale.tol) + 1e-7
    err = np.abs(W2 - fwd.table)
    assert (err <= bound).all(), (err / bound).max()
    assert (W2[:, 1 + k:] == 0).all() and int(flags[0]) == 0
    m.close()


@pytest.mark.parametrize("loss", ["logistic", "squared"])
def test_w0_is_read_before_the_launch_and_steps_by_the_mean(loss):
    m = _model(5, loss)
    rng = np.random.default_rng(4)
    rp = np.zeros(201, np.int64)                   # 200 empty examples: every prediction is w0
    labels = (rng.integers(0, 2, 200) if loss == "logistic" else rng.normal(0, 1, 200)).astype(np.float32)
    labels[::10] = np.nan
    w0 = _table(m)[NF, 0]
    r, _, W2, pred = _step(m, (rp, np.zeros(0, np.int64), np.zeros(0, np.float32), labels))
    assert (pred == np.float32(w0)).all()
    g = np.float32(w0) - labels if loss == "squared" else 1 / (1 + np.exp(-np.float64(np.float32(w0)))) - labels
    mean = np.nanmean(g.astype(np.float64))
    assert abs((W2[NF, 0] - w0) - (-m.lr * mean)) <= 8 * EPS * (abs(w0) + m.lr)
    assert m._bias_state[0][0].item() == 0 and m._bias_state[0][1].item() == 0 and m._bias_state[1].item() == 0
    m.close()


def test_predictions_equal_predict_before_the_step():
    m = _model(31, "logistic", reg=(0.01, 0.0))
    rng = np.random.default_rng(8)
    rp, cols, vals, labels = _batch(rng, 500)
    d = m.dev
    t = lambda a: torch.from_numpy(a).to(d)
    before = _table(m)
    p0 = m.predict_csr(t(rp), t(cols), t(vals))
    assert (_table(m) == before).all() and m.stats.sum().item() == 0
    p1 = m.step_csr(t(rp), t(cols), t(vals), t(labels))
    torch.cuda.synchronize()
    assert torch.equal(p0, p1)
    assert (_table(m) != before).any()
    m.close()


def test_no_host_sync_and_one_launch_per_step():
    from fps_b200.ops import native

    m = _model(15)
    rng = np.random.default_rng(2)
    rp, cols, vals, labels = _batch(rng, 256)
    d = m.dev
    args = [torch.from_numpy(a).to(d) for a in (rp, cols.astype(np.int32), vals, labels)]
    m.step_csr(*args)
    torch.cuda.synchronize()
    before = native.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(4):
            m.step_csr(*args)
        m.predict_csr(*args[:3])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert native.launch_count() - before == 5
    torch.cuda.synchronize()
    m.check()
    m.close()


def _sensitivity_counts():
    counts = {b: 0 for b in fm_ref.BREAKS}
    cases = 0
    for i, k in enumerate(KS):
        for loss in ("logistic", "squared"):
            m = _model(k, loss, reg=(0.05, 0.05))
            rng = np.random.default_rng(300 + i)
            batch = _batch(rng, 200, nnz=(1, 5), loss=loss)
            W = _table(m)
            pred, _, _ = _launch(m, batch)
            W2 = _table(m)
            assert _violations(_replay(m, W, batch), W2, pred) == 0
            for b in fm_ref.BREAKS:
                counts[b] += _violations(_replay(m, W, batch, breaks=b), W2, pred) > 0
            cases += 1
            m.close()
    return counts, cases


def test_broken_replays_fail():
    counts, cases = _sensitivity_counts()
    print(f"\nFM_SENSITIVITY failing cases of {cases}: {counts}")
    assert counts["no_xv"] > 0 and counts["no_half"] > 0 and counts["col0_factor"] > 0
    assert counts["w0_per_example"] > 0 and counts["reg_sign"] > 0


def _fit_device(loss, k):
    from fps_b200.models.fm import DeviceFactorizationMachine, roc_auc

    q = QUALITY
    torch.cuda.set_device(0)
    m = DeviceFactorizationMachine(q["num_features"], k, loss=loss, learning_rate=QUALITY_LR[loss],
                                   init_range=(-0.1, 0.1), seed=QUALITY_SEED)
    rp, c, l = planted(loss)
    n, B = q["n_train"], q["batch"]
    d = m.dev
    c_d, l_d = torch.from_numpy(c).to(d), torch.from_numpy(l).to(d)
    for _ in range(q["epochs"]):
        for b0 in range(0, n, B):
            b1 = min(b0 + B, n)
            m.step_csr(torch.from_numpy(rp[b0:b1 + 1] - rp[b0]).to(d), c_d[rp[b0]:rp[b1]], None, l_d[b0:b1])
    pred = m.predict_csr(torch.from_numpy(rp[n:] - rp[n]).to(d), c_d[rp[n]:]).cpu().numpy()
    m.check()
    m.close()
    if loss == "logistic":
        return roc_auc(pred, l[n:])
    return float(np.sqrt(np.mean((pred - l[n:]) ** 2)))


def test_quality_gate_through_the_public_model():
    auc4, auc0, rmse = _fit_device("logistic", 4), _fit_device("logistic", 0), _fit_device("squared", 4)
    print(f"\nFM_QUALITY device: logistic AUC k=4 {auc4:.4f} k=0 {auc0:.4f}; squared RMSE k=4 {rmse:.4f}")
    assert auc4 >= AUC_K4 - 0.01 and auc4 > auc0 + 0.1
    assert rmse <= RMSE_K4 + 0.01


def test_multi_rank_fm():
    from tests.test_gpu_multi import _run

    _run("mp_fm_check.py", 2, 29651, "MP_FM_CHECK_OK")
