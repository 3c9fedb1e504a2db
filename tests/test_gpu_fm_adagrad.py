"""Factorization-machine kernel under AdaGrad (``fps_fm_kernel`` with ``ADA`` set, DESIGN §2.17) against the fp64
replay of tests/fm_ref.py with ``acc``, launch by launch, and the public DeviceFactorizationMachine with
``optimizer="adagrad"``.

Every replay case reads the table and the accumulators, runs one launch, and compares both with the replay fed the
pre-launch state: every element within ``MARGIN`` times its bound, the padding of both exactly zero.  Unless a case
says otherwise no feature is shared by two entries of a launch."""
import numpy as np
import pytest
import torch

from tests import fm_ref
from tests.test_fm_adagrad_host import AUC_ADAGRAD, QUALITY_LRS
from tests.test_fm_host import QUALITY, QUALITY_SEED, planted
from tests.test_gpu_fm import KS, NF, _batch, _config, _launch

pytestmark = pytest.mark.gpu

MARGIN = fm_ref.MARGIN
EPS = fm_ref.EPS


def _model(k, loss="logistic", bias=True, partition="hash", reg=(0.0, 0.0), lr=0.05, nf=NF):
    from fps_b200.models.fm import DeviceFactorizationMachine

    torch.cuda.set_device(0)
    m = DeviceFactorizationMachine(nf, k, loss=loss, learning_rate=lr, reg_linear=reg[0], reg_factors=reg[1],
                                   init_range=(-0.3, 0.3), bias=bias, partition=partition, seed=11,
                                   optimizer="adagrad")
    g = torch.Generator(device="cuda").manual_seed(k + 1)
    m.table.local[:nf, 0] = torch.randn(nf, generator=g, device="cuda") * 0.3
    if bias:
        m.table.local[nf, 0] = 0.2
    # a non-trivial H on every live column of the feature rows (the bias row and the padding stay 0)
    ids = m.table.local_ids()
    live = (ids < nf)[:, None] & (torch.arange(m.table.stride, device="cuda") < 1 + k)[None, :]
    m._acc.local.copy_(torch.rand(m._acc.local.shape, generator=g, device="cuda") * 2.0 * live)
    return m


def _state(m):
    torch.cuda.synchronize()
    return (m.table.local.cpu().numpy().astype(np.float64), m._acc.local.cpu().numpy().astype(np.float64))


def _replay(m, W, H, batch, breaks=None, predict_only=False, **kw):
    rp, cols, vals, labels = batch
    return fm_ref.replay(W, rp, cols, vals, labels, num_features=m.num_features, dim=1 + m.k, loss=m.loss,
                         lr=m.lr, reg_linear=m.reg_linear, reg_factors=m.reg_factors, bias=m.bias, breaks=breaks,
                         predict_only=predict_only, acc=H, **kw)


def _violations(r, W2, H2, pred):
    bad = int((np.abs(W2 - r.table) > MARGIN * r.tol).sum())
    bad += int((np.abs(H2 - r.acc) > MARGIN * r.tol_acc).sum())
    bad += int((np.abs(pred - r.pred) > MARGIN * r.tol_pred + EPS * np.abs(r.pred)).sum())
    return bad


def _step(m, batch, **kw):
    W, H = _state(m)
    pred, flags, stats = _launch(m, batch, **kw)
    W2, H2 = _state(m)
    r = _replay(m, W, H, batch, predict_only=kw.get("predict_only", False))
    assert _violations(r, W2, H2, pred) == 0, (np.abs(W2 - r.table) / np.maximum(r.tol, 1e-30)).max()
    assert (W2[:, 1 + m.k:] == 0).all() and (H2[:, 1 + m.k:] == 0).all()      # padding of both
    assert (H2[m.num_features] == 0).all()                                     # w0 has no accumulator
    assert int(flags[0]) == 0 and int(flags[1]) == int(r.bad_id)
    return r, (W, H), (W2, H2), pred


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
    out = []
    for max_ctas in (0, 1, 3):
        m = _model(k, reg=(0.01, 0.01))
        if max_ctas == 0:
            _, _, (W2, H2), pred = _step(m, batch)
        else:
            pred, _, _ = _launch(m, batch, max_ctas=max_ctas)
            W2, H2 = _state(m)
        out.append((W2, H2, pred))
        m.close()
    for W2, H2, pred in out[1:]:
        assert (pred == out[0][2]).all() and (W2[:NF] == out[0][0][:NF]).all() and (H2 == out[0][1]).all()
        assert abs(W2[NF, 0] - out[0][0][NF, 0]) <= EPS * abs(out[0][0][NF, 0])


def test_edges_empty_zero_nan_long_bad_ids_short_cols():
    m = _model(20, reg=(0.01, 0.02))
    rng = np.random.default_rng(7)
    rp, cols, vals, labels = _batch(rng, 60, nnz=(0, 4), nan_every=5, zero_every=4, hi=1900)
    long_ids = np.arange(2000, 2999)
    rp = np.concatenate([rp, [rp[-1] + len(long_ids), rp[-1] + len(long_ids) + 3]])
    cols = np.concatenate([cols, long_ids, [NF, 3000, -1]])
    vals = np.concatenate([vals, rng.normal(0, 0.1, len(long_ids)), [1.0, 0.5, 1.0]]).astype(np.float32)
    labels = np.concatenate([labels, [1.0, 0.0]]).astype(np.float32)
    rp = np.concatenate([rp, [len(cols) + 5]])
    labels = np.concatenate([labels, [1.0]]).astype(np.float32)
    r, (W, H), (W2, H2), pred = _step(m, (rp, cols, vals, labels))
    assert r.bad_id
    # the rows of NaN-labelled examples keep their H
    for ex in np.nonzero(np.isnan(labels))[0]:
        ids = cols[rp[ex]:rp[ex + 1]]
        assert (H2[ids] == H[ids]).all()
    m.close()


def test_predict_only_leaves_h_alone():
    m = _model(31)
    rng = np.random.default_rng(8)
    rp, cols, vals, labels = _batch(rng, 500)
    W, H = _state(m)
    d = m.dev
    t = lambda a: torch.from_numpy(a).to(d)
    p0 = m.predict_csr(t(rp), t(cols), t(vals))
    W1, H1 = _state(m)
    assert (W1 == W).all() and (H1 == H).all()
    p1 = m.step_csr(t(rp), t(cols), t(vals), t(labels))
    torch.cuda.synchronize()
    assert torch.equal(p0, p1)
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
        cols[1::7] = cols[0::7][: len(cols[1::7])]
    else:
        sizes = rng.integers(1, 6, n)
        rp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        cols = np.minimum(rng.zipf(1.3, rp[-1]), NF - 2).astype(np.int64)
        vals = rng.normal(0, 1.0, rp[-1]).astype(np.float32)
        labels = rng.integers(0, 2, n).astype(np.float32)
    batch = (rp, cols, vals, labels)
    W, H = _state(m)
    pred, flags, _ = _launch(m, batch)
    W2, H2 = _state(m)
    fwd = _replay(m, W, H, batch)
    order = np.arange(n)[::-1]
    rrp = np.concatenate([[0], np.cumsum(np.diff(rp)[order])]).astype(np.int64)
    rcols = np.concatenate([cols[rp[i]:rp[i + 1]] for i in order])
    rvals = np.concatenate([vals[rp[i]:rp[i + 1]] for i in order])
    rev = _replay(m, W, H, (rrp, rcols, rvals, labels[order]))
    stale = _replay(m, W, H, batch, stale=True)
    live = _replay(m, W, H, batch, repull=True)
    # the kernel races its examples, and its pass 2 may read a row and H that an earlier entry of the same example
    # pushed: somewhere between CSR order, reverse order, pre-launch reads and those re-pulls.  Per element that
    # envelope does not hold for AdaGrad (the table and H exceed it 1.5-4x on the H100): a row and its H are two
    # pulls, and a push from another example can land between them, a state no replay order reproduces.  So, as
    # for shared FFM slabs (§2.16), the launch's whole update of the table and of H must each lie within twice the
    # replays' own spread of it, in norm
    others = (rev, stale, live)
    for key, got, before, tol in (("table", W2, W, "tol"), ("acc", H2, H, "tol_acc")):
        spread = np.maximum.reduce([np.abs(fwd[key] - o[key]) for o in others])
        bound = 2 * spread + MARGIN * (fwd[tol] + sum(o[tol] for o in others)) + 1e-7
        upd = np.linalg.norm(fwd[key] - before)
        rel = np.linalg.norm(got - fwd[key]) / upd
        spread_rel = max(np.linalg.norm(fwd[key] - o[key]) / upd for o in others)
        print(f"\nFM_ADAGRAD_SHARED {kind} {key}: |kernel - replay| / |update| = {rel:.2e}, replays' spread "
              f"{spread_rel:.2e}, element envelope ratio {(np.abs(got - fwd[key]) / bound).max():.2f}")
        assert rel <= 2 * spread_rel + 1e-6
    assert (W2[:, 1 + k:] == 0).all() and (H2[:, 1 + k:] == 0).all() and int(flags[0]) == 0
    m.close()


def test_no_host_sync_and_one_launch_per_step():
    from fps_b200.ops import native

    m = _model(15)
    rng = np.random.default_rng(2)
    rp, cols, vals, labels = _batch(rng, 256)
    args = [torch.from_numpy(a).to(m.dev) for a in (rp, cols.astype(np.int32), vals, labels)]
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


def test_broken_replays_fail():
    counts = {b: 0 for b in fm_ref.ADAGRAD_BREAKS}
    cases = 0
    for i, k in enumerate(KS):
        for loss in ("logistic", "squared"):
            m = _model(k, loss, reg=(0.05, 0.05))
            rng = np.random.default_rng(300 + i)
            batch = _batch(rng, 200, nnz=(1, 5), loss=loss)
            W, H = _state(m)
            pred, _, _ = _launch(m, batch)
            W2, H2 = _state(m)
            assert _violations(_replay(m, W, H, batch), W2, H2, pred) == 0
            for b in fm_ref.ADAGRAD_BREAKS:
                counts[b] += _violations(_replay(m, W, H, batch, breaks=b), W2, H2, pred) > 0
            cases += 1
            m.close()
    print(f"\nFM_ADAGRAD_SENSITIVITY failing cases of {cases}: {counts}")
    assert all(c > cases // 2 for c in counts.values()), counts


def _fit_device(k, lr):
    from fps_b200.models.fm import DeviceFactorizationMachine, roc_auc

    q = QUALITY
    torch.cuda.set_device(0)
    m = DeviceFactorizationMachine(q["num_features"], k, loss="logistic", learning_rate=lr, init_range=(-0.1, 0.1),
                                   seed=QUALITY_SEED, optimizer="adagrad")
    rp, c, l = planted("logistic")
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
    return roc_auc(pred, l[n:])


def test_quality_sweep_through_the_public_model():
    aucs = {lr: _fit_device(4, lr) for lr in QUALITY_LRS}
    print(f"\nFM_ADAGRAD_QUALITY device AUC per lr: {aucs}")
    for lr, auc in aucs.items():
        assert abs(auc - AUC_ADAGRAD[lr]) <= 0.01, (lr, auc, AUC_ADAGRAD[lr])


def test_host_step_and_accumulator_round_trip():
    from fps_b200.models.fm import DeviceFactorizationMachine
    from fps_b200.models.pa.sparse import SparseVector

    torch.cuda.set_device(0)
    m = DeviceFactorizationMachine(50, 3, learning_rate=0.2, optimizer="adagrad", seed=2)
    v = [SparseVector([1, 3], [1.0, 2.0], 50), SparseVector([7], [0.5], 50)]
    m.step(v, [1.0, 0.0])
    ids, H = m.accumulators()
    assert H.shape == (len(ids), 4) and (H >= 0).all()
    touched = {i: h for i, h in zip(ids, H)}
    assert all((touched[i] > 0).any() for i in (1, 3, 7)) and not touched[2].any()
    model = m.model()
    m2 = DeviceFactorizationMachine(50, 3, learning_rate=0.2, optimizer="adagrad", seed=9)
    m2.load_model(model)
    m2.load_accumulators(ids, H)
    assert np.array_equal(m2.accumulators()[1], H)
    p1, p2 = m.step(v, [1.0, 0.0]), m2.step(v, [1.0, 0.0])
    assert p1 == p2
    assert np.array_equal(m.accumulators()[1], m2.accumulators()[1])
    m.close()
    m2.close()


def test_multi_rank_fm_adagrad():
    from tests.test_gpu_multi import _run

    _run("mp_fm_adagrad_check.py", 2, 29653, "MP_FM_ADAGRAD_CHECK_OK")
