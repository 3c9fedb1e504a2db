"""Field-aware FM kernel under AdaGrad (``fps_ffm_kernel`` with ``ADA`` set, DESIGN §2.17) against the fp64 replay
of tests/ffm_ref.py with ``acc``, launch by launch, and the public DeviceFieldAwareFM with ``optimizer="adagrad"``.

Every replay case compares the table and the accumulators after one launch with the replay fed the pre-launch
state: every element within ``MARGIN`` times its bound, the padding of both exactly zero.  Unless a case says
otherwise no slab and no ``w`` is pushed twice in a launch."""
import numpy as np
import pytest
import torch

from tests import ffm_ref, fm_ref
from tests.test_ffm_adagrad_host import (AUC_ADAGRAD, AUC_LIBFFM_FFM, AUC_LIBFFM_FM, AUC_LIBFFM_LINEAR, LIBFFM,
                                         QUALITY_LRS)
from tests.test_ffm_host import QUALITY, QUALITY_SEED, planted
from tests.test_gpu_ffm import FS, KS, _batch, _config, _launch, _nf, _padding_ok

pytestmark = pytest.mark.gpu

MARGIN = ffm_ref.MARGIN
EPS = ffm_ref.EPS


def _model(k, F, loss="logistic", bias=True, partition="hash", reg=(0.0, 0.0), lr=0.05, nf=None):
    from fps_b200.models.fm import DeviceFieldAwareFM

    nf = _nf(F, k) if nf is None else nf
    torch.cuda.set_device(0)
    m = DeviceFieldAwareFM(nf, F, k, loss=loss, learning_rate=lr, reg_linear=reg[0], reg_factors=reg[1],
                           init_range=(-0.3, 0.3), bias=bias, partition=partition, seed=11, optimizer="adagrad")
    g = torch.Generator(device="cuda").manual_seed(k + F)
    m.table.local[:nf, 0] = torch.randn(nf, generator=g, device="cuda") * 0.3
    if bias:
        m.table.local[nf, 0] = 0.2
    # a non-trivial H on w and every slab's factors of the feature rows; columns 1..3, padding and the bias row 0
    live = torch.zeros(m.table.stride, dtype=torch.bool, device="cuda")
    live[0] = True
    for f in range(F):
        live[4 + f * m.kp: 4 + f * m.kp + k] = True
    live = (m.table.local_ids() < nf)[:, None] & live[None, :]
    m._acc.local.copy_(torch.rand(m._acc.local.shape, generator=g, device="cuda") * 2.0 * live)
    return m


def _state(m):
    torch.cuda.synchronize()
    return (m.table.local.cpu().numpy().astype(np.float64), m._acc.local.cpu().numpy().astype(np.float64))


def _replay(m, W, H, batch, breaks=None, predict_only=False, **kw):
    rp, cols, fields, vals, labels = batch
    return ffm_ref.replay(W, rp, cols, fields, vals, labels, num_features=m.num_features, num_fields=m.num_fields,
                          k=m.k, loss=m.loss, lr=m.lr, reg_linear=m.reg_linear, reg_factors=m.reg_factors, bias=m.bias,
                          breaks=breaks, predict_only=predict_only, acc=H, **kw)


def _violations(r, W2, H2, pred):
    bad = int((np.abs(W2 - r.table) > MARGIN * r.tol).sum())
    bad += int((np.abs(H2 - r.acc) > MARGIN * r.tol_acc).sum())
    bad += int((np.abs(pred - r.pred) > MARGIN * r.tol_pred + EPS * np.abs(r.pred)).sum())
    return bad


def _step(m, batch, **kw):
    W, H = _state(m)
    pred, flags, _ = _launch(m, batch, **kw)
    W2, H2 = _state(m)
    r = _replay(m, W, H, batch, predict_only=kw.get("predict_only", False))
    assert _violations(r, W2, H2, pred) == 0, ((np.abs(W2 - r.table) / np.maximum(r.tol, 1e-30)).max(),
                                              (np.abs(H2 - r.acc) / np.maximum(r.tol_acc, 1e-30)).max())
    assert _padding_ok(m, W, W2) and _padding_ok(m, H, H2) and (H2[m.num_features] == 0).all()
    assert int(flags[0]) == 0 and int(flags[1]) == int(r.bad_id)
    return r, (W, H), (W2, H2), pred


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


@pytest.mark.parametrize("k, F", [(4, 39), (17, 2), (64, 1)])
def test_grid_stride_rounds_and_one_cta_are_bitwise_equal(k, F):
    out = []
    for max_ctas in (0, 1, 3):
        m = _model(k, F, reg=(0.01, 0.01))
        batch = _batch(np.random.default_rng(k + F), 900, F, m.num_features, nnz=(0, 3), nan_every=13)
        if max_ctas == 0:
            _, _, (W2, H2), pred = _step(m, batch)
        else:
            pred, _, _ = _launch(m, batch, max_ctas=max_ctas)
            W2, H2 = _state(m)
        out.append((W2, H2, pred, m.num_features))
        m.close()
    nf = out[0][3]
    for W2, H2, pred, _ in out[1:]:
        assert (pred == out[0][2]).all() and (W2[:nf] == out[0][0][:nf]).all() and (H2 == out[0][1]).all()


def test_edges_long_example_bad_entries_nan_and_short_cols():
    k, F, nf = 4, 256, 4096
    m = _model(k, F, reg=(0.01, 0.02), nf=nf)
    rng = np.random.default_rng(7)
    rp, cols, fields, vals, labels = _batch(rng, 60, F, nf, nnz=(0, 4), nan_every=5, hi=1500)
    rp = np.concatenate([rp, [rp[-1]]])                          # an empty example
    labels = np.concatenate([labels, [1.0]])
    # one example of 320 entries: 256 kept, every field once, and 64 skipped entries spread through it
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
    rp = np.concatenate([rp, [len(cols) + 5]])                 # ends past nnz: clamped
    labels = np.concatenate([labels, [1.0]]).astype(np.float32)
    r, (W, H), (W2, H2), pred = _step(m, (rp, cols, fields, vals, labels))
    assert r.bad_id
    for ex in np.nonzero(np.isnan(labels))[0]:                 # NaN-labelled examples leave H alone
        assert (H2[cols[rp[ex]:rp[ex + 1]]] == H[cols[rp[ex]:rp[ex + 1]]]).all()
    assert (H2[ids, 4:] != H[ids, 4:]).sum() >= 255 * k        # the long example's slabs gathered gam^2
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
    fields = rng.integers(0, F, nnz).astype(np.int32)
    if kind == "zipf":
        cols = np.minimum(rng.zipf(1.3, nnz), nf - 2)
    else:
        cols = rng.permutation(np.arange(1, nf - 1))[:nnz]
        if kind == "shared":
            cols[1::7] = cols[0::7][: len(cols[1::7])]
    cols = cols.astype(np.int64)
    vals = rng.normal(0, 1.0, nnz).astype(np.float32)
    labels = rng.integers(0, 2, n).astype(np.float32)
    batch = (rp, cols, fields, vals, labels)
    W, H = _state(m)
    pred, flags, _ = _launch(m, batch)
    W2, H2 = _state(m)
    fwd = _replay(m, W, H, batch)
    order = np.arange(n)[::-1]
    rrp = np.concatenate([[0], np.cumsum(np.diff(rp)[order])]).astype(np.int64)
    seg = lambda a: np.concatenate([a[rp[i]:rp[i + 1]] for i in order])
    others = (_replay(m, W, H, (rrp, seg(cols), seg(fields), seg(vals), labels[order])),
              _replay(m, W, H, batch, stale=True), _replay(m, W, H, batch, repull=True))
    pushes = np.bincount(cols, minlength=nf + 1)[:, None]
    for got, before, key, tkey in ((W2, W, "table", "tol"), (H2, H, "acc", "tol_acc")):
        spread = np.maximum.reduce([np.abs(fwd[key] - o[key]) for o in others])
        bound = 2 * np.maximum(pushes, 1) * spread + MARGIN * (fwd[tkey] + sum(o[tkey] for o in others)) + 1e-7
        err = np.abs(got - fwd[key])
        if kind == "multi_hot":
            assert (err <= bound).all(), (key, (err / bound).max())
        else:
            # the whole-update norm check of DESIGN §2.16, with the replays' spread now including H
            upd = np.linalg.norm(fwd[key] - before)
            rel = np.linalg.norm(got - fwd[key]) / upd
            spread_rel = max(np.linalg.norm(fwd[key] - o[key]) / upd for o in others)
            print(f"\nFFM_ADAGRAD_SHARED {kind} {key}: |kernel - replay| / |update| = {rel:.2e}, "
                  f"replays' spread {spread_rel:.2e}")
            assert rel <= 2 * spread_rel + 1e-6
    assert np.isfinite(W2).all() and np.isfinite(H2).all()
    assert _padding_ok(m, W, W2) and _padding_ok(m, H, H2) and int(flags[0]) == 0
    m.close()


def test_no_host_sync_and_one_launch_per_step():
    from fps_b200.ops import native

    m = _model(8, 4)
    rng = np.random.default_rng(2)
    rp, cols, fields, vals, labels = _batch(rng, 256, 4, m.num_features)
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


def test_broken_replays_fail():
    counts = {b: 0 for b in fm_ref.ADAGRAD_BREAKS}
    cases = 0
    for i, (k, F) in enumerate([(k, F) for k in (1, 4, 5, 8, 9, 16, 17, 33, 64) for F in (2, 39)]):
        m = _model(k, F, reg=(0.05, 0.05))
        rng = np.random.default_rng(300 + i)
        batch = _batch(rng, 150, F, m.num_features, nnz=(2, 6))
        W, H = _state(m)
        pred, _, _ = _launch(m, batch)
        W2, H2 = _state(m)
        assert _violations(_replay(m, W, H, batch), W2, H2, pred) == 0
        for b in fm_ref.ADAGRAD_BREAKS:
            counts[b] += _violations(_replay(m, W, H, batch, breaks=b), W2, H2, pred) > 0
        cases += 1
        m.close()
    print(f"\nFFM_ADAGRAD_SENSITIVITY failing cases of {cases}: {counts}")
    assert all(c > cases // 2 for c in counts.values()), counts


def _fit_device(kind, lr, reg_factors=0.0, k=4):
    from fps_b200.models.fm import DeviceFactorizationMachine, DeviceFieldAwareFM, roc_auc

    q = QUALITY
    torch.cuda.set_device(0)
    if kind == "ffm":
        m = DeviceFieldAwareFM(q["num_features"], q["fields"], k, learning_rate=lr, reg_factors=reg_factors,
                               init_range=(-0.1, 0.1), seed=QUALITY_SEED, optimizer="adagrad")
    else:
        m = DeviceFactorizationMachine(q["num_features"], k, learning_rate=lr, reg_factors=reg_factors,
                                       init_range=(-0.1, 0.1), seed=QUALITY_SEED, optimizer="adagrad")
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


def test_quality_sweep_and_libffm_defaults_through_the_public_models():
    aucs = {lr: _fit_device("ffm", lr) for lr in QUALITY_LRS}
    p = LIBFFM
    ffm = _fit_device("ffm", p["lr"], p["reg_factors"], p["k"])
    fm = _fit_device("fm", p["lr"], p["reg_factors"], p["k"])
    lin = _fit_device("fm", p["lr"], p["reg_factors"], 0)
    print(f"\nFFM_ADAGRAD_QUALITY device AUC per lr: {aucs}; at libffm's defaults FFM {ffm:.4f} FM {fm:.4f} "
          f"linear {lin:.4f}")
    # at lr 0.5 the kernel's races over features shared inside a 64-example batch (240 features) move the result
    # further from the CSR-order replay: 0.700 against 0.715 on the H100
    for lr, auc in aucs.items():
        assert abs(auc - AUC_ADAGRAD[lr]) <= (0.02 if lr >= 0.5 else 0.01), (lr, auc, AUC_ADAGRAD[lr])
    assert abs(ffm - AUC_LIBFFM_FFM) <= 0.01 and abs(fm - AUC_LIBFFM_FM) <= 0.01
    assert abs(lin - AUC_LIBFFM_LINEAR) <= 0.01
    assert ffm > fm and ffm > lin


def test_host_step_and_accumulator_round_trip():
    m = _model(6, 3, nf=64)
    ex = [[(0, 5, 1.0), (1, 9, 0.5), (2, 11, 2.0)], [(2, 7, 1.0)], []]
    m.step(ex, [1.0, None, 0.0])
    ids, H = m.accumulators()
    assert H.shape == (len(ids), m.table.stride)
    m2 = _model(6, 3, nf=64)
    m2.load_model(m.model(only_nonzero=False))
    m2.load_accumulators(ids, H)
    assert np.array_equal(m2.accumulators()[1], H)
    assert m.step(ex, [1.0, None, 0.0]) == m2.step(ex, [1.0, None, 0.0])
    assert np.array_equal(m.accumulators()[1], m2.accumulators()[1])
    m.check()
    m.close()
    m2.close()


def test_multi_rank_ffm_adagrad():
    from tests.test_gpu_multi import _run

    _run("mp_ffm_adagrad_check.py", 2, 29654, "MP_FFM_ADAGRAD_CHECK_OK")
