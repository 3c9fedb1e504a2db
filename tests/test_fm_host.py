"""The factorization machine's fp64 replay (tests/fm_ref.py) against calculus and a planted model, the refusals of
its binding and model, and the ctypes mirror of ``FmArgs``.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models import fm as fm_mod
from fps_b200.models.fm import DeviceFactorizationMachine, check_fm_batch, roc_auc
from fps_b200.models.pa.sparse import SparseVector
from fps_b200.ops import native
from fps_b200.utils.synthetic import planted_fm
from tests import fm_ref
from tests.philox_ref import init_rows_ref
from tests.test_native_records_host import _layout, _nvcc

# ---- the replay's update is -lr times the gradient ---------------------------------------------------------------

NF = 12


def _example(k, repeated, rng):
    stride = 4 * -(-(1 + k) // 4)
    W = np.zeros((NF + 1, stride))
    W[:NF, : 1 + k] = rng.normal(0, 0.4, (NF, 1 + k))
    W[NF, 0] = 0.3
    cols = np.array([1, 4, 7, 10] + ([4, 1] if repeated else []), dtype=np.int64)
    vals = rng.normal(0, 1.0, len(cols))
    return W, cols, vals


CASES = [(loss, k, reg, rep) for loss in ("logistic", "squared") for k in (0, 5) for reg in ((0.0, 0.0), (0.1, 0.2))
         for rep in (False, True)]


@pytest.mark.parametrize("loss, k, reg, repeated", CASES)
def test_update_is_minus_lr_times_the_gradient(loss, k, reg, repeated):
    rng = np.random.default_rng(k * 7 + len(loss) + int(repeated))
    W, cols, vals = _example(k, repeated, rng)
    y = 1.0 if loss == "logistic" else 0.7
    lr = 0.5
    kw = dict(num_features=NF, dim=1 + k, loss=loss, reg_linear=reg[0], reg_factors=reg[1])
    r = fm_ref.replay(W, [0, len(cols)], cols, vals, [y], lr=lr, fp32=False, **kw)
    step = (r.table - W)[:, : 1 + k]
    # fp64 autograd
    t = torch.tensor(W[:, : 1 + k], dtype=torch.float64, requires_grad=True)
    fm_ref.objective(t, torch.from_numpy(cols), torch.from_numpy(vals), y, xp=torch, **kw).backward()
    np.testing.assert_allclose(step, -lr * t.grad.numpy(), rtol=1e-10, atol=1e-12)
    # central finite differences on every touched element and on w0
    f = lambda M: float(fm_ref.objective(M, cols, vals, y, **kw))
    h = 1e-6
    for i in sorted(set(cols.tolist())) + [NF]:
        for c in range(1 if i == NF else 1 + k):
            Wp, Wm = W[:, : 1 + k].copy(), W[:, : 1 + k].copy()
            Wp[i, c] += h
            Wm[i, c] -= h
            fd = (f(Wp) - f(Wm)) / (2 * h)
            assert abs(step[i, c] + lr * fd) <= 1e-6 * (1 + abs(lr * fd)), (i, c, step[i, c], -lr * fd)
    # rows no entry touches do not move (lazy regularisation), and the padding stays 0
    untouched = np.setdiff1d(np.arange(NF), cols)
    assert (r.table[untouched] == W[untouched]).all()
    assert (r.table[:, 1 + k:] == 0).all()


@pytest.mark.parametrize("loss", ["logistic", "squared"])
def test_one_example_batch_is_plain_sgd_on_w0(loss):
    rng = np.random.default_rng(3)
    W, cols, vals = _example(3, False, rng)
    y = 0.0 if loss == "logistic" else -1.5
    r = fm_ref.replay(W, [0, len(cols)], cols, vals, [y], num_features=NF, dim=4, loss=loss, lr=0.25, fp32=False)
    assert r.table[NF, 0] == W[NF, 0] - 0.25 * r.g[0]
    # two examples: the bias takes the mean gradient once, and both predictions use the pre-launch w0
    r2 = fm_ref.replay(W, [0, 2, 4], cols[:4], vals[:4], [y, y], num_features=NF, dim=4, loss=loss, lr=0.25,
                       fp32=False)
    assert np.isclose(r2.table[NF, 0], W[NF, 0] - 0.25 * np.mean(r2.g))
    solo = fm_ref.replay(W, [0, 2], cols[2:4], vals[2:4], [y], num_features=NF, dim=4, loss=loss, lr=0.25,
                         fp32=False)
    assert r2.pred[1] == solo.pred[0]


def test_predict_only_nan_labels_bad_ids_and_short_cols():
    rng = np.random.default_rng(5)
    W, cols, vals = _example(2, False, rng)
    cols = np.array([1, NF, -1, 3], dtype=np.int64)
    r = fm_ref.replay(W, [0, 2, 3, 9], cols, vals, [1.0, np.nan, 0.0], num_features=NF, dim=3, lr=0.1)
    assert r.bad_id and r.labelled == 2
    assert (r.table[NF, 1:] == 0).all()
    untouched = np.setdiff1d(np.arange(NF), [1, 3])
    assert (r.table[untouched] == W[untouched]).all()
    p = fm_ref.replay(W, [0, 2, 3, 4], cols, vals, None, num_features=NF, dim=3, predict_only=True)
    assert (p.table == W).all() and p.labelled == 0


def test_breaks_change_the_replay():
    rng = np.random.default_rng(9)
    W, cols, vals = _example(6, False, rng)
    kw = dict(num_features=NF, dim=7, loss="logistic", lr=0.3, reg_linear=0.05, reg_factors=0.05)
    base = fm_ref.replay(W, [0, 2, 4], cols[:4], vals[:4], [1.0, 0.0], **kw)
    for b in fm_ref.BREAKS:
        other = fm_ref.replay(W, [0, 2, 4], cols[:4], vals[:4], [1.0, 0.0], breaks=b, **kw)
        assert (np.abs(other.table - base.table) > 10 * (base.tol + other.tol)).any(), b


def test_fp32_bound_covers_an_fp32_evaluation():
    """The bound of yhat holds for a float32 evaluation in a different order."""
    rng = np.random.default_rng(11)
    for k in (0, 3, 17, 200):
        stride = 4 * -(-(1 + k) // 4)
        W = np.zeros((NF + 1, stride))
        W[:NF, : 1 + k] = np.float32(rng.normal(0, 0.5, (NF, 1 + k)))
        W[NF, 0] = np.float32(0.25)
        cols = rng.permutation(NF)[:7]
        vals = np.float32(rng.normal(0, 1, 7)).astype(np.float64)
        r = fm_ref.replay(W, [0, 7], cols, vals, [np.nan], num_features=NF, dim=1 + k)
        W32, x32 = W.astype(np.float32), vals.astype(np.float32)
        xv = x32[::-1, None] * W32[cols[::-1], 1:1 + k]
        s = np.float32(0)
        for f in range(k):
            col = np.float32(0)
            for t in xv[:, f]:
                col = np.float32(col + t)
            s = np.float32(s + np.float32(col * col))
        sq = np.float32(np.sum(xv * xv, dtype=np.float32))
        lin = np.float32(np.sum(x32[::-1] * W32[cols[::-1], 0], dtype=np.float32))
        y32 = np.float32(W32[NF, 0] + lin + np.float32(0.5) * np.float32(s - sq))
        assert abs(float(y32) - r.pred[0]) <= r.tol_pred[0] + 1e-7 * abs(r.pred[0]), k


# ---- quality on a planted model: these numbers are the thresholds of the GPU gate --------------------------------

QUALITY = dict(num_features=240, fields=6, planted_k=4, n_train=12000, n_test=4000, batch=64, epochs=3, seed=3)
QUALITY_LR = {"logistic": 0.05, "squared": 0.0125}
QUALITY_SEED = 5
# reached by this replay from the device's initial table; tests/test_gpu_fm.py must come within 0.01 of them
AUC_K4, AUC_K0 = 0.8107, 0.6692
RMSE_K4 = 0.2861


def planted(loss):
    q = QUALITY
    rp, c, l = planted_fm(q["num_features"], q["fields"], q["planted_k"], q["n_train"] + q["n_test"], q["seed"], loss)
    return rp.numpy(), c.numpy(), l.numpy()


def fit_replay(loss, k):
    q = QUALITY
    nf, n, B = q["num_features"], q["n_train"], q["batch"]
    rp, c, l = planted(loss)
    W = np.zeros((nf + 1, 4 * -(-(1 + k) // 4)))
    W[:nf, 1:1 + k] = init_rows_ref(np.arange(nf), 1 + k, QUALITY_SEED, -0.1, 0.1)[:, 1:1 + k]   # the K4 init
    kw = dict(num_features=nf, dim=1 + k, loss=loss)
    for _ in range(q["epochs"]):
        for b0 in range(0, n, B):
            b1 = min(b0 + B, n)
            W = fm_ref.replay(W, rp[b0:b1 + 1] - rp[b0], c[rp[b0]:rp[b1]], None, l[b0:b1], lr=QUALITY_LR[loss],
                              **kw).table
    pred = fm_ref.replay(W, rp[n:] - rp[n], c[rp[n]:], None, None, predict_only=True, **kw).pred
    if loss == "logistic":
        return roc_auc(pred, l[n:])
    return float(np.sqrt(np.mean((pred - l[n:]) ** 2)))


def test_quality_logistic_factors_beat_linear():
    auc4, auc0 = fit_replay("logistic", 4), fit_replay("logistic", 0)
    print(f"\nFM_QUALITY replay logistic held-out AUC: k=4 {auc4:.4f}  k=0 {auc0:.4f}")
    assert auc4 > auc0 + 0.1
    assert abs(auc4 - AUC_K4) < 5e-4 and abs(auc0 - AUC_K0) < 5e-4


def test_quality_squared_rmse():
    rmse = fit_replay("squared", 4)
    print(f"\nFM_QUALITY replay squared held-out RMSE: k=4 {rmse:.4f}")
    assert abs(rmse - RMSE_K4) < 5e-4


def test_roc_auc_with_ties():
    assert roc_auc([0.1, 0.4, 0.35, 0.8], [0, 0, 1, 1]) == 0.75
    assert roc_auc([1, 1, 1, 1], [0, 1, 0, 1]) == 0.5


# ---- refusals, before the library loads ---------------------------------------------------------------------------

@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the kernel library was loaded before the refusal")
    monkeypatch.setattr(native, "lib", refuse)


def _args(n=3, nnz=5, **over):
    a = dict(tab=native.ShardTableC(), row_ptr=torch.zeros(n + 1, dtype=torch.int64),
             cols=torch.zeros(nnz, dtype=torch.int32), vals=torch.ones(nnz), labels=torch.zeros(n),
             pred=torch.empty(n))
    a.update(over)
    return a


def _call(loss="logistic", extra=None, **over):
    a = _args(**over)
    return native.fm_step(a["tab"], a["row_ptr"], a["cols"], a["vals"], a["labels"], a["pred"], num_features=10,
                          loss=loss, bias_state=(None, None), **(extra or {}))


@pytest.mark.parametrize("over, err, match", [
    (dict(row_ptr=torch.zeros(4, dtype=torch.int32)), TypeError, "row_ptr must be"),
    (dict(cols=torch.zeros(5, dtype=torch.float32)), TypeError, "cols must be int32 or int64"),
    (dict(vals=torch.ones(5, dtype=torch.float64)), TypeError, "vals must be"),
    (dict(vals=torch.ones(4)), ValueError, "same length"),
    (dict(labels=torch.zeros(3, dtype=torch.float64)), TypeError, "labels must be"),
    (dict(labels=torch.zeros(2)), ValueError, "one entry per example"),
    (dict(pred=torch.empty(3, dtype=torch.float64)), TypeError, "pred must be"),
    (dict(pred=torch.empty(4)), ValueError, "one entry per example"),
    (dict(row_ptr=torch.zeros(0, dtype=torch.int64)), ValueError, "n \\+ 1 offsets"),
], ids=["row_ptr-dtype", "cols-dtype", "vals-dtype", "vals-length", "labels-dtype", "labels-length", "pred-dtype",
        "pred-length", "row_ptr-empty"])
def test_fm_step_refuses_bad_tensors(no_library, over, err, match):
    with pytest.raises(err, match=match):
        _call(**over)


def test_fm_step_refuses_bad_arguments(no_library):
    with pytest.raises(ValueError, match="loss must be one of"):
        _call(loss="hinge")
    with pytest.raises(ValueError, match=">= 0"):
        _call(extra=dict(reg_factors=-0.1))
    a = _args()
    with pytest.raises(ValueError, match="needs labels"):
        native.fm_step(a["tab"], a["row_ptr"], a["cols"], a["vals"], None, a["pred"], num_features=10,
                       bias=False)
    with pytest.raises(ValueError, match="bias_state"):
        native.fm_step(a["tab"], a["row_ptr"], a["cols"], a["vals"], a["labels"], a["pred"], num_features=10)


@pytest.mark.parametrize("kw, match", [
    (dict(num_factors=512), "num_factors must lie in \\[0, 511\\]"),
    (dict(num_factors=-1), "num_factors must lie"),
    (dict(loss="hinge"), "loss must be one of"),
    (dict(reg_linear=-1.0), "must be >= 0"),
    (dict(reg_factors=float("nan")), "must be >= 0"),
    (dict(partition="lut"), "partition must be"),
    (dict(replica=True), "direct mode only"),
    (dict(num_features=0), "num_features must be >= 1"),
])
def test_model_refuses_bad_configuration(no_library, kw, match):
    args = dict(num_features=100, num_factors=8)
    args.update(kw)
    nf, k = args.pop("num_features"), args.pop("num_factors")
    with pytest.raises(ValueError, match=match):
        DeviceFactorizationMachine(nf, k, **args)


def test_host_step_refuses_labels_and_ids_before_copying(no_library):
    v = [SparseVector([1, 3], [1.0, 2.0], 10), SparseVector([2], [1.0], 10)]
    with pytest.raises(ValueError, match="logistic labels must be 0 or 1"):
        check_fm_batch(v, [1.0, 2.0], 10, "logistic")
    with pytest.raises(ValueError, match="feature ids must lie in \\[0, 10\\)"):
        check_fm_batch([SparseVector([1, 10], [1.0, 1.0], 11)], [1.0], 10, "logistic")
    with pytest.raises(ValueError, match="feature ids must lie"):
        check_fm_batch([SparseVector([-1], [1.0], 11)], [1.0], 10, "squared")
    with pytest.raises(ValueError, match="2 vectors but 1 labels"):
        check_fm_batch(v, [1.0], 10, "logistic")
    lab = check_fm_batch(v, [None, 0.0], 10, "logistic")
    assert np.isnan(lab[0]) and lab[1] == 0 and lab.dtype == np.float32
    m = object.__new__(DeviceFactorizationMachine)
    m.num_features, m.loss = 10, "logistic"
    with pytest.raises(ValueError, match="logistic labels"):
        m.step(v, [0.5, 1.0])


# ---- the ctypes mirror of FmArgs ---------------------------------------------------------------------------------

@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_fm_args_mirror_matches_the_c_layout(tmp_path):
    mirror = native.FmArgsC
    lines = ['  printf("sizeof %zu\\n", sizeof(FmArgs));']
    lines += [f'  printf("{f} %zu\\n", offsetof(FmArgs, {f}));' for f, _ in mirror._fields_]
    want = {f: str(getattr(mirror, f).offset) for f, _ in mirror._fields_}
    want["sizeof"] = str(C.sizeof(mirror))
    assert _layout(tmp_path, "fps_fm.cu", lines) == want


def test_dispatch_rungs():
    assert fm_ref.rungs() == [(1, 1), (2, 1), (4, 1), (8, 1), (16, 1), (32, 1), (32, 2), (32, 3), (32, 4)]
    assert fm_mod.MAX_FACTORS == 511
