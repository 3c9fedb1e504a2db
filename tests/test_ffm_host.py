"""The field-aware FM's fp64 replay (tests/ffm_ref.py) against calculus and a planted model, ``read_libffm``, the
refusals of its binding and model, and the ctypes mirror of ``FfmArgs``.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models.fm import DeviceFieldAwareFM, read_libffm, roc_auc
from fps_b200.ops import native
from fps_b200.utils.synthetic import planted_ffm
from tests import ffm_ref, fm_ref
from tests.philox_ref import init_rows_ref
from tests.test_native_records_host import _layout, _nvcc

# ---- the replay's update is -lr times the gradient ---------------------------------------------------------------

NF, NFIELDS = 12, 3


def _example(k, repeated, rng):
    kp = ffm_ref.kpad(k)
    W = np.zeros((NF + 1, ffm_ref.stride(NFIELDS, k)))
    W[:NF, 0] = rng.normal(0, 0.4, NF)
    for f in range(NFIELDS):
        W[:NF, 4 + f * kp: 4 + f * kp + k] = rng.normal(0, 0.4, (NF, k))
    W[NF, 0] = 0.3
    cols = np.array([1, 4, 7, 10] + ([4, 1] if repeated else []), dtype=np.int64)
    fields = np.array([0, 1, 2, 1] + ([2, 0] if repeated else []), dtype=np.int64)   # field 1 twice
    vals = rng.normal(0, 1.0, len(cols))
    return W, cols, fields, vals


CASES = [(loss, k, reg, rep) for loss in ("logistic", "squared") for k in (1, 5) for reg in ((0.0, 0.0), (0.1, 0.2))
         for rep in (False, True)]


@pytest.mark.parametrize("loss, k, reg, repeated", CASES)
def test_update_is_minus_lr_times_the_gradient(loss, k, reg, repeated):
    rng = np.random.default_rng(k * 7 + len(loss) + int(repeated))
    W, cols, fields, vals = _example(k, repeated, rng)
    y = 1.0 if loss == "logistic" else 0.7
    lr = 0.5
    kw = dict(num_features=NF, num_fields=NFIELDS, k=k, loss=loss, reg_linear=reg[0], reg_factors=reg[1])
    r = ffm_ref.replay(W, [0, len(cols)], cols, fields, vals, [y], lr=lr, fp32=False, **kw)
    step = r.table - W
    # fp64 autograd
    t = torch.tensor(W, dtype=torch.float64, requires_grad=True)
    ffm_ref.objective(t, cols, fields, torch.from_numpy(vals), y, xp=torch, **kw).backward()
    np.testing.assert_allclose(step, -lr * t.grad.numpy(), rtol=1e-10, atol=1e-12)
    # central finite differences on every element of the touched rows and on w0
    f = lambda M: float(ffm_ref.objective(M, cols, fields, vals, y, **kw))
    h = 1e-6
    for i in sorted(set(cols.tolist())) + [NF]:
        for c in range(1 if i == NF else W.shape[1]):
            Wp, Wm = W.copy(), W.copy()
            Wp[i, c] += h
            Wm[i, c] -= h
            fd = (f(Wp) - f(Wm)) / (2 * h)
            assert abs(step[i, c] + lr * fd) <= 1e-6 * (1 + abs(lr * fd)), (i, c, step[i, c], -lr * fd)
    # rows no entry touches do not move (lazy regularisation); padding and columns 1..3 stay 0
    untouched = np.setdiff1d(np.arange(NF), cols)
    assert (r.table[untouched] == W[untouched]).all()
    assert (r.table[:, 1:4] == 0).all()
    kp = ffm_ref.kpad(k)
    for fi in range(NFIELDS):
        assert (r.table[:, 4 + fi * kp + k: 4 + (fi + 1) * kp] == 0).all()


@pytest.mark.parametrize("loss", ["logistic", "squared"])
def test_w0_takes_the_mean_step_and_every_example_reads_it_before_the_launch(loss):
    rng = np.random.default_rng(3)
    W, cols, fields, vals = _example(3, False, rng)
    y = 0.0 if loss == "logistic" else -1.5
    kw = dict(num_features=NF, num_fields=NFIELDS, k=3, loss=loss, lr=0.25, fp32=False)
    r = ffm_ref.replay(W, [0, len(cols)], cols, fields, vals, [y], **kw)
    assert r.table[NF, 0] == W[NF, 0] - 0.25 * r.g[0]
    r2 = ffm_ref.replay(W, [0, 2, 4], cols[:4], fields[:4], vals[:4], [y, y], **kw)
    assert np.isclose(r2.table[NF, 0], W[NF, 0] - 0.25 * np.mean(r2.g))
    solo = ffm_ref.replay(W, [0, 2], cols[2:4], fields[2:4], vals[2:4], [y], **kw)
    assert r2.pred[1] == solo.pred[0]


def test_skipped_entries_short_examples_and_predict_only():
    rng = np.random.default_rng(5)
    W, _, _, vals = _example(2, False, rng)
    cols = np.array([1, NF, -1, 3, 5, 6], dtype=np.int64)
    fields = np.array([0, 1, 0, 2, NFIELDS, -1], dtype=np.int64)   # bad ids at 1, 2; bad fields at 4, 5
    vals = np.ones(6)
    r = ffm_ref.replay(W, [0, 2, 3, 9], cols, fields, vals, [1.0, np.nan, 0.0], num_features=NF,
                       num_fields=NFIELDS, k=2, lr=0.1)
    assert r.bad_id and r.labelled == 2
    # example 0 keeps one entry (no pair), example 2 keeps one (id 3): only w of ids 1 and 3 moves
    moved = np.nonzero((r.table != W).any(1))[0].tolist()
    assert moved == [1, 3, NF]
    assert (r.table[[1, 3], 1:] == W[[1, 3], 1:]).all()
    p = ffm_ref.replay(W, [0, 2, 3, 4], cols, fields, vals, None, num_features=NF, num_fields=NFIELDS, k=2,
                       predict_only=True)
    assert (p.table == W).all() and p.labelled == 0


def test_breaks_change_the_replay():
    rng = np.random.default_rng(9)
    W, cols, fields, vals = _example(6, False, rng)
    kw = dict(num_features=NF, num_fields=NFIELDS, k=6, loss="logistic", lr=0.3, reg_linear=0.05,
              reg_factors=0.05)
    rp, cols, fields, vals = [0, 3, 4], cols[:4], np.array([0, 1, 2, 0]), vals[:4]
    base = ffm_ref.replay(W, rp, cols, fields, vals, [1.0, 0.0], **kw)
    for b in ffm_ref.BREAKS:
        other = ffm_ref.replay(W, rp, cols, fields, vals, [1.0, 0.0], breaks=b, **kw)
        assert (np.abs(other.table - base.table) > 10 * (base.tol + other.tol)).any(), b


def test_fp32_bound_covers_an_fp32_evaluation():
    """The bound of yhat holds for a float32 evaluation in another order."""
    rng = np.random.default_rng(11)
    for k, F in ((1, 3), (4, 7), (17, 5), (64, 9)):
        kp = ffm_ref.kpad(k)
        nf = 40
        W = np.float32(rng.normal(0, 0.5, (nf + 1, ffm_ref.stride(F, k)))).astype(np.float64)
        W[nf, 0] = np.float32(0.25)
        m = 9
        cols = rng.permutation(nf)[:m]
        fields = rng.integers(0, F, m)
        vals = np.float32(rng.normal(0, 1, m)).astype(np.float64)
        r = ffm_ref.replay(W, [0, m], cols, fields, vals, [np.nan], num_features=nf, num_fields=F, k=k)
        W32, x32 = W.astype(np.float32), vals.astype(np.float32)
        acc = np.float32(0)
        for b in range(m - 1, 0, -1):
            for a in range(b - 1, -1, -1):
                va = W32[cols[a], 4 + fields[b] * kp: 4 + fields[b] * kp + k]
                vb = W32[cols[b], 4 + fields[a] * kp: 4 + fields[a] * kp + k]
                acc = np.float32(acc + np.float32(x32[a] * x32[b]) * np.float32(np.dot(va, vb)))
        lin = np.float32(np.sum(x32[::-1] * W32[cols[::-1], 0], dtype=np.float32))
        y32 = np.float32(np.float32(W32[nf, 0] + lin) + acc)
        assert abs(float(y32) - r.pred[0]) <= r.tol_pred[0] + 1e-7 * abs(r.pred[0]), k


# ---- quality on a planted field-aware model: these numbers are the thresholds of the GPU gate --------------------

QUALITY = dict(num_features=240, fields=6, planted_k=4, n_train=12000, n_test=4000, batch=64, epochs=3, seed=3)
QUALITY_LR = 0.1
QUALITY_SEED = 5
QUALITY_K = 4
# reached by the replays from the devices' initial tables (FFM, FM at the same k, FM with k = 0); each device AUC
# of tests/test_gpu_ffm.py must come within 0.01 of its replay, so FFM must beat the others by the replay's gap
# less 0.02
AUC_FFM, AUC_FM, AUC_LINEAR = 0.6929, 0.6394, 0.6498
AUC_MARGIN_FM = round(AUC_FFM - AUC_FM - 0.02, 4)
AUC_MARGIN_LINEAR = round(AUC_FFM - AUC_LINEAR - 0.02, 4)


def planted():
    q = QUALITY
    rp, c, f, l = planted_ffm(q["num_features"], q["fields"], q["planted_k"], q["n_train"] + q["n_test"], q["seed"])
    return rp.numpy(), c.numpy(), f.numpy(), l.numpy()


def initial_ffm_table(nf, F, k, seed, lo, hi):
    """The table ``DeviceFieldAwareFM`` starts from: the K4 init, then w, columns 1..3, padding and the bias row
    zeroed."""
    kp = ffm_ref.kpad(k)
    W = np.zeros((nf + 1, ffm_ref.stride(F, k)))
    W[:nf] = init_rows_ref(np.arange(nf), W.shape[1], seed, lo, hi)
    W[:, :4] = 0.0
    for f in range(F):
        W[:, 4 + f * kp + k: 4 + (f + 1) * kp] = 0.0
    W[nf] = 0.0
    return W


def fit_replay_ffm():
    q = QUALITY
    nf, F, n, B = q["num_features"], q["fields"], q["n_train"], q["batch"]
    rp, c, f, l = planted()
    W = initial_ffm_table(nf, F, QUALITY_K, QUALITY_SEED, -0.1, 0.1)
    kw = dict(num_features=nf, num_fields=F, k=QUALITY_K, loss="logistic")
    for _ in range(q["epochs"]):
        for b0 in range(0, n, B):
            b1 = min(b0 + B, n)
            s = slice(rp[b0], rp[b1])
            W = ffm_ref.replay(W, rp[b0:b1 + 1] - rp[b0], c[s], f[s], None, l[b0:b1], lr=QUALITY_LR, **kw).table
    pred = ffm_ref.replay(W, rp[n:] - rp[n], c[rp[n]:], f[rp[n]:], None, None, predict_only=True, **kw).pred
    return roc_auc(pred, l[n:])


def fit_replay_fm(k):
    q = QUALITY
    nf, n, B = q["num_features"], q["n_train"], q["batch"]
    rp, c, _, l = planted()
    W = np.zeros((nf + 1, 4 * -(-(1 + k) // 4)))
    W[:nf, 1:1 + k] = init_rows_ref(np.arange(nf), 1 + k, QUALITY_SEED, -0.1, 0.1)[:, 1:1 + k]
    kw = dict(num_features=nf, dim=1 + k, loss="logistic")
    for _ in range(q["epochs"]):
        for b0 in range(0, n, B):
            b1 = min(b0 + B, n)
            W = fm_ref.replay(W, rp[b0:b1 + 1] - rp[b0], c[rp[b0]:rp[b1]], None, l[b0:b1], lr=QUALITY_LR,
                              **kw).table
    pred = fm_ref.replay(W, rp[n:] - rp[n], c[rp[n]:], None, None, predict_only=True, **kw).pred
    return roc_auc(pred, l[n:])


def test_quality_ffm_beats_fm_and_linear_on_planted_data():
    ffm, fm, lin = fit_replay_ffm(), fit_replay_fm(QUALITY_K), fit_replay_fm(0)
    print(f"\nFFM_QUALITY replay held-out AUC: FFM k={QUALITY_K} {ffm:.4f}  FM k={QUALITY_K} {fm:.4f}  "
          f"linear {lin:.4f}")
    assert abs(ffm - AUC_FFM) < 5e-4 and abs(fm - AUC_FM) < 5e-4 and abs(lin - AUC_LINEAR) < 5e-4
    assert ffm > fm + AUC_MARGIN_FM and ffm > lin + AUC_MARGIN_LINEAR


# ---- libffm text --------------------------------------------------------------------------------------------------

def test_read_libffm(tmp_path):
    text = "1 0:3:1 1:17:0.5 2:4:1\n\n0 1:2:2.5\n-1\n"
    p = tmp_path / "a.ffm"
    p.write_text(text)
    for src in (str(p), p, text.splitlines()):
        rp, f, c, v, l = read_libffm(src)
        assert rp.tolist() == [0, 3, 4, 4] and rp.dtype == np.int64
        assert f.tolist() == [0, 1, 2, 1] and f.dtype == np.int32
        assert c.tolist() == [3, 17, 4, 2] and c.dtype == np.int64
        assert v.tolist() == [1.0, 0.5, 1.0, 2.5] and v.dtype == np.float32
        assert l.tolist() == [1.0, 0.0, -1.0] and l.dtype == np.float32
    rp, f, c, v, l = read_libffm([])
    assert rp.tolist() == [0] and len(c) == len(l) == 0
    # bounds are the model's: a negative field parses
    assert read_libffm(["1 -1:5:1"])[1].tolist() == [-1]


@pytest.mark.parametrize("line", ["1 0:3", "1 0:3:1:2", "x 0:3:1", "1 a:3:1", "1 0:3.5:1", "1 0:3:y"])
def test_read_libffm_refuses_malformed_tokens_naming_the_line(line):
    with pytest.raises(ValueError, match="line 2: malformed"):
        read_libffm(["0 0:1:1", line])


# ---- refusals, before the library loads ---------------------------------------------------------------------------

@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the kernel library was loaded before the refusal")
    monkeypatch.setattr(native, "lib", refuse)


def _tab(F=3, k=4):
    t = native.ShardTableC()
    t.dim = t.stride = native.ffm_stride(F, k)
    return t


def _args(n=3, nnz=5, **over):
    a = dict(tab=_tab(), row_ptr=torch.zeros(n + 1, dtype=torch.int64), cols=torch.zeros(nnz, dtype=torch.int32),
             fields=torch.zeros(nnz, dtype=torch.int32), vals=torch.ones(nnz), labels=torch.zeros(n),
             pred=torch.empty(n))
    a.update(over)
    return a


def _call(loss="logistic", extra=None, num_fields=3, num_factors=4, **over):
    a = _args(**over)
    return native.ffm_step(a["tab"], a["row_ptr"], a["cols"], a["fields"], a["vals"], a["labels"], a["pred"],
                           num_features=10, num_fields=num_fields, num_factors=num_factors, loss=loss,
                           bias_state=(None, None), **(extra or {}))


@pytest.mark.parametrize("over, err, match", [
    (dict(row_ptr=torch.zeros(4, dtype=torch.int32)), TypeError, "row_ptr must be"),
    (dict(cols=torch.zeros(5, dtype=torch.float32)), TypeError, "cols must be int32 or int64"),
    (dict(fields=torch.zeros(5, dtype=torch.int64)), TypeError, "fields must be"),
    (dict(fields=torch.zeros(4, dtype=torch.int32)), ValueError, "cols and fields must have the same length"),
    (dict(vals=torch.ones(5, dtype=torch.float64)), TypeError, "vals must be"),
    (dict(vals=torch.ones(4)), ValueError, "cols and vals must have the same length"),
    (dict(labels=torch.zeros(3, dtype=torch.float64)), TypeError, "labels must be"),
    (dict(labels=torch.zeros(2)), ValueError, "one entry per example"),
    (dict(pred=torch.empty(3, dtype=torch.float64)), TypeError, "pred must be"),
    (dict(pred=torch.empty(4)), ValueError, "one entry per example"),
    (dict(row_ptr=torch.zeros(0, dtype=torch.int64)), ValueError, "n \\+ 1 offsets"),
    (dict(tab=_tab(3, 5)), ValueError, "rows must be 16 floats"),
], ids=["row_ptr-dtype", "cols-dtype", "fields-dtype", "fields-length", "vals-dtype", "vals-length", "labels-dtype",
        "labels-length", "pred-dtype", "pred-length", "row_ptr-empty", "stride"])
def test_ffm_step_refuses_bad_tensors(no_library, over, err, match):
    with pytest.raises(err, match=match):
        _call(**over)


def test_ffm_step_refuses_bad_arguments(no_library):
    with pytest.raises(ValueError, match="loss must be one of"):
        _call(loss="hinge")
    with pytest.raises(ValueError, match=">= 0"):
        _call(extra=dict(reg_factors=-0.1))
    with pytest.raises(ValueError, match="num_factors must lie in \\[1, 64\\]"):
        _call(num_factors=65)
    with pytest.raises(ValueError, match="num_factors must lie"):
        _call(num_factors=0)
    with pytest.raises(ValueError, match="num_fields must lie in \\[1, 256\\]"):
        _call(num_fields=257)
    a = _args()
    with pytest.raises(ValueError, match="needs labels"):
        native.ffm_step(a["tab"], a["row_ptr"], a["cols"], a["fields"], a["vals"], None, a["pred"], num_features=10,
                        num_fields=3, num_factors=4, bias=False)
    with pytest.raises(ValueError, match="bias_state"):
        native.ffm_step(a["tab"], a["row_ptr"], a["cols"], a["fields"], a["vals"], a["labels"], a["pred"],
                        num_features=10, num_fields=3, num_factors=4)


@pytest.mark.parametrize("kw, match", [
    (dict(num_factors=65), "num_factors must lie in \\[1, 64\\].*DeviceFactorizationMachine\\(num_factors=0\\)"),
    (dict(num_factors=0), "DeviceFactorizationMachine\\(num_factors=0\\)"),
    (dict(num_fields=0), "num_fields must lie in \\[1, 256\\]"),
    (dict(num_fields=257), "num_fields must lie in \\[1, 256\\]"),
    (dict(loss="hinge"), "loss must be one of"),
    (dict(reg_linear=-1.0), "must be >= 0"),
    (dict(reg_factors=float("nan")), "must be >= 0"),
    (dict(partition="lut"), "partition must be"),
    (dict(replica=True), "direct mode only: use replica=False"),
    (dict(num_features=0), "num_features must be >= 1"),
])
def test_model_refuses_bad_configuration(no_library, kw, match):
    args = dict(num_features=100, num_fields=4, num_factors=8)
    args.update(kw)
    nf, F, k = args.pop("num_features"), args.pop("num_fields"), args.pop("num_factors")
    with pytest.raises(ValueError, match=match):
        DeviceFieldAwareFM(nf, F, k, **args)


def test_host_step_refuses_labels_features_and_fields_before_copying(no_library):
    m = object.__new__(DeviceFieldAwareFM)
    m.num_features, m.num_fields, m.loss = 10, 3, "logistic"
    good = [[(0, 1, 1.0), (2, 9, 0.5)], [(1, 3, 1.0)]]
    with pytest.raises(ValueError, match="logistic labels must be 0 or 1"):
        m.step(good, [0.5, 1.0])
    with pytest.raises(ValueError, match="2 examples but 1 labels"):
        m.step(good, [1.0])
    with pytest.raises(ValueError, match="feature ids must lie in \\[0, 10\\)"):
        m.step([[(0, 10, 1.0)]], [1.0])
    with pytest.raises(ValueError, match="feature ids must lie"):
        m.step([[(0, -1, 1.0)]], [None])
    with pytest.raises(ValueError, match="fields must lie in \\[0, 3\\)"):
        m.step([[(3, 1, 1.0)]], [0.0])
    m.loss = "squared"
    with pytest.raises(ValueError, match="squared-loss labels must be finite"):
        m.step(good, [float("inf"), 1.0])


# ---- the ctypes mirror of FfmArgs --------------------------------------------------------------------------------

@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_ffm_args_mirror_matches_the_c_layout(tmp_path):
    mirror = native.FfmArgsC
    lines = ['  printf("sizeof %zu\\n", sizeof(FfmArgs));']
    lines += [f'  printf("{f} %zu\\n", offsetof(FfmArgs, {f}));' for f, _ in mirror._fields_]
    want = {f: str(getattr(mirror, f).offset) for f, _ in mirror._fields_}
    want["sizeof"] = str(C.sizeof(mirror))
    assert _layout(tmp_path, "fps_ffm.cu", lines) == want


def test_lane_rungs_and_strides():
    assert [ffm_ref.lanes(k) for k in (1, 4, 5, 8, 9, 16, 17, 32, 33, 64)] == [1, 1, 2, 2, 4, 4, 8, 8, 16, 16]
    assert native.ffm_stride(39, 4) == 160 and native.ffm_stride(1, 1) == 8 and native.ffm_stride(256, 64) == 16388
    assert ffm_ref.stride(39, 5) == native.ffm_stride(39, 5)
