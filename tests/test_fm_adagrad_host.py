"""AdaGrad in the factorization machine's fp64 replay (tests/fm_ref.py, DESIGN §2.17) against autograd, its breaks
and error model, a planted model, the refusals of the binding and model, and the ``acc`` field of ``FmArgs``.
No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models.fm import DeviceFactorizationMachine, check_fm_config, roc_auc
from fps_b200.ops import native
from tests import fm_ref
from tests.philox_ref import init_rows_ref
from tests.test_fm_host import NF, QUALITY, QUALITY_SEED, _args, _example, no_library, planted  # noqa: F401
from tests.test_native_records_host import _layout, _nvcc

EPS = fm_ref.EPS


def _acc_like(W, rng):
    """A non-trivial accumulator table: H >= 0 on every element of the feature rows, 0 on the padding."""
    H = np.zeros_like(W)
    H[:NF] = np.where(W[:NF] != 0, rng.uniform(0, 2.0, W[:NF].shape), 0.0)
    return H


@pytest.mark.parametrize("loss", ["logistic", "squared"])
@pytest.mark.parametrize("k", [0, 1, 5, 127, 511])
@pytest.mark.parametrize("reg", [(0.0, 0.0), (0.1, 0.2)])
def test_update_is_adagrad_of_the_gradient(loss, k, reg):
    rng = np.random.default_rng(k * 3 + len(loss))
    W, cols, vals = _example(k, False, rng)
    H = _acc_like(W, rng)
    y = 1.0 if loss == "logistic" else 0.7
    lr = 0.5
    kw = dict(num_features=NF, dim=1 + k, loss=loss, reg_linear=reg[0], reg_factors=reg[1])
    r = fm_ref.replay(W, [0, len(cols)], cols, vals, [y], lr=lr, fp32=False, acc=H, **kw)
    t = torch.tensor(W[:, : 1 + k], dtype=torch.float64, requires_grad=True)
    fm_ref.objective(t, torch.from_numpy(cols), torch.from_numpy(vals), y, xp=torch, **kw).backward()
    gam = t.grad.numpy()
    rows = np.unique(cols)
    want = -lr * gam[rows] / np.sqrt(1.0 + H[rows, : 1 + k] + gam[rows] ** 2)
    np.testing.assert_allclose((r.table - W)[rows, : 1 + k], want, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose((r.acc - H)[rows, : 1 + k], gam[rows] ** 2, rtol=1e-10, atol=1e-13)
    untouched = np.setdiff1d(np.arange(NF), cols)
    assert (r.table[untouched] == W[untouched]).all() and (r.acc[untouched] == H[untouched]).all()
    assert (r.table[:, 1 + k:] == 0).all() and (r.acc[:, 1 + k:] == 0).all()
    # w0 keeps the SGD step
    assert r.table[NF, 0] == W[NF, 0] - lr * r.g[0] and r.acc[NF, 0] == 0


def test_without_acc_the_replay_is_unchanged():
    rng = np.random.default_rng(2)
    W, cols, vals = _example(6, True, rng)
    kw = dict(num_features=NF, dim=7, loss="logistic", lr=0.3, reg_linear=0.05, reg_factors=0.05)
    b = fm_ref.replay(W, [0, 3, 6], cols, vals, [1.0, 0.0], acc=None, acc_tol=None, **kw)
    assert b.acc is None and b.tol_acc is None
    with pytest.raises(ValueError, match="unknown break"):
        fm_ref.replay(W, [0, 3, 6], cols, vals, [1.0, 0.0], breaks="acc_abs", **kw)


def test_adagrad_breaks_change_the_replay():
    rng = np.random.default_rng(9)
    W, cols, vals = _example(6, False, rng)
    H = _acc_like(W, rng)
    kw = dict(num_features=NF, dim=7, loss="logistic", lr=0.3, reg_linear=0.05, reg_factors=0.05, acc=H)
    base = fm_ref.replay(W, [0, 2, 4], cols[:4], vals[:4], [1.0, 0.0], **kw)
    for b in fm_ref.ADAGRAD_BREAKS:
        other = fm_ref.replay(W, [0, 2, 4], cols[:4], vals[:4], [1.0, 0.0], breaks=b, **kw)
        moved = (np.abs(other.table - base.table) > 10 * (base.tol + other.tol)).any()
        moved |= (np.abs(other.acc - base.acc) > 10 * (base.tol_acc + other.tol_acc)).any()
        assert moved, b


def test_fp32_bound_covers_an_fp32_evaluation():
    """adagrad()'s bound holds for the kernel's float32 step from a gam off by its own bound."""
    rng = np.random.default_rng(11)
    n = 20000
    gam = rng.normal(0, 1, n) * 10.0 ** rng.uniform(-4, 2, n)
    H = np.float32(rng.uniform(0, 1, n) * 10.0 ** rng.uniform(-3, 3, n)).astype(np.float64)
    tgam = 4 * EPS * np.abs(gam)
    gam32 = np.float32(gam * (1 + rng.choice([-1, 1], n) * 3 * EPS))   # within tgam with its own rounding
    lr = np.float32(0.2)
    d, td, dh, tdh = fm_ref.adagrad(gam, tgam, H, np.zeros(n), float(lr))
    gg32 = gam32 * gam32
    d32 = -lr * gam32 / np.sqrt(np.float32(np.float32(1) + np.float32(H)) + gg32)
    assert d32.dtype == np.float32
    assert (np.abs(d32 - d) <= td).all(), (np.abs(d32 - d) / td).max()
    assert (np.abs(gg32 - dh) <= tdh).all()


# ---- quality on the planted FM: these numbers are the thresholds of the GPU gate ---------------------------------

QUALITY_LRS = (0.02, 0.1, 0.5)
# held-out AUC (logistic, k = 4) of the fp64 replays from the device's initial table, per learning rate; the
# AdaGrad ones gate tests/test_gpu_fm_adagrad.py within 0.01, the SGD ones are DESIGN §2.17's comparison
AUC_ADAGRAD = {0.02: 0.6945, 0.1: 0.8195, 0.5: 0.8374}
AUC_SGD = {0.02: 0.7414, 0.1: 0.7761, 0.5: 0.5078}


def fit_replay(k, lr, optimizer, reg=(0.0, 0.0), planted_data=None):
    """Train the replay over ``QUALITY``'s planted data for its epochs and return the held-out AUC."""
    q = QUALITY
    nf, n, B = q["num_features"], q["n_train"], q["batch"]
    rp, c, l = planted("logistic") if planted_data is None else planted_data
    W = np.zeros((nf + 1, 4 * -(-(1 + k) // 4)))
    W[:nf, 1:1 + k] = init_rows_ref(np.arange(nf), 1 + k, QUALITY_SEED, -0.1, 0.1)[:, 1:1 + k]
    H = np.zeros_like(W) if optimizer == "adagrad" else None
    kw = dict(num_features=nf, dim=1 + k, loss="logistic", reg_linear=reg[0], reg_factors=reg[1])
    for _ in range(q["epochs"]):
        for b0 in range(0, n, B):
            b1 = min(b0 + B, n)
            r = fm_ref.replay(W, rp[b0:b1 + 1] - rp[b0], c[rp[b0]:rp[b1]], None, l[b0:b1], lr=lr, acc=H, **kw)
            W, H = r.table, r.acc
    pred = fm_ref.replay(W, rp[n:] - rp[n], c[rp[n]:], None, None, predict_only=True, **kw).pred
    return roc_auc(pred, l[n:])


@pytest.mark.parametrize("lr", QUALITY_LRS)
def test_quality_replay_sweep(lr):
    ada, sgd = fit_replay(4, lr, "adagrad"), fit_replay(4, lr, "sgd")
    print(f"\nFM_ADAGRAD_QUALITY replay lr={lr}: AdaGrad AUC {ada:.4f}  SGD AUC {sgd:.4f}")
    assert abs(ada - AUC_ADAGRAD[lr]) < 5e-4 and abs(sgd - AUC_SGD[lr]) < 5e-4


# ---- refusals, before the library loads ---------------------------------------------------------------------------

def _tab(stride=8, dim=6, rows=100, base=0x1000):
    t = native.ShardTableC()
    t.base[0], t.stride, t.dim, t.rows_per_shard, t.div, t.num_shards = base, stride, dim, rows, rows, 1
    return t


@pytest.mark.parametrize("field, value", [("stride", 12), ("dim", 5), ("rows_per_shard", 99), ("div", 7),
                                          ("num_shards", 2), ("mode", 1)])
def test_fm_step_refuses_an_accumulator_of_another_geometry(no_library, field, value):
    acc = _tab(base=0x2000)
    setattr(acc, field, value)
    a = _args()
    with pytest.raises(ValueError, match="accumulator table's geometry"):
        native.fm_step(_tab(), a["row_ptr"], a["cols"], a["vals"], a["labels"], a["pred"], num_features=10,
                       bias=False, acc=acc)


def test_fm_step_refuses_an_accumulator_that_is_not_a_table(no_library):
    a = _args()
    with pytest.raises(TypeError, match="acc must be a ShardTableC"):
        native.fm_step(_tab(), a["row_ptr"], a["cols"], a["vals"], a["labels"], a["pred"], num_features=10,
                       bias=False, acc=torch.zeros(8))
    with pytest.raises(ValueError, match="no shard 0"):
        native.fm_step(_tab(), a["row_ptr"], a["cols"], a["vals"], a["labels"], a["pred"], num_features=10,
                       bias=False, acc=_tab(base=0))


def test_model_refuses_an_unknown_optimizer(no_library):
    with pytest.raises(ValueError, match=r"optimizer must be one of \['sgd', 'adagrad'\]"):
        DeviceFactorizationMachine(100, 8, optimizer="ftrl")
    with pytest.raises(ValueError, match="optimizer must be one of"):
        check_fm_config(100, 0, "logistic", 0.0, 0.0, "hash", False, optimizer="Adagrad")
    check_fm_config(100, 0, "logistic", 0.0, 0.0, "hash", False, optimizer="adagrad")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_fm_args_acc_is_appended_to_the_c_layout(tmp_path):
    mirror = native.FmArgsC
    assert mirror._fields_[-1] == ("acc", native.ShardTableC)
    lines = ['  printf("sizeof %zu\\n", sizeof(FmArgs));', '  printf("acc %zu\\n", offsetof(FmArgs, acc));']
    assert _layout(tmp_path, "fps_fm.cu", lines) == {"sizeof": str(C.sizeof(mirror)), "acc": str(mirror.acc.offset)}
