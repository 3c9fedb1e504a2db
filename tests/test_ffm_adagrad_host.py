"""AdaGrad in the field-aware FM's fp64 replay (tests/ffm_ref.py, DESIGN §2.17) against autograd, its breaks, a
planted field-aware model at libffm's settings, the refusals of the binding and model, and the ``acc`` field of
``FfmArgs``.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models.fm import DeviceFieldAwareFM, check_ffm_config, roc_auc
from fps_b200.ops import native
from tests import ffm_ref, fm_ref
from tests.test_ffm_host import (NF, QUALITY, QUALITY_SEED, _args, _example, initial_ffm_table,  # noqa: F401
                                 no_library, planted)
from tests.test_native_records_host import _layout, _nvcc


def _acc_like(W, rng, F, k):
    """H >= 0 on w and every slab's factors of the feature rows, 0 on columns 1..3 and the padding."""
    kp = ffm_ref.kpad(k)
    H = np.zeros_like(W)
    H[:NF, 0] = rng.uniform(0, 2.0, NF)
    for f in range(F):
        H[:NF, 4 + f * kp: 4 + f * kp + k] = rng.uniform(0, 2.0, (NF, k))
    return H


def _example_f(k, F, rng):
    """Rows of F fields, and one example over distinct features with distinct fields (two entries at F = 1), so no
    slab is pushed twice: AdaGrad steps each pair's push on its own, and autograd sums them."""
    kp = ffm_ref.kpad(k)
    W = np.zeros((NF + 1, ffm_ref.stride(F, k)))
    W[:NF, 0] = rng.normal(0, 0.4, NF)
    for f in range(F):
        W[:NF, 4 + f * kp: 4 + f * kp + k] = rng.normal(0, 0.4, (NF, k))
    W[NF, 0] = 0.3
    m = max(2, min(4, F))
    cols = np.array([1, 4, 7, 10][:m], dtype=np.int64)
    fields = np.arange(m, dtype=np.int64) % F
    return W, cols, fields, rng.normal(0, 1.0, m)


@pytest.mark.parametrize("loss", ["logistic", "squared"])
@pytest.mark.parametrize("k, F", [(1, 1), (4, 2), (5, 3), (17, 4), (64, 3)])
@pytest.mark.parametrize("reg", [(0.0, 0.0), (0.1, 0.2)])
def test_update_is_adagrad_of_the_gradient(loss, k, F, reg):
    rng = np.random.default_rng(k * 3 + F + len(loss))
    W, cols, fields, vals = _example_f(k, F, rng)
    H = _acc_like(W, rng, F, k)
    y = 1.0 if loss == "logistic" else 0.7
    lr = 0.5
    kw = dict(num_features=NF, num_fields=F, k=k, loss=loss, reg_linear=reg[0], reg_factors=reg[1])
    r = ffm_ref.replay(W, [0, len(cols)], cols, fields, vals, [y], lr=lr, fp32=False, acc=H, **kw)
    t = torch.tensor(W, dtype=torch.float64, requires_grad=True)
    ffm_ref.objective(t, cols, fields, torch.from_numpy(vals), y, xp=torch, **kw).backward()
    gam = t.grad.numpy()
    feat = np.zeros(NF + 1, dtype=bool)
    feat[cols] = True
    # every element of the touched feature rows: gam is 0 where the example does not reach (those stay put)
    want = -lr * gam[feat] / np.sqrt(1.0 + H[feat] + gam[feat] ** 2)
    np.testing.assert_allclose((r.table - W)[feat], want, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose((r.acc - H)[feat], gam[feat] ** 2, rtol=1e-10, atol=1e-13)
    assert (r.table[~feat][:-1] == W[~feat][:-1]).all() and (r.acc[~feat] == H[~feat]).all()
    assert (r.acc[:, 1:4] == 0).all() and (r.table[:, 1:4] == 0).all()
    kp = ffm_ref.kpad(k)
    for fi in range(F):
        assert (r.acc[:, 4 + fi * kp + k: 4 + (fi + 1) * kp] == 0).all()
    assert r.table[NF, 0] == W[NF, 0] - lr * r.g[0]   # w0 keeps the SGD step


def test_without_acc_the_replay_is_unchanged():
    rng = np.random.default_rng(2)
    W, cols, fields, vals = _example(5, True, rng)
    F = (W.shape[1] - 4) // ffm_ref.kpad(5)
    kw = dict(num_features=NF, num_fields=F, k=5, loss="logistic", lr=0.3, reg_linear=0.05, reg_factors=0.05)
    for extra in (dict(), dict(repull=True), dict(stale=True)):
        b = ffm_ref.replay(W, [0, 3, len(cols)], cols, fields, vals, [1.0, 0.0], acc=None, **kw, **extra)
        assert b.acc is None and b.tol_acc is None


def test_adagrad_breaks_change_the_replay():
    rng = np.random.default_rng(9)
    W, cols, fields, vals = _example(5, False, rng)
    F = (W.shape[1] - 4) // ffm_ref.kpad(5)
    H = _acc_like(W, rng, F, 5)
    kw = dict(num_features=NF, num_fields=F, k=5, loss="logistic", lr=0.3, reg_linear=0.05, reg_factors=0.05, acc=H)
    base = ffm_ref.replay(W, [0, 2, len(cols)], cols, fields, vals, [1.0, 0.0], **kw)
    for b in fm_ref.ADAGRAD_BREAKS:
        other = ffm_ref.replay(W, [0, 2, len(cols)], cols, fields, vals, [1.0, 0.0], breaks=b, **kw)
        moved = (np.abs(other.table - base.table) > 10 * (base.tol + other.tol)).any()
        moved |= (np.abs(other.acc - base.acc) > 10 * (base.tol_acc + other.tol_acc)).any()
        assert moved, b


def test_repull_reads_h_as_the_earlier_pushes_left_it():
    """One example that pushes the same slab twice: the repull end reads H with the first pair's gam^2."""
    k, F = 4, 2
    W = np.zeros((NF + 1, ffm_ref.stride(F, k)))
    rng = np.random.default_rng(4)
    W[:NF, 4:] = rng.normal(0, 0.5, (NF, F * k))
    cols, fields = np.array([1, 2, 3]), np.array([0, 1, 1])      # V[1, 1] pairs with both 2 and 3
    kw = dict(num_features=NF, num_fields=F, k=k, lr=0.5, acc=np.zeros_like(W))
    a = ffm_ref.replay(W, [0, 3], cols, fields, None, [1.0], **kw)
    b = ffm_ref.replay(W, [0, 3], cols, fields, None, [1.0], repull=True, **kw)
    assert not np.array_equal(a.table[1], b.table[1])


# ---- quality on the planted field-aware model --------------------------------------------------------------------

QUALITY_LRS = (0.02, 0.1, 0.5)
# held-out AUC of the fp64 replays from the devices' initial tables (FFM, k = 4, logistic, no L2), per learning
# rate; the AdaGrad ones gate tests/test_gpu_ffm_adagrad.py within 0.01, the SGD ones are DESIGN §2.17's comparison
AUC_ADAGRAD = {0.02: 0.6762, 0.1: 0.7047, 0.5: 0.7153}
AUC_SGD = {0.02: 0.6745, 0.1: 0.6929, 0.5: 0.5357}
# libffm's defaults under AdaGrad: eta 0.2, lambda 2e-5 (on the factors), k 4
LIBFFM = dict(lr=0.2, reg_factors=2e-5, k=4)
AUC_LIBFFM_FFM, AUC_LIBFFM_FM, AUC_LIBFFM_LINEAR = 0.7083, 0.6534, 0.6737


def fit_replay_ffm(lr, optimizer, reg_factors=0.0, k=4):
    q = QUALITY
    nf, F, n, B = q["num_features"], q["fields"], q["n_train"], q["batch"]
    rp, c, f, l = planted()
    W = initial_ffm_table(nf, F, k, QUALITY_SEED, -0.1, 0.1)
    H = np.zeros_like(W) if optimizer == "adagrad" else None
    kw = dict(num_features=nf, num_fields=F, k=k, loss="logistic", reg_factors=reg_factors)
    for _ in range(q["epochs"]):
        for b0 in range(0, n, B):
            b1 = min(b0 + B, n)
            s = slice(rp[b0], rp[b1])
            r = ffm_ref.replay(W, rp[b0:b1 + 1] - rp[b0], c[s], f[s], None, l[b0:b1], lr=lr, acc=H, **kw)
            W, H = r.table, r.acc
    pred = ffm_ref.replay(W, rp[n:] - rp[n], c[rp[n]:], f[rp[n]:], None, None, predict_only=True, **kw).pred
    return roc_auc(pred, l[n:])


def fit_replay_fm_on_ffm_data(lr, optimizer, reg_factors=0.0, k=4):
    from tests.test_fm_adagrad_host import fit_replay

    rp, c, _, l = planted()
    return fit_replay(k, lr, optimizer, reg=(0.0, reg_factors), planted_data=(rp, c, l))


@pytest.mark.parametrize("lr", QUALITY_LRS)
def test_quality_replay_sweep(lr):
    ada, sgd = fit_replay_ffm(lr, "adagrad"), fit_replay_ffm(lr, "sgd")
    print(f"\nFFM_ADAGRAD_QUALITY replay lr={lr}: AdaGrad AUC {ada:.4f}  SGD AUC {sgd:.4f}")
    assert abs(ada - AUC_ADAGRAD[lr]) < 5e-4 and abs(sgd - AUC_SGD[lr]) < 5e-4


def test_quality_at_libffm_defaults_ffm_beats_fm_and_linear():
    p = LIBFFM
    ffm = fit_replay_ffm(p["lr"], "adagrad", p["reg_factors"], p["k"])
    fm = fit_replay_fm_on_ffm_data(p["lr"], "adagrad", p["reg_factors"], p["k"])
    lin = fit_replay_fm_on_ffm_data(p["lr"], "adagrad", p["reg_factors"], 0)
    print(f"\nFFM_ADAGRAD_QUALITY replay at libffm's defaults: FFM {ffm:.4f}  FM {fm:.4f}  linear {lin:.4f}")
    assert abs(ffm - AUC_LIBFFM_FFM) < 5e-4 and abs(fm - AUC_LIBFFM_FM) < 5e-4 and abs(lin - AUC_LIBFFM_LINEAR) < 5e-4
    assert ffm > fm + 0.02 and ffm > lin + 0.02


# ---- refusals, before the library loads ---------------------------------------------------------------------------

def _tab(F=3, k=4, rows=100, base=0x1000):
    t = native.ShardTableC()
    s = native.ffm_stride(F, k)
    t.base[0], t.stride, t.dim, t.rows_per_shard, t.div, t.num_shards = base, s, s, rows, rows, 1
    return t


def _ffm(acc):
    a = _args()
    native.ffm_step(_tab(), a["row_ptr"], a["cols"], a["fields"], a["vals"], a["labels"], a["pred"],
                    num_features=10, num_fields=3, num_factors=4, bias=False, acc=acc)


@pytest.mark.parametrize("field, value", [("stride", 24), ("dim", 12), ("rows_per_shard", 99), ("div", 7),
                                          ("num_shards", 2), ("mode", 1)])
def test_ffm_step_refuses_an_accumulator_of_another_geometry(no_library, field, value):
    acc = _tab(base=0x2000)
    setattr(acc, field, value)
    with pytest.raises(ValueError, match="accumulator table's geometry"):
        _ffm(acc)


def test_ffm_step_refuses_an_accumulator_that_is_not_a_table(no_library):
    with pytest.raises(TypeError, match="acc must be a ShardTableC"):
        _ffm(torch.zeros(8))


def test_model_refuses_an_unknown_optimizer(no_library):
    with pytest.raises(ValueError, match=r"optimizer must be one of \['sgd', 'adagrad'\]"):
        DeviceFieldAwareFM(100, 3, 4, optimizer="ftrl")
    with pytest.raises(ValueError, match="optimizer must be one of"):
        check_ffm_config(100, 3, 4, "logistic", 0.0, 0.0, "hash", False, optimizer="")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_ffm_args_acc_is_appended_to_the_c_layout(tmp_path):
    mirror = native.FfmArgsC
    assert mirror._fields_[-1] == ("acc", native.ShardTableC)
    lines = ['  printf("sizeof %zu\\n", sizeof(FfmArgs));', '  printf("acc %zu\\n", offsetof(FfmArgs, acc));']
    assert _layout(tmp_path, "fps_ffm.cu", lines) == {"sizeof": str(C.sizeof(mirror)),
                                                      "acc": str(mirror.acc.offset)}
