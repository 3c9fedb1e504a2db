"""Host-side checks of the pairwise (BPR) loss: the numpy reference step, the synthetic implicit-feedback
set, the quality a sequential run reaches on it, and the host tiers refusing the loss."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models.mf.common import Rating, bpr_delta
from fps_b200.utils.synthetic import lowrank_implicit
from tests import bpr_quality as Q


def _objective(u, vi, vj, reg):
    x = float(np.dot(u, vi - vj))
    return np.logaddexp(0.0, -x) + reg / 2 * (u @ u + vi @ vi + vj @ vj)


@pytest.mark.parametrize("reg", [0.0, 0.03])
@pytest.mark.parametrize("scale", [0.3, 3.0])
def test_bpr_delta_is_minus_lr_times_the_gradient(reg, scale):
    rng = np.random.default_rng(11)
    u, vi, vj = (rng.normal(0, scale, 7) for _ in range(3))
    lr, h = 0.05, 1e-6
    du, dvi, dvj, loss = bpr_delta(u, vi, vj, lr, reg)
    assert loss == pytest.approx(np.logaddexp(0.0, -float(u @ (vi - vj))), rel=1e-12)
    for which, got in ((0, du), (1, dvi), (2, dvj)):
        grad = np.zeros(7)
        for c in range(7):
            args = [u.copy(), vi.copy(), vj.copy()]
            args[which][c] += h
            up = _objective(*args, reg)
            args[which][c] -= 2 * h
            grad[c] = (up - _objective(*args, reg)) / (2 * h)
        np.testing.assert_allclose(got, -lr * grad, rtol=1e-5, atol=1e-9)


def test_bpr_delta_loss_is_stable_for_large_margins():
    u = np.array([100.0]); vi = np.array([10.0]); vj = np.array([0.0])
    assert bpr_delta(u, vi, vj, 0.1, 0.0)[3] == pytest.approx(np.exp(-1000.0), abs=1e-300)
    assert bpr_delta(-u, vi, vj, 0.1, 0.0)[3] == pytest.approx(1000.0)


def test_lowrank_implicit_deterministic_and_disjoint():
    a = lowrank_implicit(300, 500, 12, 3, seed=5)
    b = lowrank_implicit(300, 500, 12, 3, seed=5)
    c = lowrank_implicit(300, 500, 12, 3, seed=6)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert not torch.equal(a[1], c[1])
    tu, ti, eu, ei = a
    assert tu.numel() == 300 * 9 and eu.numel() == 300 * 3
    train = set(zip(tu.tolist(), ti.tolist()))
    test = set(zip(eu.tolist(), ei.tolist()))
    assert len(train) == tu.numel() and len(test) == eu.numel()     # distinct items per user
    assert not train & test
    assert int(ti.max()) < 500 and int(tu.max()) < 300


def test_lowrank_implicit_follows_the_lowrank_scores():
    """Consumed items score higher under the ground-truth model than random ones."""
    from fps_b200.utils.synthetic import lowrank_ratings

    tu, ti, _, _ = lowrank_implicit(200, 400, 10, 2, seed=1)
    chosen = lowrank_ratings(tu, ti, seed=1).mean()
    rand = lowrank_ratings(tu, torch.randint(0, 400, ti.shape, generator=torch.Generator().manual_seed(0)),
                           seed=1).mean()
    assert chosen > rand + 0.3


def test_sequential_numpy_bpr_beats_random_on_heldout():
    tu, ti, eu, ei = Q.data()
    U, V = Q.train_numpy(tu, ti)
    auc, recall = Q.metrics(U, V, (tu, ti), (eu, ei))
    assert auc >= Q.AUC_GATE and recall >= Q.RECALL_GATE, (auc, recall)
    # an untrained model sits at chance
    rng = np.random.default_rng(0)
    auc0, recall0 = Q.metrics(torch.from_numpy(rng.uniform(-0.1, 0.1, U.shape)),
                              torch.from_numpy(rng.uniform(-0.1, 0.1, V.shape)), (tu, ti), (eu, ei))
    assert auc0 < 0.56 and recall0 < 0.04, (auc0, recall0)


_RATINGS = [Rating(u, i, 1.0) for u in range(4) for i in range(3)]


@pytest.mark.parametrize("backend", ["local", "native"])
@pytest.mark.parametrize("kw", [dict(loss="bpr"), dict(regularization=0.1)])
def test_host_backends_refuse_bpr_mf(backend, kw):
    from fps_b200.models.mf.offline import psOfflineMF
    from fps_b200.models.mf.online import psOnlineMF

    with pytest.raises(ValueError, match="backend='device'"):
        psOnlineMF(_RATINGS, backend=backend, negativeSampleRate=1, **kw)
    with pytest.raises(ValueError, match="backend='device'"):
        psOfflineMF(_RATINGS, backend=backend, negativeSampleRate=1, iterations=1, **kw)


@pytest.mark.parametrize("backend", ["local", "native"])
def test_host_backends_refuse_bpr_learner(backend):
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator

    with pytest.raises(ValueError, match="backend='device'"):
        psOnlineLearnerAndGenerator(_RATINGS, backend=backend, negativeSampleRate=1, loss="bpr")


def test_experiment_main_passes_loss_through(tmp_path):
    from fps_b200.models.mf.experiments import OnlineMFImplicit

    src = tmp_path / "in.txt"
    src.write_text("0 1 2\n1 2 3\n")
    with pytest.raises(ValueError, match="backend='device'"):
        OnlineMFImplicit([str(src), str(tmp_path / "u"), str(tmp_path / "i")], loss="bpr")


@pytest.mark.parametrize("kw, match", [
    (dict(regularization=0.1), "regularization"),
    (dict(loss="bpr", output_ring=object()), "output ring"),
    (dict(loss="bpr", kernel="tma"), "tma"),
    (dict(loss="bpr", item_blocking=True), "item_blocking"),
    (dict(loss="hinge"), "loss"),
])
def test_device_model_refuses_unsupported_bpr_settings(kw, match):
    """Checked before the model touches a device."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    with pytest.raises(ValueError, match=match):
        DeviceOnlineMF(16, 16, 8, **kw)


def test_device_mf_refuses_update_output_with_bpr():
    """The per-update output ring is pointwise only; the check runs before any device work."""
    from fps_b200.models.mf.online import psOnlineMF

    with pytest.raises(ValueError, match="updateOutput"):
        psOnlineMF(_RATINGS, backend="device", negativeSampleRate=1, loss="bpr", updateOutput=1)
