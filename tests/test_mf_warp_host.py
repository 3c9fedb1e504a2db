"""Host-side checks of the WARP loss: the numpy reference step, the quality a sequential run reaches on the
BPR quality set, and every refusal that is checked before the device is touched."""
import math

import numpy as np
import pytest

import fps_b200  # noqa: F401
from fps_b200.models.mf.common import Rating, warp_delta
from tests import bpr_quality as Q
from tests import warp_quality as W


def test_first_violator_is_taken_in_draw_order():
    u, vi = np.array([1.0, 0.0]), np.array([2.0, 0.0])
    rows = [np.array([0.0, 5.0]), np.array([1.5, 0.0]), np.array([3.0, 0.0])]   # x = 2.0, 0.5, -1.0
    du, dvi, t, dvj, n, L, loss = warp_delta(u, vi, rows, 1.0, 0.1, 0.0, 101)
    assert t == 1 and n == 2
    assert L == pytest.approx(math.log(50))
    assert loss == pytest.approx(math.log(50) * 0.5)
    np.testing.assert_allclose(dvj, -0.1 * math.log(50) * u)
    np.testing.assert_allclose(du, 0.1 * math.log(50) * (vi - rows[1]))


def test_void_candidates_are_not_counted():
    u, vi = np.array([1.0]), np.array([2.0])
    rows = [None, np.array([0.0]), None, None, np.array([1.5])]          # x = 2.0 (no), 0.5 (violates)
    _, _, t, _, n, L, _ = warp_delta(u, vi, rows, 1.0, 0.1, 0.0, 11)
    assert t == 4 and n == 2 and L == pytest.approx(math.log(5))


def test_no_violator_means_no_update_and_counts_every_live_candidate():
    u, vi = np.array([1.0]), np.array([2.0])
    du, dvi, t, dvj, n, L, loss = warp_delta(u, vi, [np.array([0.0]), None, np.array([-1.0])], 1.0, 0.1, 0.0, 11)
    assert du is None and dvi is None and t is None and dvj is None
    assert n == 2 and L == 0.0 and loss == 0.0


@pytest.mark.parametrize("N, n, want", [(11, 5, math.log(2)), (11, 6, 0.0), (11, 10, 0.0), (2, 1, 0.0),
                                        (1000, 1, math.log(999))])
def test_rank_weight_edges(N, n, want):
    """``L = ln(max(1, (N - 1) // n))``: 0 once ``n > (N - 1) / 2``, and 0 for two items."""
    u, vi = np.array([1.0]), np.array([0.0])
    rows = [np.array([-5.0])] * (n - 1) + [np.array([0.0])]             # x = 5 for the first n - 1, then 0
    _, _, t, _, got_n, L, _ = warp_delta(u, vi, rows, 1.0, 0.1, 0.0, N)
    assert t == n - 1 and got_n == n
    assert L == pytest.approx(want, abs=1e-15)


def _objective(u, vi, vj, L, margin, reg):
    return L * (margin - float(u @ (vi - vj))) + reg / 2 * (u @ u + vi @ vi + vj @ vj)


@pytest.mark.parametrize("reg", [0.0, 0.03])
@pytest.mark.parametrize("scale", [0.3, 3.0])
def test_warp_delta_is_minus_lr_times_the_gradient(reg, scale):
    """At fixed ``L`` the deltas are ``-lr`` times the gradient of the weighted hinge plus the L2 term."""
    rng = np.random.default_rng(11)
    u, vi, vj = (rng.normal(0, scale, 7) for _ in range(3))
    margin = float(u @ (vi - vj)) + 1.0                                    # the candidate violates
    lr, h = 0.05, 1e-6
    du, dvi, t, dvj, n, L, loss = warp_delta(u, vi, [vj], margin, lr, reg, 50)
    assert t == 0 and n == 1 and L == pytest.approx(math.log(49))
    assert loss == pytest.approx(L * 1.0)
    for which, got in ((0, du), (1, dvi), (2, dvj)):
        grad = np.zeros(7)
        for c in range(7):
            args = [u.copy(), vi.copy(), vj.copy()]
            args[which][c] += h
            up = _objective(*args, L, margin, reg)
            args[which][c] -= 2 * h
            grad[c] = (up - _objective(*args, L, margin, reg)) / (2 * h)
        np.testing.assert_allclose(got, -lr * grad, rtol=1e-5, atol=1e-8)


def test_sequential_numpy_warp_beats_random_on_heldout():
    tu, ti, eu, ei = Q.data()
    U, V = W.train_numpy(tu, ti)
    auc, recall = Q.metrics(U, V, (tu, ti), (eu, ei))
    assert auc >= W.AUC_GATE and recall >= W.RECALL_GATE, (auc, recall)


# ---- refusals: each names the fix and is raised before any device work --------------------------------------
@pytest.mark.parametrize("kw, match", [
    (dict(loss="warp", optimizer="adagrad"), "optimizer='sgd'"),
    (dict(loss="warp", negative_sampling="seen", negative_sample_rate=2), "negative_sampling='uniform'"),
    (dict(loss="warp", output_ring=object()), "output ring"),
    (dict(loss="warp", kernel="tma"), "tma"),
    (dict(loss="warp", item_blocking=True), "item_blocking"),
    (dict(loss="bpr", margin=0.5), "loss='warp'"),
    (dict(margin=0.5), "loss='warp'"),
    (dict(loss="warp", margin=float("nan")), "finite"),
    (dict(loss="warp", margin=float("inf")), "finite"),
])
def test_device_model_refuses_unsupported_warp_settings(kw, match):
    from fps_b200.models.mf.device import DeviceOnlineMF

    with pytest.raises(ValueError, match=match):
        DeviceOnlineMF(16, 16, 8, **kw)


def test_check_warp_default_margin():
    from fps_b200.models.mf.device import check_warp

    assert check_warp("warp", None, optimizer="sgd", negative_sampling="uniform") == 1.0
    assert check_warp("warp", 0.25, optimizer="sgd", negative_sampling="uniform") == 0.25
    assert check_warp("bpr", None, optimizer="adagrad", negative_sampling="seen") is None


_RATINGS = [Rating(u, i, 1.0) for u in range(4) for i in range(3)]


@pytest.mark.parametrize("backend", ["local", "native"])
@pytest.mark.parametrize("kw", [dict(loss="warp"), dict(margin=0.5), dict(loss="warp", margin=0.5)])
def test_host_backends_refuse_warp(backend, kw):
    from fps_b200.models.mf.offline import psOfflineMF
    from fps_b200.models.mf.online import psOnlineMF
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator

    with pytest.raises(ValueError, match="backend='device'"):
        psOnlineMF(_RATINGS, backend=backend, negativeSampleRate=1, **kw)
    with pytest.raises(ValueError, match="backend='device'"):
        psOfflineMF(_RATINGS, backend=backend, negativeSampleRate=1, iterations=1, **kw)
    with pytest.raises(ValueError, match="backend='device'"):
        psOnlineLearnerAndGenerator(_RATINGS, backend=backend, negativeSampleRate=1, **kw)


def test_device_mf_refuses_update_output_with_warp():
    from fps_b200.models.mf.online import psOnlineMF

    with pytest.raises(ValueError, match="updateOutput"):
        psOnlineMF(_RATINGS, backend="device", negativeSampleRate=1, loss="warp", updateOutput=1)


@pytest.mark.parametrize("kw, match", [
    (dict(loss="warp", negativeSampleRate=0), "negativeSampleRate >= 1"),
    (dict(loss="warp", negativeSampleRate=2, margin=float("nan")), "finite"),
    (dict(loss="bpr", negativeSampleRate=2, margin=0.5), "loss='warp'"),
    (dict(loss="hinge", negativeSampleRate=2), "loss must be"),
])
def test_learner_refuses_unsupported_warp_settings(kw, match):
    """Checked before the learner builds its tables."""
    from fps_b200.models.mf.device_api import ps_online_learner_and_generator_device

    with pytest.raises(ValueError, match=match):
        ps_online_learner_and_generator_device(_RATINGS, **kw)


def test_binding_refuses_bad_margin_and_trial_block():
    """Checked before any tensor is looked at."""
    from fps_b200.ops import native

    with pytest.raises(ValueError, match="margin"):
        native.mf_warp_fused(None, None, None, None, None, 0.1, margin=float("nan"))
    with pytest.raises(ValueError, match="trial_block"):
        native.mf_warp_fused(None, None, None, None, None, 0.1, trial_block=3)
