"""Row-wise AdaGrad without a GPU: the numpy reference rule, the step-window and refusal rules of
``DeviceOnlineMF(optimizer=...)`` and the host tiers' refusal."""
import math

import numpy as np
import pytest

import fps_b200  # noqa: F401
from fps_b200.models.mf.common import Rating, require_pointwise, rowwise_adagrad
from fps_b200.models.mf.device import check_optimizer, step_window_size


def test_rowwise_adagrad_two_steps_by_hand():
    """k = 2, lr = 0.5, row (1, 0), deltas (3, 4) then (0, 2):
    step 1: s = 25 / 2 = 12.5, G' = 12.5, row += 0.5 * (3, 4) / sqrt(12.5);
    step 2: s = 4 / 2 = 2, G' = 14.5, row += 0.5 * (0, 2) / sqrt(14.5)."""
    row, G = np.array([1.0, 0.0]), 0.0
    row, s = rowwise_adagrad(row, G, [3.0, 4.0], 0.5, 2)
    assert s == 12.5
    G += s
    r1 = 1.0 / math.sqrt(12.5)
    np.testing.assert_allclose(row, [1.0 + 1.5 * r1, 2.0 * r1], rtol=1e-7)   # eps = 1e-8 moves the result by ~3e-9
    row, s = rowwise_adagrad(row, G, [0.0, 2.0], 0.5, 2)
    assert s == 2.0
    G += s
    assert G == 14.5
    np.testing.assert_allclose(row, [1.0 + 1.5 * r1, 2.0 * r1 + 1.0 / math.sqrt(14.5)], rtol=1e-7)   # eps = 1e-8 moves the result by ~3e-9


def test_rowwise_adagrad_zero_delta_leaves_row_and_accumulator():
    row, s = rowwise_adagrad(np.array([0.25, -1.0, 2.0]), 3.0, np.zeros(3), 0.1, 3)
    assert s == 0.0
    np.testing.assert_array_equal(row, [0.25, -1.0, 2.0])


def test_step_window_is_off_for_adagrad():
    kw = dict(world=1, item_cache=False, loss="pointwise", table_rows=1_000_000, stride=64)
    assert step_window_size(None, **kw) > 0
    assert step_window_size(None, optimizer="adagrad", **kw) == 0
    assert step_window_size(8, optimizer="adagrad", **kw) == 0


def test_check_optimizer_accepts_sgd_everywhere_and_adagrad_direct():
    check_optimizer("sgd", item_cache=True, output_ring=object(), kernel="tma")
    check_optimizer("adagrad", item_cache=False)
    check_optimizer("adagrad", item_cache=False, kernel="reg")


@pytest.mark.parametrize("kw, fix", [
    (dict(item_cache=True), "item_cache=False"),
    (dict(item_cache=False, output_ring=object()), "output_ring=None"),
    (dict(item_cache=False, kernel="tma"), "kernel=None"),
])
def test_check_optimizer_refusals_name_the_fix(kw, fix):
    with pytest.raises(ValueError, match=fix.replace("(", r"\(")):
        check_optimizer("adagrad", **kw)


def test_check_optimizer_unknown_name():
    with pytest.raises(ValueError, match="'sgd' or 'adagrad'"):
        check_optimizer("adam", item_cache=False)


@pytest.mark.parametrize("backend", ["local", "native"])
def test_host_tiers_refuse_adagrad(backend):
    with pytest.raises(ValueError, match="backend='device'"):
        require_pointwise(backend, {"optimizer": "adagrad"})
    require_pointwise(backend, {"optimizer": "sgd"})
    require_pointwise("device", {"optimizer": "adagrad"})


@pytest.mark.parametrize("entry", ["online", "offline"])
def test_host_entry_points_refuse_adagrad(entry):
    from fps_b200.models.mf.offline import psOfflineMF
    from fps_b200.models.mf.online import psOnlineMF

    recs = [Rating(0, 1, 1.0), Rating(1, 0, 0.5)]
    fn = psOnlineMF if entry == "online" else psOfflineMF
    with pytest.raises(ValueError, match="optimizer='adagrad' needs backend='device'"):
        fn(recs, numFactors=4, backend="local", optimizer="adagrad")
