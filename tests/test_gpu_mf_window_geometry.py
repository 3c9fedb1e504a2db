"""Lane geometries of the step-window drain (fps_mf_window.cu): rows held as several float4 per lane give the
per-launch tables bitwise for every width of a bucket and every kernel variant, and the drain's phase timer
reports its build and apply time without changing what it computes."""
import pytest
import torch

from tests.test_gpu_mf_window import _conflict_free_steps, _pair, _same_stats, _same_tables

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture
def variant(monkeypatch):
    from fps_b200.ops import native

    def use(v):
        monkeypatch.setenv("FPS_MF_WINDOW_VARIANT", str(v))
    yield use
    native.lib().fps_set_mf_window_variant(0)


# k = 36, 40, 52: rows of 9, 10 and 13 float4 in the 16-lane bucket, so some lanes hold fewer float4 than others
@pytest.mark.parametrize("k", [16, 36, 40, 52, 64, 128])
@pytest.mark.parametrize("knob", [0, 1, 2])
def test_every_width_and_variant_is_bitwise(dev, variant, k, knob):
    variant(knob)
    win, ref = _pair(k=k, err_mode=0)
    g = torch.Generator().manual_seed(k + 100 * knob)
    for step in _conflict_free_steps(g, dev, 4, 5, 1_000, True):
        for b in step:
            win.step(*b)
            ref.step(*b)
    _same_tables(win, ref)
    _same_stats(win, ref)
    win.close(); ref.close()


def test_phase_timer_reports_build_and_apply(dev):
    win, ref = _pair(k=64)
    win._win_phase_ns = torch.zeros(4, dtype=torch.int64, device=dev)
    g = torch.Generator().manual_seed(3)
    for step in _conflict_free_steps(g, dev, 3, 5, 1_000, True):
        for b in step:
            win.step(*b)
            ref.step(*b)
        win.flush()
    build, apply, windows, _ = win._win_phase_ns.tolist()
    assert windows == 3           # one conflict-free window per drained step
    assert build > 0 and apply > 0
    _same_tables(win, ref)
    win.close(); ref.close()

