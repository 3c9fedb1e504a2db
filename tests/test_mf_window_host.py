"""Eligibility rules of the MF step window (pure functions, no GPU)."""
import torch

from fps_b200.models.mf.device import WINDOW_BUDGET, step_window_size, step_windowable
from fps_b200.ops import native


def _size(step_window=None, **kw):
    args = dict(world=1, item_cache=False, loss="pointwise", table_rows=1_000_000, stride=64, env=None)
    args.update(kw)
    return step_window_size(step_window, **args)


def test_auto_is_on_for_one_worker_with_a_table_above_l2():
    assert _size() == native.WINDOW_MAX == 8
    assert _size(table_rows=100_000) == 0                  # 25.6 MB table: L2 absorbs the re-reads
    assert _size(env="0") == 0
    assert _size(env="1") == 8
    assert _size(world=2) == 0
    assert _size(item_cache=True) == 0
    assert _size(loss="bpr") == 0
    assert _size(stride=256) == 0                           # k > 128: no window kernel


def test_explicit_sizes():
    assert _size(0) == 0 and _size(1) == 0
    assert _size(2) == 2 and _size(5) == 5
    assert _size(64) == 8                                   # at most WINDOW_MAX
    assert _size(4, table_rows=100) == 4                    # forced on for a small table
    assert _size(4, world=2) == 0


def test_memory_budget_lowers_the_window():
    # 20 B per row and slot: 8 x 1M rows = 160 MB fits the 256 MB budget
    assert _size(table_rows=1_000_000) == 8
    assert _size(table_rows=3_000_000) == WINDOW_BUDGET // (3_000_000 * 20) == 4
    assert _size(table_rows=7_000_000) == 0                 # only one slot would fit


def _ok(**kw):
    args = dict(neg=0, output_ring=None, pull_limit=0, credits=None, kernel=None, kernel_env="reg",
                reg_variant_env=None, l2_hints=False, packed=True, dtypes=(torch.int64,), n_records=1000,
                table_rows=1000, on_gpu=True, capturing=False)
    args.update(kw)
    return step_windowable(**args)


def test_step_eligibility():
    assert _ok()
    assert _ok(kernel="reg") and _ok(reg_variant_env="0")
    assert _ok(packed=False, dtypes=(torch.int32, torch.int32, torch.float32))
    assert not _ok(packed=False, dtypes=(torch.int64, torch.int64, torch.float32))
    assert not _ok(n_records=1001)
    assert not _ok(neg=1)
    assert not _ok(output_ring=object())
    assert not _ok(pull_limit=64)
    assert not _ok(kernel="tma")
    assert not _ok(kernel_env="tma")
    assert not _ok(reg_variant_env="3")
    assert not _ok(l2_hints=True)
    assert not _ok(capturing=True)
    assert not _ok(on_gpu=False)
