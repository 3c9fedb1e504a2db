"""CPU checks of the replay helpers the pointwise MF GPU suite relies on (tests/philox_ref.py), of the K5 rejection
rule, and of the argument refusals of the pointwise step that need no device."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests.philox_ref import init_rows_f64_ref, k5_negative, k5_shift, philox4x32


# Known-answer vectors of Philox4x32-10 published with the Random123 library (kat_vectors).
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(x) for x in philox4x32(*ctr, *key)) == want


def test_k5_negative_key_and_draw():
    """Negative j of record pos: counter (pos_lo, pos_hi, j, step_lo), key (seed_lo, seed_hi); the draw is
    ((x << 32) | y) % num_items."""
    pos, j, step, seed, n = (3 << 32) + 11, 2, (1 << 32) + 9, (5 << 32) + 77, 1_000_003
    x, y, z, _ = philox4x32(11, 3, 2, 9, 77, 5)
    raw = ((int(x) << 32) | int(y)) % n
    neg, r = k5_negative([pos], j, [-1], n, step, seed)
    assert r[0] == raw and neg[0] == raw
    neg, _ = k5_negative([pos], j, [raw], n, step, seed)           # the positive: moved by the shift
    assert neg[0] == (raw + 1 + (int(z) % 7) % (n - 1)) % n != raw
    # another j, step or seed word changes the draw
    others = {int(k5_negative([pos], jj, [-1], n, st, sd)[1][0])
              for jj, st, sd in ((1, step, seed), (j, 9 + 1, seed), (j, step, seed ^ (1 << 40)))}
    assert raw not in others


@pytest.mark.parametrize("num_items", range(2, 10))
def test_shift_never_lands_on_the_positive(num_items):
    items = np.repeat(np.arange(num_items), 7)
    z = np.tile(np.arange(7), num_items)
    moved = k5_shift(items, z, num_items)
    assert np.all(moved != items) and np.all((moved >= 0) & (moved < num_items))
    old = (items + 1 + z) % num_items                              # the rule before the modulo
    if num_items >= 8:
        assert np.array_equal(moved, old)                          # unchanged from 8 items up
    else:
        assert np.any(old == items)                                # the old rule could return the positive


def test_init_rows_f64_ref_by_hand():
    dim, seed, lo, hi = 5, (9 << 32) + 4, -0.25, 0.5
    ids = np.array([0, 7, (1 << 33) + 5])
    got = init_rows_f64_ref(ids, dim, seed, lo, hi)
    assert got.shape == (3, 6) and not got[:, 5].any()
    assert np.all((got[:, :dim] >= lo) & (got[:, :dim] < hi))
    for row, i in enumerate(ids.tolist()):
        for col in range(dim):
            w = philox4x32(i & 0xFFFFFFFF, i >> 32, col // 2, 1, seed & 0xFFFFFFFF, seed >> 32)
            m = ((int(w[2 * (col % 2)]) << 32) | int(w[2 * (col % 2) + 1])) >> 11
            assert got[row, col] == float(Fraction(lo) + Fraction(hi - lo) * Fraction(m, 1 << 53))


# ---- refusals of the pointwise step before any device tensor is touched -----------------------------------------

def _args(n=4, dtype=torch.int32, n_items=None, n_ratings=None, item_dtype=None):
    return (torch.zeros(n, dtype=dtype), torch.zeros(n if n_items is None else n_items, dtype=item_dtype or dtype),
            torch.ones(n if n_ratings is None else n_ratings))


FUSED = [lambda u, i, r, **kw: native.mf_sgd_fused(u, i, r, None, 1, None, 0.1, **kw),
         lambda u, i, r, **kw: native.mf_sgd_fused_f64(u, i, r, None, 1, None, 0.1, **kw)]


@pytest.mark.parametrize("call", FUSED, ids=["fp32", "fp64"])
@pytest.mark.parametrize("err_mode", [-1, 3, 7])
def test_unknown_err_mode_is_refused(call, err_mode):
    with pytest.raises(ValueError, match="err_mode"):
        call(*_args(), err_mode=err_mode)


@pytest.mark.parametrize("call", FUSED, ids=["fp32", "fp64"])
@pytest.mark.parametrize("lengths", [dict(n_items=3), dict(n_ratings=5)])
def test_record_lengths_must_agree(call, lengths):
    with pytest.raises(ValueError, match="same length"):
        call(*_args(**lengths))


@pytest.mark.parametrize("call", FUSED, ids=["fp32", "fp64"])
def test_id_dtypes_must_agree(call):
    with pytest.raises(TypeError, match="share an integer dtype"):
        call(*_args(item_dtype=torch.int64))


@pytest.mark.parametrize("call", FUSED, ids=["fp32", "fp64"])
def test_packed_records_must_be_int64(call):
    with pytest.raises(TypeError, match="packed"):
        call(torch.zeros(4, dtype=torch.int32), None, None)


@pytest.mark.parametrize("num_items", [0, 1])
def test_sampled_negatives_need_two_items(num_items):
    with pytest.raises(ValueError, match="num_items >= 2"):
        native.mf_sgd_fused(*_args(), None, 1, None, 0.1, neg_rate=1, num_items=num_items)
