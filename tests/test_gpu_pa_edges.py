"""Passive-aggressive kernels (ops/csrc/fps_pa.cu) against the fp64 replay of tests/pa_ref.py, launch by launch.

Every case reads the table, runs one ``native.pa_step`` launch, reads the table and outputs back, and compares
with the replay fed the pre-launch table: predictions, the ``loss`` output (prefilled with NaN, so an entry the
kernel must not write stays NaN), the non-finite flag, every table element within ``MARGIN`` times its bound, and
the padding columns.  Multi-launch runs start each launch from the kernel's own state, so no error accumulates.
Examples of one batch use disjoint features, so the batch has one correct result however the kernel races them."""
import numpy as np
import pytest
import torch

from tests import pa_ref

pytestmark = pytest.mark.gpu

UNL = pa_ref.UNLABELLED
MARGIN = pa_ref.MARGIN
C_OF = {"PA": 0.0, "PAI": 0.05, "PAII": 0.5, "PB": 0.0, "ML": 0.0}

WARP_L = [1, 3, 4, 7, 11, 16, 23, 37, 64, 100, 128]
BLOCK_L = [129, 515, 1024]
FORCED_L = [1, 7, 11, 23, 37, 100]
RUNGS = [(L, 0) for L in WARP_L + BLOCK_L] + [(L, 1) for L in FORCED_L]
GRID_CASES = [(1, 0, "PA", False), (7, 0, "PB", False), (11, 0, "ML", False), (23, 0, "PAI", False),
              (37, 0, "PAII", False), (100, 0, "ML", True), (1, 1, "PAI", False), (7, 1, "PA", False),
              (11, 1, "PB", True), (23, 1, "ML", False), (37, 1, "PAII", False), (1024, 0, "PB", False)]


def _algos(L):
    if L == 1:
        return [("PA", False), ("PAI", False), ("PAII", False)]
    return [("PA", False), ("PAI", False), ("PAII", False), ("PB", False), ("PB", True), ("ML", False),
            ("ML", True)]


def _cost(L):
    a = np.arange(L)
    return np.where(a[:, None] == a[None, :], 0.0, 1.0 + 0.25 * np.abs(a[:, None] - a[None, :])).astype(np.float32)


class _Variant:
    """``fps_set_pa_variant`` for the duration of a case, reset to automatic dispatch in any event."""

    def __init__(self, v):
        self.v = v

    def __enter__(self):
        from fps_b200.ops import native
        native.lib().fps_set_pa_variant(self.v)

    def __exit__(self, *exc):
        from fps_b200.ops import native
        native.lib().fps_set_pa_variant(0)


def _model(feats, L, algo, cost=False, range_part=False):
    from fps_b200.models.pa.device import DevicePassiveAggressive

    torch.cuda.set_device(0)
    return DevicePassiveAggressive(feats, L, L == 1, algo, C_OF[algo], _cost(L) if cost else None, range_part)


def _table(pa):
    torch.cuda.synchronize()
    return pa.table.local.cpu().numpy()


def _set_table(pa, W):
    pa.table.local[: W.shape[0], : W.shape[1]] = torch.from_numpy(np.asarray(W, dtype=np.float32)).cuda()


def _batch(rng, n, feats, L, nnz=(1, 6), mix=False, x_scale=1.0):
    """CSR batch over disjoint features.  ``mix``: every 11th example empty, zero-valued, with a repeated
    feature, or unlabelled."""
    perm = rng.permutation(feats)
    pos = 0
    rp, cols, vals, labels = [0], [], [], []
    for ex in range(n):
        kind = ex % 11 if mix else -1
        k = 0 if kind == 0 else int(rng.integers(nnz[0], nnz[1] + 1))
        idx = list(perm[pos:pos + k])
        pos += k
        x = list(rng.normal(0, x_scale, k))
        if kind == 1:
            x = [0.0] * k
        if kind == 2:
            idx.append(idx[0])
            x.append(float(rng.normal(0, x_scale)))
        cols += idx
        vals += x
        rp.append(len(cols))
        if kind == 3:
            labels.append(UNL)
        else:
            labels.append(int(rng.choice([-1, 1])) if L == 1 else int(rng.integers(L)))
    assert pos <= feats
    return (np.array(rp, np.int64), np.array(cols, np.int64), np.array(vals, np.float32), np.array(labels, np.int32))


def _launch(pa, batch, id64=False):
    from fps_b200.ops import native

    rp, cols, vals, labels = batch
    dev = pa.dev
    n = len(labels)
    pred = torch.full((n,), -7, dtype=torch.int32, device=dev)
    loss = torch.full((n,), float("nan"), dtype=torch.float32, device=dev)
    pa.nan_flag.zero_()
    native.pa_step(pa.table.table_c, torch.from_numpy(rp).to(dev),
                   torch.from_numpy(cols.astype(np.int64 if id64 else np.int32)).to(dev),
                   torch.from_numpy(vals).to(dev), torch.from_numpy(labels).to(dev), pred, binary=pa.binary,
                   num_labels=pa.L, algo=pa.algo, aggressiveness=pa.C, cost=pa.cost, loss=loss,
                   nan_flag=pa.nan_flag)
    torch.cuda.synchronize()
    return pred.cpu().numpy(), loss.cpu().numpy().astype(np.float64), int(pa.nan_flag.item())


def _step(pa, batch, id64=False, exact_nonfinite=True):
    """One launch against the replay; returns (replay, kernel pred, worst |error| / bound)."""
    L = pa.L
    before = _table(pa)
    rp, cols, vals, labels = batch
    cost = None if pa.cost is None else pa.cost.cpu().numpy()
    rep = pa_ref.replay(before[:, :L].astype(np.float64), rp, cols, vals.astype(np.float64), labels,
                        algo=pa.algo, binary=pa.binary, C=pa.C, cost=cost)
    pred, loss, flag = _launch(pa, batch, id64)
    after = _table(pa)
    assert (after[:, L:] == 0).all(), "padding columns written"
    assert flag == int(rep.bad.any())
    dec = rep.decided
    if pa.algo in ("PB", "ML"):
        assert dec.all(), "a PB / ML choice is within the bounds"
    # one OVA-PA launch on a fresh model leaves equal weights in every violated column, so the next launch
    # meets genuine near-ties of the prediction; it feeds no update, and only decided ones are compared
    assert dec.mean() > 0.5
    np.testing.assert_array_equal(pred[dec], rep.pred[dec])
    assert set(np.unique(pred)) <= set(range(max(L, 2)))
    np.testing.assert_array_equal(np.isnan(loss), np.isnan(rep.loss))
    m = ~np.isnan(rep.loss)
    assert (np.abs(loss[m] - rep.loss[m]) <= MARGIN * rep.tol_loss[m]).all()
    got = after[:, :L].astype(np.float64)
    fin = np.isfinite(rep.table)
    if exact_nonfinite:
        np.testing.assert_array_equal(got[~fin], rep.table[~fin])
    err = np.abs(got[fin] - rep.table[fin])
    tol = rep.tol[fin]
    assert (err <= MARGIN * tol).all(), float((err - MARGIN * tol).max())
    worst = float((err / np.where(tol > 0, tol, np.inf)).max()) if err.size else 0.0
    return rep, pred, worst


def _run(L, variant, algo, cost, *, n=64, launches=2, nnz=(1, 6), mix=True, id64=False, range_part=False,
         fresh=False, seed=0):
    rng = np.random.default_rng([L, variant, seed, len(algo), int(cost)])
    feats = n * (nnz[1] + 1) + 8
    pa = _model(feats, L, algo, cost, range_part)
    try:
        if not fresh:
            _set_table(pa, rng.normal(0, 0.3, (feats, L)))
        worst = 0.0
        with _Variant(variant):
            for _ in range(launches):
                batch = _batch(rng, n, feats, L, nnz, mix)
                rep, pred, w = _step(pa, batch, id64)
                worst = max(worst, w)
                assert rep.updated.sum() > n // 4
                if fresh:
                    assert (pred == 0).all()
                    fresh = False
        return worst
    finally:
        pa.close()


# ---- every rung of both kernels -------------------------------------------------------------------------------

def test_rung_cases_cover_the_dispatch_table():
    covered = {pa_ref.geometry(L, v) for L, v in RUNGS}
    assert covered == set(pa_ref.dispatch_table())
    assert {pa_ref.geometry(L, v) for L, v, _, _ in GRID_CASES} == set(pa_ref.dispatch_table())


@pytest.mark.parametrize("L,variant,algo,cost",
                         [(L, v, a, c) for L, v in RUNGS for a, c in _algos(L)])
def test_rung_matches_replay(L, variant, algo, cost):
    _run(L, variant, algo, cost)


# ---- grid-stride rounds, with empty, zero-valued, repeated-feature and unlabelled examples --------------------

@pytest.mark.parametrize("L,variant,algo,cost", GRID_CASES)
def test_grid_stride_batch_matches_replay(L, variant, algo, cost):
    from fps_b200.ops import native

    kernel = pa_ref.geometry(L, variant)[0]
    n = 2 * pa_ref.cap(kernel, native.sm_count(0)) + 3
    _run(L, variant, algo, cost, n=n, launches=1, nnz=(1, 2) if L > 128 else (1, 3))


@pytest.mark.parametrize("L,variant,algo", [(37, 0, "ML"), (7, 1, "PB"), (515, 0, "PA"), (1, 0, "PAII")])
def test_fresh_model_batch_predicts_zero(L, variant, algo):
    from fps_b200.ops import native

    kernel = pa_ref.geometry(L, variant)[0]
    n = 2 * pa_ref.cap(kernel, native.sm_count(0)) + 3
    _run(L, variant, algo, False, n=n, launches=2, nnz=(1, 2), fresh=True)


@pytest.mark.parametrize("id64", [False, True])
@pytest.mark.parametrize("range_part", [False, True])
@pytest.mark.parametrize("L,algo,cost", [(7, "ML", True), (515, "PB", True)])
def test_ids_and_partitioning(L, algo, cost, id64, range_part):
    _run(L, 0, algo, cost, id64=id64, range_part=range_part)


# ---- flush to zero --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("L,variant", [(1, 0), (1, 1), (7, 0), (200, 0)])
def test_subnormal_pushes_leave_the_table_unchanged(L, variant):
    """PA-I with C = 1e-30 and |x| ~ 1e-10: every push is ~1e-40, subnormal, and red.add flushes it."""
    rng = np.random.default_rng(L)
    feats = 600
    pa = _model(feats, L, "PAI")
    pa.C = 1e-30
    try:
        _set_table(pa, rng.normal(0, 0.3, (feats, L)))
        before = _table(pa)
        with _Variant(variant):
            batch = _batch(rng, 64, feats, L, (1, 6), mix=False)
            batch = (batch[0], batch[1], (batch[2] * 1e-10).astype(np.float32), batch[3])
            rep, _, _ = _step(pa, batch)
        assert rep.updated.sum() == 64
        np.testing.assert_array_equal(_table(pa), before)
    finally:
        pa.close()


# ---- the block kernel's non-finite check covers all four columns of a chunk -----------------------------------

@pytest.mark.parametrize("L,variant,label", [(5, 1, 1), (200, 0, 101)])
def test_block_kernel_flags_an_infinite_push_in_any_column(L, variant, label):
    from fps_b200.errors import FactorIsNotANumberException
    from fps_b200.models.pa.sparse import SparseVector

    assert pa_ref.geometry(L, variant)[0] == "block" and label % 4 != 0
    feats = 16
    pa = _model(feats, L, "PA")
    try:
        w = np.zeros(L, np.float32)
        w[label] = -3e38
        pa.load_model([(3, w)])
        batch = (np.array([0, 1]), np.array([3]), np.array([10.0], np.float32), np.array([label], np.int32))
        with _Variant(variant):
            rep = pa_ref.replay(_table(pa)[:, :L].astype(np.float64), *batch, algo="PA", binary=False)
            assert rep.bad[0]
            pred = pa.step([SparseVector([3], [10.0], feats)], [label])
        assert pred == [int(rep.pred[0])]
        with pytest.raises(FactorIsNotANumberException):
            pa.check_finite()
    finally:
        pa.close()


# ---- the warp kernel's arg-max with every decision entry at or below -3e38 ------------------------------------

LOW = {  # name: (rows {feature: value of every column}, entries [(feature, x)])
    "minus_inf": ({3: -np.inf}, [(3, 1.0)]),
    "low_norm1": ({3: np.float32(-3.2e38)}, [(3, 1.0)]),
    "low_norm101": ({3: np.float32(-3.2e38), 5: 0.0}, [(3, 1.0), (5, 10.0)]),
}


def _low_case(L, algo, cost, kind):
    from fps_b200.errors import FactorIsNotANumberException

    rows, entries = LOW[kind]
    feats = 16
    pa = _model(feats, L, algo, cost)
    try:
        pa.load_model([(f, np.full(L, v, np.float32)) for f, v in rows.items()])
        batch = (np.array([0, len(entries)]), np.array([f for f, _ in entries]),
                 np.array([x for _, x in entries], np.float32), np.array([L - 1], np.int32))
        before = _table(pa)[:, :L].astype(np.float64)
        rep = pa_ref.replay(before, *batch, algo=algo, binary=False, cost=_cost(L) if cost else None)
        assert rep.pred[0] == 0 and rep.decided[0] and rep.updated[0]
        pred, _, flag = _launch(pa, batch)
        assert pred[0] == 0, pred[0]
        if rep.bad[0]:
            with pytest.raises(FactorIsNotANumberException):
                pa.check_finite()
        else:
            assert flag == 0
            _launch_free_compare(pa, rep, L)
    finally:
        pa.close()


def _launch_free_compare(pa, rep, L):
    got = _table(pa)[:, :L].astype(np.float64)
    np.testing.assert_array_equal(np.isfinite(got), np.isfinite(rep.table))
    fin = np.isfinite(rep.table)
    assert (np.abs(got[fin] - rep.table[fin]) <= MARGIN * rep.tol[fin]).all()


@pytest.mark.parametrize("kind", list(LOW))
@pytest.mark.parametrize("algo", ["PA", "PB"])
@pytest.mark.parametrize("L", [7, 37])
def test_low_decisions_predict_the_first_class(L, algo, kind):
    """OVA and cost-free PB: no cost-matrix read, whatever the arg-max returns."""
    _low_case(L, algo, False, kind)


@pytest.mark.parametrize("kind", list(LOW))
@pytest.mark.parametrize("algo,cost", [("PB", True), ("ML", False), ("ML", True)])
@pytest.mark.parametrize("L", [7, 37])
def test_low_decisions_cost_based(L, algo, cost, kind):
    _low_case(L, algo, cost, kind)


# ---- labels and label counts the kernels cannot take are refused before any launch ---------------------------

@pytest.mark.parametrize("L,labels", [(5, [5]), (5, [-1]), (5, [2, 7]), (1, [0]), (1, [2]), (1, [False])])
def test_bad_labels_are_refused_before_launch(L, labels):
    from fps_b200.models.pa.sparse import SparseVector
    from fps_b200.ops import native

    pa = _model(16, L, "PA")
    try:
        before = _table(pa)
        launches = native.launch_count()
        with pytest.raises(ValueError):
            pa.step([SparseVector([1 + i], [1.0], 16) for i in range(len(labels))], labels)
        assert native.launch_count() == launches
        np.testing.assert_array_equal(_table(pa), before)
    finally:
        pa.close()


@pytest.mark.parametrize("num_labels", [0, 1025])
def test_bad_label_counts_are_refused(num_labels):
    from fps_b200.models.pa.device import DevicePassiveAggressive
    from fps_b200.ops import native

    with pytest.raises(ValueError):
        DevicePassiveAggressive(16, num_labels, False, "PA")
    pa = _model(16, 4, "PA")
    try:
        dev = pa.dev
        pred = torch.empty(1, dtype=torch.int32, device=dev)
        with pytest.raises(RuntimeError):
            native.pa_step(pa.table.table_c, torch.tensor([0, 1], device=dev), torch.tensor([1], dtype=torch.int32,
                           device=dev), torch.ones(1, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
                           pred, binary=False, num_labels=num_labels, algo="PA")
    finally:
        pa.close()
