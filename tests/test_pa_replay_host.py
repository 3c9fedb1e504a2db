"""The fp64 passive-aggressive replay (tests/pa_ref.py) against the host algorithms and a brute-force fp32
evaluation, its dispatch table against the kernel source, and the label refusals of the device wrapper."""
import re
import zlib
from pathlib import Path

import numpy as np
import pytest

from tests import pa_ref

UNL = pa_ref.UNLABELLED
SRC = Path(__file__).resolve().parents[1] / "flink-parameter-server_b200" / "ops" / "csrc" / "fps_pa.cu"

# (host builder, replay algo, binary, C, cost)
_COST = lambda a, b: 0.0 if a == b else 1.0 + 0.25 * abs(a - b)
CASES = {
    "bin_PA": ("PA", True, 0.0, None), "bin_PAI": ("PAI", True, 0.05, None),
    "bin_PAII": ("PAII", True, 0.5, None), "ova_PA": ("PA", False, 0.0, None),
    "ova_PAI": ("PAI", False, 0.1, None), "ova_PAII": ("PAII", False, 0.3, None),
    "PB": ("PB", False, 0.0, _COST), "ML": ("ML", False, 0.0, _COST),
}


def _host(name, L):
    from fps_b200.models.pa.algorithms import PassiveAggressiveBinaryAlgorithm as B
    from fps_b200.models.pa.algorithms import PassiveAggressiveCostBased as CB
    from fps_b200.models.pa.algorithms import PassiveAggressiveOneVersusAll as OVA

    C = CASES[name][2]
    return {"bin_PA": lambda: B.buildPA(), "bin_PAI": lambda: B.buildPAI(C), "bin_PAII": lambda: B.buildPAII(C),
            "ova_PA": lambda: OVA.buildPA(L), "ova_PAI": lambda: OVA.buildPAI(L, C),
            "ova_PAII": lambda: OVA.buildPAII(L, C), "PB": lambda: CB.buildPB(_COST, L),
            "ML": lambda: CB.buildML(_COST, L)}[name]()


def _cost(name, L):
    c = CASES[name][3]
    return None if c is None else np.array([[c(i, j) for j in range(L)] for i in range(L)])


def _batch(rng, n, feats, L, binary, repeats=True, edges=False):
    """Sequential batch over a small feature space (examples overlap), some with a repeated feature."""
    rp, cols, vals, labels = [0], [], [], []
    for ex in range(n):
        k = int(rng.integers(1, 7))
        idx = list(rng.choice(feats, k, replace=False))
        if repeats and ex % 3 == 0:
            idx.append(idx[0])
        x = list(rng.normal(0, 1, len(idx)))
        if edges and ex % 7 == 3:
            idx, x = [], []
        if edges and ex % 7 == 5:
            x = [0.0] * len(idx)
        cols += idx
        vals += x
        rp.append(len(cols))
        if edges and ex % 5 == 4:
            labels.append(UNL)
        else:
            labels.append(int(rng.choice([-1, 1])) if binary else int(rng.integers(L)))
    return (np.array(rp), np.array(cols, dtype=np.int64), np.float32(np.array(vals)).astype(np.float64),
            np.array(labels))


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("L", [3, 6])
def test_replay_without_rounding_equals_host_algorithms(name, L):
    from fps_b200.models.pa.sparse import SparseVector

    algo, binary, C, _ = CASES[name]
    L = 1 if binary else L
    rng = np.random.default_rng(zlib.crc32(f"{name}{L}".encode()))
    feats = 12
    rp, cols, vals, labels = _batch(rng, 40, feats, L, binary)
    W0 = rng.normal(0, 0.3, (feats, L))
    host = _host(name, L)
    rep = pa_ref.replay(W0, rp, cols, vals, labels, algo=algo, binary=binary, C=C, cost=_cost(name, L),
                        fp32=False)
    w = {i: (W0[i, 0] if binary else W0[i].copy()) for i in range(feats)}
    for ex in range(len(labels)):
        v = SparseVector(cols[rp[ex]:rp[ex + 1]], vals[rp[ex]:rp[ex + 1]], feats)
        assert v.activeSize == rp[ex + 1] - rp[ex]          # repeats are kept
        model = {i: w[i] for i in v.indices.tolist()}
        p = host.predict(v, model)
        assert int(p) == rep.pred[ex], ex
        y = labels[ex]
        for i, d in host.delta(v, model, (y > 0) if binary else y):
            w[i] = w[i] + d
    got = np.array([[w[i]] if binary else w[i] for i in range(feats)])
    np.testing.assert_allclose(rep.table, got, rtol=1e-12, atol=1e-12)
    assert rep.updated.all() and not rep.bad.any()


# ---- brute-force fp32 evaluation ---------------------------------------------------------------------------

def _order(k, how, rng):
    if how == "forward":
        return list(range(k))
    if how == "reverse":
        return list(range(k))[::-1]
    return list(rng.permutation(k))


def _sum32(rows, how, rng):
    """fp32 column sums of ``rows`` [k, m]: sequential in some order, or pairwise."""
    if how == "pairwise":
        rows = [r for r in rows]
        if not rows:
            return None
        while len(rows) > 1:
            rows = [rows[i] + rows[i + 1] if i + 1 < len(rows) else rows[i] for i in range(0, len(rows), 2)]
        return rows[0]
    acc = None
    for j in _order(len(rows), how, rng):
        acc = rows[j] if acc is None else acc + rows[j]
    return acc


def fp32_step(table, rp, cols, vals, labels, algo, binary, C, cost, how, seed=0):
    """The kernel's expressions, every operation an np.float32 one, sums in the order ``how``; pushes flushed."""
    f = np.float32
    rng = np.random.default_rng(seed)
    W = np.asarray(table, dtype=np.float32).copy()
    L = W.shape[1]
    C = f(C)
    cm = np.where(np.eye(L, dtype=bool), f(0), f(1)) if cost is None else np.asarray(cost, dtype=np.float32)
    sq = np.sqrt(cm)
    ftz = lambda v: np.where(np.abs(v) < f(pa_ref.FLT_MIN), f(0), v).astype(np.float32)
    n = len(labels)
    pred, loss, bad = np.zeros(n, np.int64), np.full(n, np.nan, np.float32), np.zeros(n, bool)
    with np.errstate(all="ignore"):
        for ex in range(n):
            b, e = int(rp[ex]), int(rp[ex + 1])
            x = np.asarray(vals[b:e], dtype=np.float32)
            idx = cols[b:e]
            d = _sum32([x[j] * W[idx[j]] for j in range(e - b)], how, rng)
            n2 = _sum32([np.array([x[j] * x[j]], np.float32) for j in range(e - b)], how, rng)
            d = np.zeros(L, np.float32) if d is None else d
            n2 = f(0) if n2 is None else n2[0]
            pred[ex] = int(d[0] > 0) if binary else int(np.argmax(d))
            label = int(labels[ex])
            if label == UNL or e == b or not n2 > 0:
                continue
            if binary or algo in ("PA", "PAI", "PAII"):
                y = np.full(L, f(label)) if binary else np.where(np.arange(L) == label, f(1), f(-1)).astype(np.float32)
                l = np.maximum(f(0), f(1) - y * d)
                if algo == "PA":
                    tau = l / n2
                elif algo == "PAI":
                    tau = np.minimum(C, l / n2)
                else:
                    tau = l / (n2 + f(1) / (f(2) * C))
                mult = (tau * y).astype(np.float32)
                if L == 1:
                    loss[ex] = l[0]
            else:
                q = pred[ex]
                if algo == "ML":
                    q = int(np.argmax((d - d[label]) + sq[label]))
                if q == label:
                    continue
                lq = (d[q] - d[label]) + sq[label, q]
                loss[ex] = lq
                tau = lq / (f(2) * n2)
                mult = np.zeros(L, np.float32)
                mult[label], mult[q] = tau, -tau
            for j in range(b, e):
                p = (x[j - b] * mult).astype(np.float32)
                for c0 in range(0, L, 4):
                    s = slice(c0, min(c0 + 4, L))
                    if not (p[s] != 0).any():
                        continue
                    if not np.abs(p[s]).sum(dtype=np.float32) <= f(3e38):
                        bad[ex] = True
                    W[cols[j], s] = ftz(W[cols[j], s] + ftz(p[s]))
    return W, pred, loss, bad


@pytest.mark.parametrize("name,L", [(n, L) for n in CASES for L in ((1,) if CASES[n][1] else (5, 13))])
def test_fp32_evaluation_within_replay_bound(name, L):
    algo, binary, C, _ = CASES[name]
    rng = np.random.default_rng(zlib.crc32(f"{name}{L}fp32".encode()))
    feats = 16
    rp, cols, vals, labels = _batch(rng, 60, feats, L, binary, edges=True)
    W0 = np.float32(rng.normal(0, 0.5, (feats, L))).astype(np.float64)
    cost = _cost(name, L)
    rep = pa_ref.replay(W0, rp, cols, vals, labels, algo=algo, binary=binary, C=C, cost=cost)
    # OVA-PA drives violated margins to exactly -1, so one-feature examples meet near-ties of the prediction
    # on purpose; those never feed an update outside PB and ML
    assert rep.decided.mean() > 0.9 and (rep.decided | (algo not in ("PB", "ML"))).all()
    worst = 0.0
    for how in ("forward", "reverse", "shuffled", "pairwise"):
        for seed in range(3 if how == "shuffled" else 1):
            W, pred, loss, bad = fp32_step(W0, rp, cols, vals, labels, algo, binary, C, cost, how, seed)
            np.testing.assert_array_equal(pred[rep.decided], rep.pred[rep.decided])
            np.testing.assert_array_equal(bad, rep.bad)
            err = np.abs(W - rep.table)
            assert (err <= rep.tol).all(), (how, (err - rep.tol).max())
            worst = max(worst, float((err / np.where(rep.tol > 0, rep.tol, 1)).max()))
            np.testing.assert_array_equal(np.isnan(loss), np.isnan(rep.loss))
            m = ~np.isnan(rep.loss)
            assert (np.abs(loss[m] - rep.loss[m]) <= rep.tol_loss[m]).all()
    assert rep.updated.sum() > 10
    assert worst > 0 or not rep.updated.any()


def test_replay_edge_semantics():
    """Fresh model: exact zero decisions predict 0 clearly; empty, zero-valued and unlabelled examples
    do not update; loss is written only where the kernel writes it."""
    L = 5
    W0 = np.zeros((8, L))
    rp = np.array([0, 2, 2, 3, 4])
    cols = np.array([0, 1, 2, 3])
    vals = np.array([1.0, -2.0, 0.0, 3.0])
    labels = np.array([2, 1, 4, UNL])
    for algo in ("PA", "PB", "ML"):
        r = pa_ref.replay(W0, rp, cols, vals, labels, algo=algo, binary=False)
        assert r.pred.tolist() == [0, 0, 0, 0] and r.decided.all()
        assert r.updated.tolist() == [True, False, False, False]
        assert (r.table[2:] == 0).all()
        assert np.isnan(r.loss[1:]).all()
        assert np.isnan(r.loss[0]) == (algo == "PA")
    # ML without a cost matrix at a zero decision: every other class ties at 1, the first one wins
    r = pa_ref.replay(W0, rp, cols, vals, np.array([0, UNL, UNL, UNL]), algo="ML", binary=False)
    assert r.loss[0] == 1.0 and r.table[0, 1] == -0.1 and r.table[0, 0] == 0.1 and r.decided.all()


def test_replay_flushes_subnormal_pushes():
    W0 = np.zeros((2, 1))
    r = pa_ref.replay(W0, [0, 1], [0], [1e-10], [1], algo="PAI", binary=True, C=1e-30)
    assert r.updated[0] and (r.table == 0).all()
    r = pa_ref.replay(W0, [0, 1], [0], [1e-10], [1], algo="PAI", binary=True, C=1e-30, fp32=False)
    assert r.table[0, 0] > 0


def test_replay_all_minus_inf_decisions_predict_the_first_class():
    L = 6
    W0 = np.zeros((3, L))
    W0[0] = -np.inf
    W0[1] = np.float32(-3.2e38)
    for f, x in ((0, 1.0), (1, 1.0)):
        r = pa_ref.replay(W0, [0, 1], [f], [x], [3], algo="PB", binary=False)
        assert r.pred[0] == 0 and r.decided[0]
    # -3.2e38 with ||x||^2 = 1 pushes 3.2e38 (flagged); with ||x||^2 = 101 it stays finite
    r = pa_ref.replay(W0, [0, 1], [1], [1.0], [3], algo="PA", binary=False)
    assert r.bad[0]
    r = pa_ref.replay(W0, [0, 2], [1, 2], [1.0, 10.0], [3], algo="PA", binary=False)
    assert not r.bad[0] and np.isfinite(r.table[1:]).all() and r.decided[0]


def test_geometry_matches_the_dispatch_ladder():
    src = SRC.read_text()
    body = src[src.index("static int dispatch_pa"):]
    body = body[:body.index("\n}\n")]
    warp = [(int(a), int(b)) for a, b in re.findall(r"nvec <= (\d+)\) fps_pa_step_warp_kernel<IdT, (\d+)>", body)]
    block = [(int(a), int(b)) for a, b in re.findall(r"nvec <= (\d+)\) fps_pa_step_kernel<IdT, (\d+)>", body)]
    assert warp == block == [(1, 1), (2, 2), (4, 4), (8, 8), (16, 16)]
    assert "nvec <= 32 && a.num_labels <= 128 && g_pa_variant == 0" in body
    assert "constexpr int VPL = LPR < 32 ? 1 : PA_MAX_LABELS / 4 / 32;" in src
    assert "#define PA_MAX_LABELS 1024" in src

    def ladder(nvec):
        for lim, lpr in warp:
            if nvec <= lim:
                return lpr
        return 32

    for L in range(1, 1025):
        nvec = -(-L // 4)
        want_warp = ("warp", ladder(nvec), 1) if nvec <= 32 and L <= 128 else ("block", ladder(nvec),
                                                                             8 if ladder(nvec) == 32 else 1)
        assert pa_ref.geometry(L, 0) == want_warp, L
        assert pa_ref.geometry(L, 1) == ("block", ladder(nvec), 8 if ladder(nvec) == 32 else 1), L
    assert len(pa_ref.dispatch_table()) == 12
    for bad in (0, 1025):
        with pytest.raises(ValueError):
            pa_ref.geometry(bad)


def test_device_wrapper_refuses_bad_labels_on_the_host():
    from fps_b200.models.pa.device import DevicePassiveAggressive, labels_array

    assert labels_array([1, -1, None], True, 1).tolist() == [1, -1, UNL]
    assert labels_array([0, 4, None], False, 5).tolist() == [0, 4, UNL]
    for lab in ([0], [2], [False], [-2]):
        with pytest.raises(ValueError):
            labels_array(lab, True, 1)
    for lab in ([5], [-1], [1 << 40]):
        with pytest.raises(ValueError):
            labels_array(lab, False, 5)
    for L in (0, 1025, -3):
        with pytest.raises(ValueError):
            DevicePassiveAggressive(10, L, False, "PA")
