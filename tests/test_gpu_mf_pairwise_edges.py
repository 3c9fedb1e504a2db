"""The pairwise MF steps (``fps_mf_bpr_kernel`` under SGD and row-wise AdaGrad, ``fps_mf_warp_kernel``) and the
pointwise row-wise AdaGrad step (``fps_mf_sgd_fused_kernel`` with ``ADA``) against the fp64 replays of
``tests/pairwise_ref.py`` and ``tests/pointwise_ref.py``, at every dispatch rung, through the native bindings.

Every case is built so that its result does not depend on the order the lane-groups run in: each row is read and
written by one positive (a negative repeated inside one positive's list is replayed in list order), or, for hot rows,
only on coordinates one record owns.  Every table and accumulator is a slice of a larger tensor whose guard rows hold
a sentinel; each case checks the touched rows against the replay within MARGIN times its bound, and that the guard
rows, the padding columns and every row outside the batch are bitwise unchanged."""
import os

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests.pairwise_ref import MARGIN, bpr_replay, geometry, sampled_candidates, warp_replay
from tests.philox_ref import k5_negative
from tests.pointwise_ref import loss_bound, replay as pointwise_replay
from tests.test_gpu_mf_pointwise_edges import SEED, STEP, Guarded, _check_table, _ids, _shift_covering_steps, _table

pytestmark = pytest.mark.gpu

IDS = ("int32", "int64", "packed64")


def _stride(dim):
    return (dim + 3) // 4 * 4


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _rung(dim, max_nvec=128):
    return geometry(_stride(dim), max_nvec)


# dispatch_bpr / dispatch_warp (csrc/fps_mf_bpr.cu, fps_mf_warp.cu): dim -> nvec -> <LPR, VPL>.  Every dim leaves
# lanes or columns empty: 129 puts 2 float4 on lane 0 and 1 on the others, 385 is <32, 4> with uneven lanes.
#   3 <1,1>  7 <2,1>  13 <4,1>  29 <8,1>  61 <16,1>  125 <32,1>  129, 253 <32,2>  300 <32,3>  385, 509 <32,4>
PAIR_DIMS = [3, 7, 13, 29, 61, 125, 129, 253, 300, 385, 509]
PAIR_RUNGS = {(1, 1), (2, 1), (4, 1), (8, 1), (16, 1), (32, 1), (32, 2), (32, 3), (32, 4)}
# dispatch_mf's AdaGrad branch adds <32, 8> (up to 1024 floats)
ADA_DIMS = [3, 7, 13, 29, 61, 125, 253, 300, 509, 1021]
ADA_RUNGS = PAIR_RUNGS | {(32, 8)}
WARP_CS = (1, 2, 4, 8)

# ---- largest observed |error| / (MARGIN * bound), per kernel ---------------------------------------------------
_RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    path = os.environ.get("FPS_BOUND_REPORT")
    if path:
        with open(path, "w") as f:
            for k, v in sorted(_RATIOS.items()):
                f.write(f"{k} {v:.4g}\n")


def _within(got, want, tol, what, kernel):
    got = np.asarray(got, dtype=np.float64)
    err = np.abs(got - want)
    bad = err > MARGIN * tol
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} elements off, worst "
                           f"{float(np.max(err - MARGIN * tol)):.3g} beyond the bound")
    pos = tol > 0
    if pos.any():
        _RATIOS[kernel] = max(_RATIOS.get(kernel, 0.0), float((err[pos] / (MARGIN * tol[pos])).max()))


def _np(t):
    return t.double().cpu().numpy()


def _rows(g, rows, dim):
    return _np(g.t[torch.as_tensor(np.asarray(rows, dtype=np.int64), device=g.t.device), :dim])


def _acc(rows, gen, dev, random):
    g = Guarded(rows, 1, torch.float32, dev)
    g.t.zero_()
    if random:
        g.t[:, 0] = torch.rand(rows, generator=gen, device=dev) * 0.5
    return g


def _neg_tensor(negs, form, dev):
    return torch.from_numpy(np.asarray(negs, dtype=np.int64)).to(dev, torch.int64 if form == "int64" else torch.int32)


def _check_acc(g, before, touched, what):
    _check_table(g, before, 1, touched, what)


# ---- BPR (SGD and AdaGrad) -------------------------------------------------------------------------------------

def _bpr(dev, dim, form, *, ada=False, anchor_div=1, anchor_sharded=False, cand_div=1, cand_sharded=True, reg=0.0,
         n_neg=1, n_pos=600, G_random=True, lr=0.05, seed=0, mixes=True, void_anchors=0, repeat=False, push=False,
         **kw):
    """One mf_bpr_fused launch on a batch whose positives share no row.  ``mixes``: voided negatives, negatives equal
    to their positive and ``rating <= 0`` records; ``repeat``: negatives 2.. repeat negative 0.  Returns the tables
    for bitwise comparisons."""
    gen = torch.Generator(device=dev).manual_seed(1000 * dim + seed)
    rng = np.random.default_rng(1000 * dim + seed)
    kernel = "bpr_adagrad" if ada else "bpr"
    scale = dim ** -0.25
    n_c = n_pos * (1 + n_neg)
    A, Cc = _table(n_pos, dim, scale, gen, dev), _table(n_c, dim, scale, gen, dev)
    A0, C0 = A.t.clone(), Cc.t.clone()
    slots = rng.permutation(n_pos)
    perm = rng.permutation(n_c)
    item_rows, negs = perm[:n_pos], perm[n_pos:].reshape(n_pos, n_neg).copy()
    if repeat:
        negs[:, 2::2] = negs[:, :1]
        negs[:, 3::2] = negs[:, 1:2] if n_neg > 1 else negs[:, :1]
    ratings = np.ones(n_pos, dtype=np.float32)
    if mixes:
        negs[rng.random(negs.shape) < 0.15] = -1
        eq = rng.random(negs.shape) < 0.08
        negs[eq] = np.broadcast_to(item_rows[:, None], negs.shape)[eq]
        ratings[rng.random(n_pos) < 0.1] = np.float32(0.0)
        ratings[rng.random(n_pos) < 0.05] = np.float32(-1.0)
    anchors = slots if anchor_sharded else slots * anchor_div + (anchor_div - 1)
    if void_anchors:
        anchors = np.where(np.arange(n_pos) % void_anchors == 0, -1, anchors)
    cid = (lambda r: r) if cand_sharded else (lambda r: r * cand_div + (cand_div - 1))
    neg_ids = np.where(negs >= 0, cid(negs), -1)
    Ga = Gc = None
    kwargs = dict(negatives=_neg_tensor(neg_ids, form, dev), anchor_div=anchor_div, cand_div=cand_div, **kw)
    if ada:
        Ga, Gc = _acc(n_pos, gen, dev, G_random), _acc(n_c, gen, dev, G_random)
        Ga0, Gc0 = Ga.t.clone(), Gc.t.clone()
        kwargs.update(cand_acc=native.local_table(Gc.t, 1),
                      anchor_acc=native.local_table(Ga.t, 1) if anchor_sharded else Ga.t.view(-1))
    Pt = None
    if push:
        Pt = Guarded(n_c, _stride(dim), torch.float32, dev)
        Pt.t.zero_()
        kwargs["push_tab"] = native.local_table(Pt.t, dim)
    stats = torch.zeros(3, device=dev)
    nan = torch.zeros(1, dtype=torch.int32, device=dev)
    a, b, c = _ids(anchors, cid(item_rows), ratings, form, dev)
    native.mf_bpr_fused(a, b, c, native.local_table(A.t, dim) if anchor_sharded else A.t,
                        native.local_table(Cc.t, dim) if cand_sharded else Cc.t, lr, reg, stats=stats, nan_flag=nan,
                        **kwargs)
    torch.cuda.synchronize()
    # the replay over the positives the kernel takes
    ok = (ratings > 0) & (anchors >= 0)
    s, it = slots[ok], item_rows[ok]
    nr = np.where(negs[ok] == it[:, None], -1, negs[ok])
    u, vi = _np(A0[torch.from_numpy(s).to(dev), :dim]), _np(C0[torch.from_numpy(it).to(dev), :dim])
    vj = _np(C0[torch.from_numpy(np.maximum(nr, 0)).to(dev), :dim]) * (nr >= 0)[..., None]
    acc = None
    if ada:
        acc = (_np(Ga0[torch.from_numpy(s).to(dev), 0]), _np(Gc0[torch.from_numpy(it).to(dev), 0]),
               _np(Gc0[torch.from_numpy(np.maximum(nr, 0)).to(dev), 0]), dim)
    res = bpr_replay(u, vi, vj, nr, lr, reg, _stride(dim), acc)
    _within(_rows(A, s, dim), res.u, res.tol_u, "anchor rows", kernel)
    dest = Pt if push else Cc
    if push:   # the push table receives the deltas; the candidate table stays as it was
        assert torch.equal(Cc.t, C0)
        Cc.check_guards()
        _within(_rows(Pt, it, dim), res.vi - vi, res.tol_vi, "pushed v_i deltas", kernel)
    else:
        _within(_rows(Cc, it, dim), res.vi, res.tol_vi, "positive rows", kernel)
    final, Gfinal = {}, {}
    for t in range(nr.shape[1]):
        for p in np.flatnonzero(nr[:, t] >= 0):
            final[int(nr[p, t])] = (res.vj[p, t] - (vj[p, t] if push else 0.0), res.tol_vj[p, t])
            if ada:
                Gfinal[int(nr[p, t])] = (res.Gj[p, t], res.tol_Gj[p, t])
    if final:
        rows = np.array(sorted(final))
        _within(_rows(dest, rows, dim), np.stack([final[r][0] for r in rows]),
                np.stack([final[r][1] for r in rows]), "negative rows", kernel)
    touched_c = np.concatenate([it, np.array(sorted(final), dtype=np.int64)])
    _check_table(A, A0, dim, s, "anchor table")
    if push:
        _check_table(Pt, torch.zeros_like(Pt.t), dim, touched_c, "push table")
    else:
        _check_table(Cc, C0, dim, touched_c, "candidate table")
    if ada:
        assert res.smooth
        _within(_np(Ga.t[torch.from_numpy(s).to(dev), 0]), res.Gu, res.tol_Gu, "anchor G", kernel)
        _within(_np(Gc.t[torch.from_numpy(it).to(dev), 0]), res.Gi, res.tol_Gi, "positive G", kernel)
        if Gfinal:
            rows = np.array(sorted(Gfinal))
            _within(_np(Gc.t[torch.from_numpy(rows).to(dev), 0]), np.array([Gfinal[r][0] for r in rows]),
                    np.array([Gfinal[r][1] for r in rows]), "negative G", kernel)
        _check_acc(Ga, Ga0, s[res.n_live > 0], "anchor accumulators")
        _check_acc(Gc, Gc0, np.concatenate([it[res.n_live > 0], np.array(sorted(Gfinal), dtype=np.int64)]),
                   "candidate accumulators")
    st = stats.cpu().numpy().astype(np.float64)
    assert st[1] == res.count
    assert abs(st[0] - res.loss) <= MARGIN * res.tol_loss
    assert res.xpos_lo <= st[2] <= res.xpos_hi
    assert int(nan.item()) == 0
    return A.t, Cc.t, (Ga.t if ada else None), (Gc.t if ada else None), res


def _bpr_cases(ada):
    """Every (rung, id form) pair; anchor forms local (div 1, 3, 4) and ShardTable; candidates local (div 1, 3) and
    ShardTable (AdaGrad: ShardTable only); reg 0 and 0.01; n_neg 1 and 4; AdaGrad from random and from zero G."""
    cases = []
    for i, dim in enumerate(PAIR_DIMS):
        for f, form in enumerate(IDS):
            j = i + f
            anchor = ("local", 1) if j % 4 == 0 else ("local", 3) if j % 4 == 1 else ("local", 4) if j % 4 == 2 \
                else ("shard", 1)
            cand = ("shard", 1) if ada or j % 3 == 0 else ("local", 1 + 2 * (j % 2))
            cases.append((dim, form, anchor, cand, 0.01 * (j % 2), 4 if (j // 2) % 2 else 1, j % 3 != 2))
    return cases


BPR_CASES = {False: _bpr_cases(False), True: _bpr_cases(True)}


def test_rung_cases_cover_the_ladders():
    for ada in (False, True):
        cases = BPR_CASES[ada]
        assert {(_rung(d), f) for d, f, *_ in cases} == {(r, f) for r in PAIR_RUNGS for f in IDS}
        assert {a for _, _, a, *_ in cases} == {("local", 1), ("local", 3), ("local", 4), ("shard", 1)}
        assert {n for *_, n, _ in cases} == {1, 4} and {r for *_, r, _, _ in cases} == {0.0, 0.01}
        assert {c for _, _, _, c, *_ in cases} == ({("shard", 1)} if ada else {("shard", 1), ("local", 1),
                                                                               ("local", 3)})
    assert {g for *_, g in BPR_CASES[True]} == {True, False}
    assert {(_rung(d), c) for d, _, c, *_ in WARP_CASES} == {(r, c) for r in PAIR_RUNGS for c in WARP_CS}
    assert {(c, f) for _, f, c, *_ in WARP_CASES} == {(c, f) for c in WARP_CS for f in IDS}
    assert {_rung(d, 256) for d, *_ in ADA_CASES} == ADA_RUNGS
    assert {(e, ud, sh) for _, _, e, ud, sh, _ in ADA_CASES} >= {(e, 1, False) for e in range(3)}


@pytest.mark.parametrize("dim,form,anchor,cand,reg,n_neg,G_random", BPR_CASES[False])
def test_bpr_rung_matches_fp64_replay(dev, dim, form, anchor, cand, reg, n_neg, G_random):
    _bpr(dev, dim, form, anchor_sharded=anchor[0] == "shard", anchor_div=anchor[1],
         cand_sharded=cand[0] == "shard", cand_div=cand[1], reg=reg, n_neg=n_neg)


@pytest.mark.parametrize("dim,form,anchor,cand,reg,n_neg,G_random", BPR_CASES[True])
def test_bpr_adagrad_rung_matches_fp64_replay(dev, dim, form, anchor, cand, reg, n_neg, G_random):
    _bpr(dev, dim, form, ada=True, anchor_sharded=anchor[0] == "shard", anchor_div=anchor[1], reg=reg, n_neg=n_neg,
         G_random=G_random)


@pytest.mark.parametrize("ada", [False, True])
def test_bpr_dim_above_512_is_refused(dev, ada):
    A, Cc = torch.zeros(8, 516, device=dev), torch.zeros(8, 516, device=dev)
    ids = torch.arange(4, dtype=torch.int32, device=dev)
    kw = dict(cand_acc=native.local_table(torch.zeros(8, 1, device=dev), 1),
              anchor_acc=torch.zeros(8, device=dev)) if ada else {}
    with pytest.raises(RuntimeError, match="-1000"):
        native.mf_bpr_fused(ids, ids, torch.ones(4, device=dev), A, native.local_table(Cc, 513), 0.1,
                            negatives=ids.view(4, 1).flip(0).contiguous(), **kw)
    torch.cuda.synchronize()
    assert not A.any() and not Cc.any()


# ---- a negative repeated in one positive's list ------------------------------------------------------------------

@pytest.mark.parametrize("ada", [False, True])
@pytest.mark.parametrize("dim,form", [(7, "int32"), (61, "int64"), (125, "packed64"), (300, "int32")])
def test_repeated_negative_is_applied_in_list_order(dev, ada, dim, form):
    """Negatives [a, b, a, b]: the repeat reads the row with the earlier push applied and, under AdaGrad, G_j + s_j
    of the earlier triple, on every lane of the group."""
    _bpr(dev, dim, form, ada=ada, n_neg=4, repeat=True, reg=0.01, mixes=False, G_random=dim != 61)


# ---- WARP ------------------------------------------------------------------------------------------------------

def _warp(dev, dim, form, C, *, T=6, margin=-0.25, rank_items=1 << 20, n_pos=600, reg=0.01, lr=0.05, seed=0,
          cand_sharded=True, void_anchors=0, push=False, mixes=True, **kw):
    gen = torch.Generator(device=dev).manual_seed(7000 + 1000 * dim + seed)
    rng = np.random.default_rng(7000 + 1000 * dim + seed)
    scale = dim ** -0.25
    n_c = n_pos * (1 + T)
    A, Cc = _table(n_pos, dim, scale, gen, dev), _table(n_c, dim, scale, gen, dev)
    A0, C0 = A.t.clone(), Cc.t.clone()
    slots = rng.permutation(n_pos)
    perm = rng.permutation(n_c)
    item_rows, negs = perm[:n_pos], perm[n_pos:].reshape(n_pos, T).copy()
    ratings = np.ones(n_pos, dtype=np.float32)
    if mixes:
        negs[rng.random(negs.shape) < 0.15] = -1
        eq = rng.random(negs.shape) < 0.05
        negs[eq] = np.broadcast_to(item_rows[:, None], negs.shape)[eq]
        ratings[rng.random(n_pos) < 0.1] = np.float32(0.0)
    anchors = slots.copy()
    if void_anchors:
        anchors = np.where(np.arange(n_pos) % void_anchors == 0, -1, anchors)
    Pt = None
    if push:
        Pt = Guarded(n_c, _stride(dim), torch.float32, dev)
        Pt.t.zero_()
        kw["push_tab"] = native.local_table(Pt.t, dim)
    stats = torch.zeros(4, device=dev)
    nan = torch.zeros(1, dtype=torch.int32, device=dev)
    a, b, c = _ids(anchors, item_rows, ratings, form, dev)
    native.mf_warp_fused(a, b, c, A.t, native.local_table(Cc.t, dim) if cand_sharded else Cc.t, lr, reg,
                         margin=margin, rank_items=rank_items, negatives=_neg_tensor(negs, form, dev), stats=stats,
                         nan_flag=nan, trial_block=C, **kw)
    torch.cuda.synchronize()
    ok = (ratings > 0) & (anchors >= 0)
    s, it = slots[ok], item_rows[ok]
    nr = np.where(negs[ok] == it[:, None], -1, negs[ok])
    u, vi = _np(A0[torch.from_numpy(s).to(dev), :dim]), _np(C0[torch.from_numpy(it).to(dev), :dim])
    vj = _np(C0[torch.from_numpy(np.maximum(nr, 0)).to(dev), :dim])
    res = warp_replay(u, vi, vj, nr >= 0, lr, reg, margin, rank_items, _stride(dim))
    assert res.decided.all(), f"{int((~res.decided).sum())} positives with an x within the bound of the margin"
    h = res.hit
    js = nr[np.flatnonzero(h), res.tstar[h]]
    _within(_rows(A, s, dim), res.u, res.tol_u, "anchor rows", "warp")
    dest = Pt if push else Cc
    base_i = vi[h] if push else 0.0
    base_j = vj[np.flatnonzero(h), res.tstar[h]] if push else 0.0
    _within(_rows(dest, it[h], dim), res.vi[h] - base_i, res.tol_vi[h], "positive rows", "warp")
    _within(_rows(dest, js, dim), res.vs[h] - base_j, res.tol_vs[h], "violator rows", "warp")
    _check_table(A, A0, dim, s[h], "anchor table")
    if push:
        assert torch.equal(Cc.t, C0)
        Cc.check_guards()
        _check_table(Pt, torch.zeros_like(Pt.t), dim, np.concatenate([it[h], js]), "push table")
    else:
        _check_table(Cc, C0, dim, np.concatenate([it[h], js]), "candidate table")
    st = stats.cpu().numpy().astype(np.float64)
    assert st[1] == res.updated and st[2] == res.examined and st[3] == ok.sum()
    assert abs(st[0] - res.loss) <= MARGIN * res.tol_loss
    assert int(nan.item()) == 0
    return A.t, Cc.t, res


# Every (geometry, C) pair; forms cycle so that every (C, id form) pair occurs.  The margin alternates between
# -0.25 (the first violator anywhere from t = 0 to none) and 0.1; rank_items 2 makes L = 0 (a decay-only update
# that still counts), 5 a small L that depends on n, 2^20 a large one.
WARP_DIMS = [3, 7, 13, 29, 61, 125, 253, 300, 509]
WARP_CASES = [(dim, IDS[(i + ci) % 3], C, (-0.25, 0.1)[(i + ci) % 2], (2, 5, 1 << 20)[(i + 2 * ci) % 3])
              for i, dim in enumerate(WARP_DIMS) for ci, C in enumerate(WARP_CS)]


@pytest.mark.parametrize("dim,form,C,margin,rank_items", WARP_CASES)
def test_warp_geometry_and_trial_block_match_fp64_replay(dev, dim, form, C, margin, rank_items):
    _, _, res = _warp(dev, dim, form, C, margin=margin, rank_items=rank_items, cand_sharded=(dim + C) % 2 == 0)
    if margin < 0:   # the first violator at t = 0, in the middle, at the last slot, and none
        t = set(res.tstar.tolist())
        assert {-1, 0, 5} <= t and t & {1, 2, 3, 4}
    if rank_items == 2:
        assert (res.L == 0).all() and res.updated > 0


# ---- pointwise AdaGrad -----------------------------------------------------------------------------------------

def _pw_adagrad(dev, dim, form, err_mode, *, user_div=1, user_sharded=False, n=2000, rows=2400, G_random=True,
                seed=0, lr=0.1, **kw):
    gen = torch.Generator(device=dev).manual_seed(3000 + 1000 * dim + seed)
    rng = np.random.default_rng(3000 + 1000 * dim + seed)
    scale = dim ** -0.25
    U, V = _table(rows, dim, scale, gen, dev), _table(rows, dim, scale, gen, dev)
    Ua, Va = _acc(rows, gen, dev, G_random), _acc(rows, gen, dev, G_random)
    U0, V0, Ua0, Va0 = U.t.clone(), V.t.clone(), Ua.t.clone(), Va.t.clone()
    slots, items = rng.permutation(rows)[:n], rng.permutation(rows)[:n]
    r = (rng.integers(1, 9, size=n) * 0.5 if err_mode == 1 else rng.integers(0, 2, size=n)).astype(np.float32)
    users = slots if user_sharded else slots * user_div + (user_div - 1)
    stats = torch.zeros(2, device=dev)
    nan = torch.zeros(1, dtype=torch.int32, device=dev)
    a, b, c = _ids(users, items, r, form, dev)
    native.mf_sgd_fused(a, b, c, native.local_table(U.t, dim) if user_sharded else U.t, user_div,
                        native.local_table(V.t, dim), lr, err_mode=err_mode, stats=stats, nan_flag=nan,
                        item_acc=native.local_table(Va.t, 1),
                        user_acc=native.local_table(Ua.t, 1) if user_sharded else Ua.t.view(-1), **kw)
    torch.cuda.synchronize()
    ts, ti = torch.from_numpy(slots).to(dev), torch.from_numpy(items).to(dev)
    res = pointwise_replay(_np(U0[ts, :dim]), _np(V0[ti, :dim]), r.astype(np.float64), lr, err_mode,
                           _rung(dim, 256)[0], acc=(_np(Ua0[ts, 0]), _np(Va0[ti, 0])))
    assert res.e_ok
    _within(_rows(U, slots, dim), res.u, res.tol_u, "user rows", "pointwise_adagrad")
    _within(_rows(V, items, dim), res.v, res.tol_v, "item rows", "pointwise_adagrad")
    _within(_np(Ua.t[ts, 0]), res.Gu, res.tol_Gu, "user G", "pointwise_adagrad")
    _within(_np(Va.t[ti, 0]), res.Gv, res.tol_Gv, "item G", "pointwise_adagrad")
    for g, g0, t, what in ((U, U0, slots, "user table"), (V, V0, items, "item table")):
        _check_table(g, g0, dim, t, what)
    _check_acc(Ua, Ua0, slots, "user accumulators")
    _check_acc(Va, Va0, items, "item accumulators")
    st = stats.cpu().numpy().astype(np.float64)
    assert st[1] == n
    assert abs(st[0] - (res.resid ** 2).sum()) <= MARGIN * loss_bound(res.resid, res.tol_resid)
    assert int(nan.item()) == 0
    return U.t, V.t, Ua.t, Va.t


# Each rung twice: a worker-local user table (user_div 1 or 3) with a [n] user_acc tensor, and a ShardTable user
# table with a stride-1 ShardTable user_acc; error rules and id forms cycle; G from random and from zero.
ADA_CASES = [(dim, IDS[(i + s) % 3], (i + s) % 3, 3 if (i + s) % 2 and not s else 1, s == 1, (i + s) % 2 == 0)
             for i, dim in enumerate(ADA_DIMS) for s in (0, 1)]


@pytest.mark.parametrize("dim,form,err_mode,user_div,user_sharded,G_random", ADA_CASES)
def test_pointwise_adagrad_rung_matches_fp64_replay(dev, dim, form, err_mode, user_div, user_sharded, G_random):
    _pw_adagrad(dev, dim, form, err_mode, user_div=user_div, user_sharded=user_sharded, G_random=G_random)


# ---- in-kernel negatives, replayed -------------------------------------------------------------------------------

def _disjoint(items, negs):
    """Positives whose rows (positive and candidates, all different) meet no earlier kept positive's rows."""
    used, keep = set(), np.zeros(len(items), dtype=bool)
    for p in range(len(items)):
        rows = {int(items[p]), *map(int, negs[p])}
        if len(rows) == 1 + negs.shape[1] and not rows & used:
            used |= rows
            keep[p] = True
    return keep


@pytest.mark.parametrize("form,n_neg", [("int32", 1), ("int64", 3), ("packed64", 2)])
def test_bpr_sampled_negatives_match_the_replayed_stream(dev, form, n_neg):
    """All-zero candidate table, reg 0: x = 0 and g = lr / 2 exactly, so u stays bitwise, v_i becomes n_live g u
    and each drawn row -g u, bitwise."""
    dim, n_pos, num_items, lr = 29, 1500, 1 << 16, 0.25
    gen = torch.Generator(device=dev).manual_seed(11)
    A = _table(n_pos, dim, 0.5, gen, dev)
    Cc = Guarded(num_items, _stride(dim), torch.float32, dev)
    Cc.t.zero_()
    A0 = A.t.clone()
    rng = np.random.default_rng(12)
    items = rng.integers(0, num_items, n_pos)
    items[:200] = k5_negative(np.arange(200), 1, np.full(200, -1), num_items, STEP, SEED)[1]   # rejection fires
    negs = sampled_candidates(n_pos, items, n_neg, num_items, STEP, SEED)
    keep = _disjoint(items, negs)
    assert 0.8 * n_pos < keep.sum() < n_pos
    anchors = np.where(keep, rng.permutation(n_pos), -1) if form != "packed64" else rng.permutation(n_pos)
    ratings = np.where(keep, 1.0, 0.0).astype(np.float32)
    stats = torch.zeros(3, device=dev)
    a, b, c = _ids(anchors, items, ratings, form, dev)
    native.mf_bpr_fused(a, b, c, A.t, native.local_table(Cc.t, dim), lr, 0.0, n_neg=n_neg, num_items=num_items,
                        seed=SEED, step=STEP, stats=stats)
    torch.cuda.synchronize()
    A.check_guards()
    Cc.check_guards()
    assert torch.equal(A.t, A0)
    g = np.float32(lr) / np.float32(2)
    u = A0.cpu().numpy()
    want = np.zeros((num_items, _stride(dim)), dtype=np.float32)
    for p in np.flatnonzero(keep):
        uu = u[anchors[p]]
        want[items[p]] = (np.float32(n_neg) * g) * uu
        for j in negs[p]:
            want[j] = (-g) * uu
    assert np.array_equal(Cc.t.cpu().numpy(), want)
    assert stats[1].item() == keep.sum() * n_neg and stats[2].item() == 0


@pytest.mark.parametrize("form,T", [("int32", 4), ("int64", 7), ("packed64", 3)])
def test_warp_sampled_candidates_match_the_replayed_stream(dev, form, T):
    """Random rows: which candidate violates, and so stats[2] (the live candidates examined), follows the draws."""
    dim, n_pos, num_items, lr, margin = 13, 1200, 1 << 16, 0.05, -0.2
    gen = torch.Generator(device=dev).manual_seed(13)
    A, Cc = _table(n_pos, dim, 0.6, gen, dev), _table(num_items, dim, 0.6, gen, dev)
    A0, C0 = A.t.clone(), Cc.t.clone()
    rng = np.random.default_rng(14)
    items = rng.integers(0, num_items, n_pos)
    negs = sampled_candidates(n_pos, items, T, num_items, STEP, SEED)
    keep = _disjoint(items, negs)
    slots = rng.permutation(n_pos)
    ratings = np.where(keep, 1.0, 0.0).astype(np.float32)
    stats = torch.zeros(4, device=dev)
    a, b, c = _ids(slots, items, ratings, form, dev)
    native.mf_warp_fused(a, b, c, A.t, native.local_table(Cc.t, dim), lr, 0.01, margin=margin, n_neg=T,
                         num_items=num_items, seed=SEED, step=STEP, stats=stats)
    torch.cuda.synchronize()
    s, it, nr = slots[keep], items[keep], negs[keep]
    u, vi = _np(A0[torch.from_numpy(s).to(dev), :dim]), _np(C0[torch.from_numpy(it).to(dev), :dim])
    vj = _np(C0[torch.from_numpy(nr).to(dev), :dim])
    res = warp_replay(u, vi, vj, np.ones(nr.shape, bool), lr, 0.01, margin, num_items, _stride(dim))
    assert res.decided.all() and res.n.min() == 1 and (~res.hit).any()
    h = res.hit
    js = nr[np.flatnonzero(h), res.tstar[h]]
    _within(_rows(A, s, dim), res.u, res.tol_u, "anchor rows", "warp")
    _within(_rows(Cc, js, dim), res.vs[h], res.tol_vs[h], "violator rows", "warp")
    _check_table(A, A0, dim, s[h], "anchor table")
    _check_table(Cc, C0, dim, np.concatenate([it[h], js]), "candidate table")
    st = stats.cpu().numpy()
    assert st[1] == res.updated and st[2] == res.examined and st[3] == keep.sum()


def test_small_catalogue_candidates_follow_the_stream(dev):
    """One positive per launch whose item is its own first raw draw, catalogues of 2..9 items, steps covering every
    s.z % 7: BPR's four sampled negatives (repeats replayed in list order) and WARP's first violator and count."""
    dim, lr = 13, 0.1
    gen = torch.Generator(device=dev).manual_seed(15)
    for num_items in range(2, 10):
        for step in _shift_covering_steps():
            raw = k5_negative([0], 1, [-1], num_items, step, SEED)[1]
            negs = sampled_candidates(1, raw, 4, num_items, step, SEED)
            assert (negs != raw[0]).all()
            A, Cc = _table(1, dim, 0.5, gen, dev), _table(num_items, dim, 0.5, gen, dev)
            A0, C0 = A.t.clone(), Cc.t.clone()
            a, b, c = _ids([0], raw, [1.0], "int32", dev)
            native.mf_bpr_fused(a, b, c, A.t, native.local_table(Cc.t, dim), lr, 0.01, n_neg=4, num_items=num_items,
                                seed=SEED, step=step)
            torch.cuda.synchronize()
            u, vi = _np(A0[:1, :dim]), _np(C0[torch.from_numpy(raw).to(dev), :dim])
            res = bpr_replay(u, vi, _np(C0[torch.from_numpy(negs[0]).to(dev), :dim])[None], negs, lr, 0.01,
                             _stride(dim))
            _within(_rows(A, [0], dim), res.u, res.tol_u, "anchor", "bpr")
            _within(_rows(Cc, raw, dim), res.vi, res.tol_vi, "positive", "bpr")
            last = {int(j): t for t, j in enumerate(negs[0])}
            rows = np.array(sorted(last))
            _within(_rows(Cc, rows, dim), res.vj[0, [last[r] for r in rows]], res.tol_vj[0, [last[r] for r in rows]],
                    "negatives", "bpr")
            _check_table(Cc, C0, dim, np.concatenate([raw, rows]), "candidate table")
            # WARP on fresh tables: the margin puts the first violator at the first candidate whose x is lowest
            A.t.copy_(A0)
            Cc.t.copy_(C0)
            vj = _np(C0[torch.from_numpy(negs[0]).to(dev), :dim])[None]
            x = (u[0] * (vi[0] - vj[0])).sum(1)
            margin = float(x.min()) + 1e-3
            stats = torch.zeros(4, device=dev)
            native.mf_warp_fused(a, b, c, A.t, native.local_table(Cc.t, dim), lr, 0.0, margin=margin, n_neg=4,
                                 num_items=num_items, seed=SEED, step=step, stats=stats)
            torch.cuda.synchronize()
            wr = warp_replay(u, vi, vj, np.ones((1, 4), bool), lr, 0.0, margin, num_items, _stride(dim))
            assert wr.decided.all() and wr.hit[0]
            assert stats[2].item() == wr.n[0] == wr.tstar[0] + 1
            j = int(negs[0, wr.tstar[0]])
            _within(_rows(Cc, [j], dim), wr.vs, wr.tol_vs, "violator", "warp")
            _check_table(Cc, C0, dim, np.array([raw[0], j]), "candidate table")


@pytest.mark.parametrize("form,neg_rate", [("int32", 1), ("int64", 3)])
def test_pointwise_adagrad_sampled_negatives_match_the_replay(dev, form, neg_rate):
    """The implicit-feedback setting (negative_sample_rate > 0, optimizer="adagrad"): item table all zero, so each
    user row and its G stay bitwise (delta_u = e v = 0), and each drawn row takes lr e u / (sqrt(G + s) + eps) with
    e = r - 1/2 (err_mode 2)."""
    dim, n_pos, num_items, lr = 29, 1500, 1 << 18, 0.1
    gen = torch.Generator(device=dev).manual_seed(16)
    U = _table(n_pos, dim, 0.5, gen, dev)
    V = Guarded(num_items, _stride(dim), torch.float32, dev)
    V.t.zero_()
    Ua, Va = _acc(n_pos, gen, dev, True), _acc(num_items, gen, dev, True)
    U0, Ua0, Va0 = U.t.clone(), Ua.t.clone(), Va.t.clone()
    pos = np.arange(n_pos)
    items = k5_negative(pos, 1, np.full(n_pos, -1), num_items, STEP, SEED)[1]
    negs = np.stack([k5_negative(pos, j, items, num_items, STEP, SEED)[0] for j in range(1, neg_rate + 1)], 1)
    keep = _disjoint(items, negs)
    users = np.where(keep, np.random.default_rng(17).permutation(n_pos), -1)
    stats = torch.zeros(2, device=dev)
    a, b, c = _ids(users, items, np.ones(n_pos, np.float32), form, dev)
    native.mf_sgd_fused(a, b, c, U.t, 1, native.local_table(V.t, dim), lr, err_mode=2, neg_rate=neg_rate,
                        num_items=num_items, seed=SEED, step=STEP, stats=stats, item_acc=native.local_table(Va.t, 1),
                        user_acc=Ua.t.view(-1))
    torch.cuda.synchronize()
    assert torch.equal(U.t, U0) and torch.equal(Ua.t, Ua0)
    U.check_guards()
    Ua.check_guards()
    kp = np.flatnonzero(keep)
    uu = _np(U0[torch.from_numpy(users[kp]).to(dev), :dim])
    u_all = np.concatenate([uu] + [uu] * neg_rate)
    r = np.concatenate([np.ones(len(kp))] + [np.zeros(len(kp))] * neg_rate)
    rows = np.concatenate([items[kp]] + [negs[kp, j] for j in range(neg_rate)])
    tr = torch.from_numpy(rows).to(dev)
    res = pointwise_replay(u_all, np.zeros_like(u_all), r, lr, 2, _rung(dim, 256)[0],
                           acc=(np.zeros(len(r)), _np(Va0[tr, 0])))
    assert res.e_ok
    _within(_rows(V, rows, dim), res.v, res.tol_v, "drawn rows", "pointwise_adagrad")
    _within(_np(Va.t[tr, 0]), res.Gv, res.tol_Gv, "drawn G", "pointwise_adagrad")
    _check_table(V, torch.zeros_like(V.t), dim, rows, "item table")
    _check_acc(Va, Va0, rows, "item accumulators")
    assert stats[1].item() == len(kp) * (1 + neg_rate)


# ---- hot rows ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("loss,dim", [("bpr", 13), ("bpr", 125), ("warp", 13), ("warp", 61)])
def test_hot_positive_is_schedule_free(dev, loss, dim):
    """Anchors i = 0..dim-1 with rows c_i e_i share one positive h, each with its own negative, reg 0: record i
    reads and pushes only coordinate i of v_h, so v_h ends at the replay's value and every negative row is its
    record's.  Anchor coordinate k != i reads v_h[k] before or after record k's push: either replay is accepted."""
    lr = 0.05
    gen = torch.Generator(device=dev).manual_seed(dim)
    rng = np.random.default_rng(dim)
    n = dim
    Cc = _table(n + 1, dim, 0.5, gen, dev)
    C0 = Cc.t.clone()
    A = Guarded(n, _stride(dim), torch.float32, dev)
    A.t.zero_()
    cvals = (rng.random(n) * 0.9 + 0.1).astype(np.float32)
    A.t[torch.arange(n, device=dev), torch.arange(n, device=dev)] = torch.from_numpy(cvals).to(dev)
    A0 = A.t.clone()
    hot = n
    order = rng.permutation(n)
    negs = np.arange(n)[order][:, None]
    a, b, c = _ids(order, np.full(n, hot), np.ones(n, np.float32), "int32", dev)
    kw = dict(negatives=_neg_tensor(negs, "int32", dev))
    if loss == "bpr":
        native.mf_bpr_fused(a, b, c, A.t, native.local_table(Cc.t, dim), lr, 0.0, **kw)
    else:
        native.mf_warp_fused(a, b, c, A.t, native.local_table(Cc.t, dim), lr, 0.0, margin=10.0, rank_items=50, **kw)
    torch.cuda.synchronize()
    u = _np(A0[:, :dim])
    vh = np.repeat(_np(C0[hot:hot + 1, :dim]), n, 0)
    vj = _np(C0[:n, :dim])[:, None]
    neg_ids = np.arange(n)[:, None]

    def replay(vi):
        if loss == "bpr":
            r = bpr_replay(u, vi, vj, neg_ids, lr, 0.0, _stride(dim))
            return r, r.vi, r.tol_vi, r.vj[:, 0], r.tol_vj[:, 0]
        r = warp_replay(u, vi, vj, np.ones((n, 1), bool), lr, 0.0, 10.0, 50, _stride(dim))
        assert r.hit.all() and r.decided.all()
        return r, r.vi, r.tol_vi, r.vs, r.tol_vs

    before, vi1, tvi, vj1, tvj = replay(vh)
    eye = np.eye(n, dtype=bool)
    hot_want, hot_tol = vh[0].copy(), np.zeros(dim)
    hot_want[eye.any(0)] = vi1[eye]
    hot_tol[eye.any(0)] = tvi[eye]
    kern = "bpr" if loss == "bpr" else "warp"
    _within(_np(Cc.t[hot, :dim]), hot_want, hot_tol, "hot row", kern)
    _within(_np(Cc.t[:n, :dim]), vj1, tvj, "negative rows", kern)
    # record i's g from its own coordinate; off it, u[k] = g (v_h[k] - v_j[k]) with v_h[k] before or after record k
    vjd = vj[:, 0]
    g = (before.u - u)[eye] / (vh[0] - vjd)[eye]
    after_u = u + g[:, None] * (hot_want[None] - vjd)
    after_tol = before.tol_u + np.abs(g)[:, None] * hot_tol[None]
    got = _np(A.t[:, :dim])
    ok_b = np.abs(got - before.u) <= MARGIN * before.tol_u
    ok_a = np.abs(got - after_u) <= MARGIN * after_tol
    assert (ok_b | ok_a).all(), f"{int((~(ok_b | ok_a)).sum())} anchor elements match neither schedule"
    assert not A.t[:, dim:].any()
    A.check_guards()
    Cc.check_guards()


# ---- grid-stride rounds ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel,dim,C", [("bpr", 13, 0), ("bpr", 300, 0), ("bpr_adagrad", 61, 0),
                                          ("warp", 29, 1), ("warp", 61, 4), ("pointwise_adagrad", 7, 0)])
def test_grid_stride_rounds_equal_the_default_grid(dev, kernel, dim, C):
    """A grid capped to one CTA by max_inflight_rows and to one CTA per SM by reserve_total: every lane-group runs
    two or more rounds with a partial last one (WARP: with very different trial counts per positive), bitwise equal
    to the default grid."""
    lpr = _rung(dim, 256)[0]
    n = native.sm_count(0) * (256 // lpr) * (2 if kernel == "pointwise_adagrad" else 1)
    n = n + n // 2 + 1
    runs = []
    for kw in ({}, {"max_inflight_rows": 1}, {"reserve_total": 1 << 20}):
        if kernel in ("bpr", "bpr_adagrad"):
            runs.append(_bpr(dev, dim, "int32", ada=kernel == "bpr_adagrad", n_neg=2, n_pos=n, reg=0.01, **kw)[:4])
        elif kernel == "warp":
            runs.append(_warp(dev, dim, "int64", C, T=8, margin=-0.3, n_pos=n, **kw)[:2])
        else:
            runs.append(_pw_adagrad(dev, dim, "int32", 1, n=n, rows=n + 300, **kw))
    for other in runs[1:]:
        for x, y in zip(runs[0], other):
            assert x is None or torch.equal(x, y)


# ---- voids and no-ops --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel,form", [("bpr", "int32"), ("bpr", "int64"), ("bpr_adagrad", "int32"),
                                         ("bpr_adagrad", "int64"), ("warp", "int32"), ("warp", "int64")])
def test_void_anchor_addresses_a_guard_row_never_a_live_one(dev, kernel, form):
    """anchor -1 with anchor_div 1 is the row (and accumulator) before the table: a guard row here."""
    if kernel == "warp":
        _warp(dev, 29, form, 1, void_anchors=3)
    else:
        _bpr(dev, 29, form, ada=kernel == "bpr_adagrad", n_neg=2, void_anchors=3)


@pytest.mark.parametrize("loss", ["bpr", "warp"])
def test_empty_negatives_and_empty_batch_are_no_ops(dev, loss):
    gen = torch.Generator(device=dev).manual_seed(3)
    A, Cc = _table(50, 13, 0.5, gen, dev), _table(50, 13, 0.5, gen, dev)
    A0, C0 = A.t.clone(), Cc.t.clone()
    fn = native.mf_bpr_fused if loss == "bpr" else native.mf_warp_fused
    stats = torch.zeros(4, device=dev)
    ids = torch.arange(10, dtype=torch.int32, device=dev)
    fn(ids, ids, torch.ones(10, device=dev), A.t, native.local_table(Cc.t, 13), 0.1, 0.01,
       negatives=torch.empty(10, 0, dtype=torch.int32, device=dev), stats=stats)
    e = torch.empty(0, dtype=torch.int32, device=dev)
    fn(e, e, torch.empty(0, device=dev), A.t, native.local_table(Cc.t, 13), 0.1, 0.01,
       negatives=torch.empty(0, 2, dtype=torch.int32, device=dev), stats=stats)
    torch.cuda.synchronize()
    A.check_guards()
    Cc.check_guards()
    assert torch.equal(A.t, A0) and torch.equal(Cc.t, C0)
    assert not stats.any()


# ---- push_tab ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("loss,form", [("bpr", "int32"), ("bpr", "int64"), ("warp", "int32"), ("warp", "packed64")])
def test_push_tab_receives_the_candidate_deltas(dev, loss, form):
    """The candidate table stays bitwise unchanged, the push table receives exactly the replayed candidate deltas,
    and the anchor row is updated in place."""
    if loss == "bpr":
        _bpr(dev, 61, form, n_neg=3, reg=0.01, push=True)
    else:
        _warp(dev, 61, form, 2, push=True)
