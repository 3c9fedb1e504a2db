"""WARP matrix factorisation on the device: ``fps_mf_warp`` against a torch fp32 oracle of ``warp_delta``, where its
candidates come from, its independence of the trial block, what it leaves alone, the quality it reaches and the
public entry points."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests import bpr_quality as Q
from tests import philox_ref
from tests import warp_quality as W

pytestmark = pytest.mark.gpu


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _warp_reference(U, V, users, items, cand, live, margin, lr, reg, N):
    """fp32 torch oracle of ``warp_delta`` for a batch whose anchors, positives and candidates are all distinct:
    ``cand`` [b, T] row indices of V, ``live`` [b, T] which of them count.  Returns the new tables and the stats."""
    u, vi, vj = U[users], V[items], V[cand.clamp(min=0)]
    x = (u[:, None, :] * (vi[:, None, :] - vj)).sum(-1)
    viol = live & (x < margin)
    has = viol.any(1)
    first = viol.float().argmax(1)                                   # the first violator
    n_at = live.to(torch.int64).cumsum(1).gather(1, first[:, None])[:, 0]
    n = torch.where(has, n_at, live.sum(1))
    L = torch.log(torch.clamp((N - 1) // n.clamp(min=1), min=1).double()).float()
    rows = torch.arange(users.numel(), device=U.device)[has]
    g = (lr * L[rows])[:, None]
    xs, js = x[rows, first[rows]], cand[rows, first[rows]]
    uu, vvi, vvj = u[rows], vi[rows], vj[rows, first[rows]]
    U2 = U.clone().index_add_(0, users[rows], g * (vvi - vvj) - lr * reg * uu)
    V2 = V.clone().index_add_(0, items[rows], g * uu - lr * reg * vvi).index_add_(0, js, -g * uu - lr * reg * vvj)
    stats = torch.tensor([float((L[rows] * (margin - xs)).sum()), float(has.sum()), float(n.sum()),
                          float(users.numel())])
    return U2, V2, stats


def _conflict_free(dev, nu, ni, b, T, seed=0):
    g = torch.Generator().manual_seed(seed)
    users = torch.randperm(nu, generator=g)[:b].to(dev)
    ids = torch.randperm(ni, generator=g)[:b * (1 + T)].to(dev)
    items, cand = ids[:b], ids[b:].view(b, T).clone()
    void = torch.rand(b, T, generator=g).to(dev) < 0.15
    cand[void] = -1
    same = torch.rand(b, T, generator=g).to(dev) < 0.1               # a candidate equal to its positive is void
    cand = torch.where(same & ~void, items[:, None].expand(-1, T), cand)
    live = (cand >= 0) & (cand != items[:, None])
    return users, items, cand, live


def _check_stats(got, want):
    got = got.cpu()
    assert got[1].item() == want[1].item() and got[2].item() == want[2].item() and got[3].item() == want[3].item()
    assert abs(got[0].item() - want[0].item()) <= 1e-4 * abs(want[0].item()) + 1e-3


@pytest.mark.parametrize("fmt", ["int32", "int64", "packed64"])
@pytest.mark.parametrize("k", [10, 64, 128, 300, 512])
def test_warp_conflict_free_matches_reference(dev, k, fmt):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, b, T, lr, reg, margin = 3000, 12000, 1500, 6, 0.05, 0.01, -1.0
    m = DeviceOnlineMF(nu, ni, k, range_min=-0.5, range_max=0.5, learning_rate=lr, seed=5, loss="warp",
                       regularization=reg, margin=margin)
    U = m.users[:, :k].clone(); V = m.items.local[:, :k].clone()
    users, items, cand, live = _conflict_free(dev, nu, ni, b, T)
    ratings = torch.ones(b, device=dev)
    ratings[::7] = 0.0                                                 # not positives: skipped whole
    if fmt == "packed64":
        m.step(native.pack_ratings(users, items, ratings), negatives=cand.int().contiguous())
    else:
        idt = torch.int32 if fmt == "int32" else torch.int64
        m.step(users.to(idt), items.to(idt), ratings, negatives=cand.to(idt).contiguous())
    torch.cuda.synchronize()
    pos = ratings > 0
    U2, V2, want = _warp_reference(U, V, users[pos], items[pos], cand[pos], live[pos], margin, lr, reg, ni)
    torch.testing.assert_close(m.users[:, :k], U2, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(m.items.local[:, :k], V2, rtol=1e-5, atol=1e-5)
    assert 0 < want[1] < pos.sum()                                     # some positives update, some do not
    _check_stats(m.stats, want)
    m.check_finite()
    m.close()


@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
@pytest.mark.parametrize("cand_div", [3, 4])
def test_warp_learner_orientation_matches_reference(dev, cand_div, idt):
    """Anchors (users) read from and pushed to a PS ``ShardTable``, candidates (items) in a worker-local table at
    slot ``item // cand_div``, ``rank_items`` the global item count."""
    from fps_b200.store.sharded_table import ShardedTable

    nu, n_slots, k, b, T, lr, reg, margin, N = 5000, 9000, 64, 1000, 5, 0.05, 0.01, -0.5, 40000
    users_tab = ShardedTable(nu, k, init="uniform", init_range=(-0.5, 0.5), seed=11)
    items = torch.rand((n_slots, users_tab.stride), device=dev) - 0.5
    items[:, k:] = 0
    U = users_tab.local[:nu, :k].clone(); V = items[:, :k].clone()
    users, slots, cslots, live = _conflict_free(dev, nu, n_slots, b, T, seed=3)
    ids = slots * cand_div + 1                                         # the ids this worker owns
    cids = torch.where(cslots >= 0, cslots * cand_div + 1, cslots)
    stats = torch.zeros(4, device=dev)
    native.mf_warp_fused(users.to(idt), ids.to(idt), torch.ones(b, device=dev), users_tab.table_c, items, lr, reg,
                         margin=margin, rank_items=N, negatives=cids.to(idt).contiguous(), cand_div=cand_div,
                         stats=stats)
    torch.cuda.synchronize()
    U2, V2, want = _warp_reference(U, V, users, slots, cslots, live, margin, lr, reg, N)
    torch.testing.assert_close(users_tab.local[:nu, :k], U2, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(items[:, :k], V2, rtol=1e-5, atol=1e-5)
    _check_stats(stats, want)
    users_tab.close()


def _bpr_negative0(pos, items, num_items, step, seed):
    """BPR's negative 0 of record ``pos`` (the K5 key (pos, 1, step, seed)), replayed with tests/philox_ref.py."""
    return philox_ref.k5_negative(pos, 1, items, num_items, step, seed)[0]


def test_sampled_candidates_are_bprs_negatives(dev):
    """A huge margin: every positive stops at its first candidate, BPR's negative 0, and updates it."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, b, T, seed = 4000, 50000, 2000, 5, 77
    m = DeviceOnlineMF(nu, ni, 32, range_min=-0.5, range_max=0.5, learning_rate=0.05, negative_sample_rate=T,
                       seed=seed, loss="warp", margin=1e30)
    V0 = m.items.local[:ni].clone()
    g = torch.Generator().manual_seed(1)
    users = torch.randperm(nu, generator=g)[:b].int().to(dev)
    items = torch.randint(0, ni, (b,), generator=g).int().to(dev)
    m.step(users, items, torch.ones(b, device=dev))                  # step 0
    torch.cuda.synchronize()
    s = m.stats.cpu()
    assert s[1].item() == b and s[2].item() == b and s[3].item() == b
    neg0 = _bpr_negative0(np.arange(b), items.cpu().numpy(), ni, 0, seed)
    assert not np.any(neg0 == items.cpu().numpy())
    want = np.zeros(ni, dtype=bool)
    want[items.cpu().numpy()] = True
    want[neg0] = True
    changed = (m.items.local[:ni] != V0).any(1).cpu().numpy()
    assert np.array_equal(changed, want)
    m.close()


def test_no_violator_writes_nothing(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, b, T = 4000, 50000, 2000, 7
    m = DeviceOnlineMF(nu, ni, 64, range_min=-0.5, range_max=0.5, learning_rate=0.05, negative_sample_rate=T,
                       seed=3, loss="warp", regularization=0.1, margin=-1e30)
    U0, V0 = m.users.clone(), m.items.local.clone()
    g = torch.Generator().manual_seed(2)
    users = torch.randint(0, nu, (b,), generator=g).int().to(dev)
    items = torch.randint(0, ni, (b,), generator=g).int().to(dev)
    m.step(users, items, torch.ones(b, device=dev))
    torch.cuda.synchronize()
    assert torch.equal(m.users, U0) and torch.equal(m.items.local, V0)
    s = m.stats.cpu()
    assert s[0].item() == 0 and s[1].item() == 0 and s[2].item() == T * b and s[3].item() == b
    m.close()


@pytest.mark.parametrize("k", [16, 64, 256, 512])
@pytest.mark.parametrize("margin", [-1.0, 0.5])
def test_tables_are_bitwise_independent_of_the_trial_block(dev, k, margin):
    from fps_b200.store.sharded_table import ShardedTable

    nu, ni, b, T = 3000, 20000, 1500, 10
    users, items, cand, _ = _conflict_free(dev, nu, ni, b, T, seed=9)
    g = torch.Generator().manual_seed(4)
    U0 = (torch.rand((nu, (k + 3) // 4 * 4), generator=g) - 0.5).to(dev)
    V0 = (torch.rand((ni, U0.shape[1]), generator=g) - 0.5).to(dev)
    out = []
    for tb in (0,) + native.WARP_TRIAL_BLOCKS:
        Ut, Vt, st = U0.clone(), V0.clone(), torch.zeros(4, device=dev)
        native.mf_warp_fused(users.int(), items.int(), torch.ones(b, device=dev), Ut, Vt, 0.05, 0.01,
                             margin=margin, negatives=cand.int().contiguous(), num_items=ni, stats=st,
                             trial_block=tb)
        torch.cuda.synchronize()
        out.append((tb, Ut, Vt, st))
    for tb, Ut, Vt, st in out[1:]:
        assert torch.equal(Ut, out[0][1]) and torch.equal(Vt, out[0][2]), tb
        assert torch.equal(st[1:], out[0][3][1:]), tb
    assert not torch.equal(out[0][1], U0)


def test_rows_outside_the_batch_stay_bitwise(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, b = 3000, 5000, 1000
    m = DeviceOnlineMF(nu, ni, 64, learning_rate=0.05, seed=2, loss="warp", regularization=0.1, margin=0.0,
                       range_min=-0.5, range_max=0.5)
    U0, V0 = m.users.clone(), m.items.local.clone()
    g = torch.Generator().manual_seed(4)
    users = torch.randint(0, nu // 2, (b,), generator=g).to(dev)
    items = torch.randint(0, ni // 2, (b,), generator=g).to(dev)
    negs = torch.randint(0, ni // 2, (b, 3), generator=g).to(dev)
    negs[::3, 1] = -1
    ratings = torch.ones(b, device=dev)
    ratings[1::4] = 0.0
    m.step(users, items, ratings, negatives=negs)
    torch.cuda.synchronize()
    live = ratings > 0
    touched_u = torch.zeros(nu, dtype=torch.bool, device=dev); touched_u[users[live]] = True
    touched_i = torch.zeros(ni, dtype=torch.bool, device=dev); touched_i[items[live]] = True
    n = negs[live]
    touched_i[n[n >= 0]] = True
    assert torch.equal(m.users[~touched_u], U0[~touched_u])
    assert torch.equal(m.items.local[:ni][~touched_i], V0[:ni][~touched_i])
    assert not torch.equal(m.users[touched_u], U0[touched_u])
    assert m.stats[3].item() == int(live.sum())
    m.close()


def test_same_seed_models_end_bitwise_equal(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    out = []
    for _ in range(2):
        m = DeviceOnlineMF(64, 1000, 64, learning_rate=0.05, negative_sample_rate=5, seed=3, loss="warp",
                           regularization=0.01, range_min=-0.3, range_max=0.3, margin=0.5)
        g = torch.Generator().manual_seed(9)
        for _ in range(40):                # one positive per step: its pushes land in program order
            u = torch.randint(0, 64, (1,), generator=g, dtype=torch.int32).to(dev)
            i = torch.randint(0, 1000, (1,), generator=g, dtype=torch.int32).to(dev)
            m.step(u, i, torch.ones(1, device=dev))
        torch.cuda.synchronize()
        out.append((m.users.clone(), m.items.local.clone(), m.stats.clone()))
        m.close()
    for a, b in zip(*out):
        assert torch.equal(a, b)
    assert out[0][2][1].item() > 0


def test_warp_rejects_unsupported_steps(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    m = DeviceOnlineMF(16, 16, 8, loss="warp")
    u = torch.arange(4, device=dev, dtype=torch.int32)
    with pytest.raises(ValueError, match="negative_sample_rate"):
        m.step(u, u, torch.ones(4, device=dev))
    m.close()
    m = DeviceOnlineMF(16, 16, 8, loss="warp", item_cache=True)
    with pytest.raises(ValueError, match="replica"):
        m.step(u, u, torch.ones(4, device=dev), negatives=u[:, None].contiguous())
    m.close()


def test_warp_quality_gate(dev):
    """Same data, epochs and rate as the sequential numpy run of tests/test_mf_warp_host.py."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    tu, ti, eu, ei = Q.data()
    m = DeviceOnlineMF(Q.NUM_USERS, Q.NUM_ITEMS, Q.K, range_min=-Q.INIT, range_max=Q.INIT, learning_rate=W.LR,
                       negative_sample_rate=W.T, seed=1, loss="warp", regularization=Q.REG, margin=W.MARGIN)
    du, di = tu.int().to(dev), ti.int().to(dev)
    ones = torch.ones(du.numel(), device=dev)
    for _ in range(Q.EPOCHS):
        for a in range(0, du.numel(), 128):
            m.step(du[a:a + 128], di[a:a + 128], ones[a:a + 128])
    torch.cuda.synchronize()
    m.check_finite()
    auc, recall = Q.metrics(m.users[:, :Q.K], m.items.local[:Q.NUM_ITEMS, :Q.K], (tu, ti), (eu, ei))
    assert auc >= W.AUC_GATE and recall >= W.RECALL_GATE, (auc, recall)
    s = m.stats.cpu()
    assert s[2].item() > s[3].item()                  # trained: positives examine more than one candidate on average
    m.close()


def test_ps_online_mf_device_warp_returns_vectors(dev):
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.online import psOnlineMF

    tu, ti, _, _ = Q.data()
    recs = [Rating(int(u), int(i), 1.0) for u, i in zip(tu[:2000], ti[:2000])]

    def run(lr):
        return psOnlineMF(recs, numFactors=8, learningRate=lr, negativeSampleRate=5, backend="device",
                          loss="warp", margin=0.5, regularization=0.01, seed=1).collect()

    res, frozen = run(0.02), run(0.0)
    users = {r.value[0]: r.value[1] for r in res if r.is_left}
    items = {r.value[0]: r.value[1] for r in res if r.is_right}
    assert len(users) == len(set(tu[:2000].tolist())) and len(items) == 1 + int(ti[:2000].max())
    assert all(len(v) == 8 and all(abs(x) < 10 for x in v) for v in list(users.values()) + list(items.values()))
    users0 = {r.value[0]: r.value[1] for r in frozen if r.is_left}
    assert any((users[u] != users0[u]).any() for u in users)


def test_learner_and_generator_warp_beats_an_untrained_model(dev):
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator

    tu, ti, _, _ = Q.data()
    recs = [Rating(int(u), int(i), 1.0, t) for t, (u, i) in enumerate(zip(tu.tolist(), ti.tolist()))]

    def hit_rate(lr):
        out = psOnlineLearnerAndGenerator(recs, numFactors=16, rangeMin=-0.1, rangeMax=0.1, learningRate=lr,
                                          negativeSampleRate=10, K=20, backend="device", loss="warp",
                                          batch_size=256, seed=1)
        second = out[len(out) // 2:]
        return sum(item in {i for _, i in top} for _, item, _, top in second) / len(second)

    trained, frozen = hit_rate(0.05), hit_rate(0.0)
    assert trained > frozen + 0.01, (trained, frozen)


@pytest.mark.timeout(900)                  # torchrun children: their own 420 s limit applies first
def test_multi_rank_warp():
    from tests.test_gpu_multi import _run

    _run("mp_warp_check.py", 2, 29645, "MP_WARP_CHECK_OK")
