"""Pairwise (BPR) matrix factorisation on the device: ``fps_mf_bpr`` against a torch fp32 oracle, where its
negatives come from, what it leaves alone, the quality it reaches and the public entry points."""
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests import bpr_quality as Q

pytestmark = pytest.mark.gpu


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _bpr_reference(U, V, users, items, negs, lr, reg):
    u, vi, vj = U[users], V[items], V[negs]
    x = (u * (vi - vj)).sum(1)
    g = (lr * torch.sigmoid(-x))[:, None]
    U2 = U.clone().index_add_(0, users, g * (vi - vj) - lr * reg * u)
    V2 = V.clone().index_add_(0, items, g * u - lr * reg * vi).index_add_(0, negs, -g * u - lr * reg * vj)
    return U2, V2, torch.nn.functional.softplus(-x).sum(), int((x > 0).sum())


@pytest.mark.parametrize("reg", [0.0, 0.01])
@pytest.mark.parametrize("fmt", ["int32", "int64", "packed64"])
@pytest.mark.parametrize("k", [10, 64, 128, 300])
def test_bpr_conflict_free_matches_reference(dev, k, fmt, reg):
    """Distinct users and distinct i / j => every delta is computed from the initial rows: the kernel must
    equal fp32 torch, stats included."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, b, lr = 6000, 9000, 4000, 0.05
    m = DeviceOnlineMF(nu, ni, k, range_min=-0.5, range_max=0.5, learning_rate=lr, seed=5, loss="bpr",
                       regularization=reg)
    U = m.users[:, :k].clone(); V = m.items.local[:, :k].clone()
    users = torch.randperm(nu, device=dev)[:b]
    ij = torch.randperm(ni, device=dev)[:2 * b]
    items, negs = ij[:b], ij[b:]
    ratings = torch.rand(b, device=dev) + 0.5
    if fmt == "packed64":
        ratings = torch.ones(b, device=dev)
        m.step(native.pack_ratings(users, items, ratings), negatives=negs.int()[:, None].contiguous())
    else:
        idt = torch.int32 if fmt == "int32" else torch.int64
        m.step(users.to(idt), items.to(idt), ratings, negatives=negs.to(idt)[:, None].contiguous())
    torch.cuda.synchronize()
    U2, V2, loss, n_ok = _bpr_reference(U, V, users, items, negs, lr, reg)
    torch.testing.assert_close(m.users[:, :k], U2, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m.items.local[:, :k], V2, rtol=1e-5, atol=1e-6)
    s = m.stats.cpu()
    assert s[1].item() == b
    assert abs(s[0].item() - loss.item()) / loss.item() < 1e-4
    assert abs(s[2].item() - n_ok) <= 1
    m.check_finite()
    m.close()


@pytest.mark.parametrize("reg", [0.0, 0.01])
@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
@pytest.mark.parametrize("cand_div", [3, 4])
def test_bpr_learner_orientation_matches_reference(dev, cand_div, idt, reg):
    """The online learner's orientation: anchors (users) read from and pushed to a PS ``ShardTable``,
    candidates (items) in a worker-local table at slot ``item // cand_div``.  Conflict-free batch."""
    from fps_b200.store.sharded_table import ShardedTable

    nu, n_slots, k, b, lr = 5000, 7000, 64, 2000, 0.05
    users_tab = ShardedTable(nu, k, init="uniform", init_range=(-0.5, 0.5), seed=11)
    items = torch.rand((n_slots, users_tab.stride), device=dev) - 0.5
    items[:, k:] = 0
    U = users_tab.local[:nu, :k].clone(); V = items[:, :k].clone()
    users = torch.randperm(nu, device=dev)[:b]
    slots = torch.randperm(n_slots, device=dev)[:2 * b]
    ids = slots * cand_div + 1                      # the ids this worker owns: item % cand_div == 1
    ratings = torch.rand(b, device=dev) + 0.5
    stats = torch.zeros(3, device=dev)
    native.mf_bpr_fused(users.to(idt), ids[:b].to(idt).contiguous(), ratings, users_tab.table_c, items, lr, reg,
                        negatives=ids[b:].to(idt)[:, None].contiguous(), cand_div=cand_div, stats=stats)
    torch.cuda.synchronize()
    U2, V2, loss, n_ok = _bpr_reference(U, V, users, slots[:b], slots[b:], lr, reg)
    torch.testing.assert_close(users_tab.local[:nu, :k], U2, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(items[:, :k], V2, rtol=1e-5, atol=1e-6)
    assert stats[1].item() == b
    assert abs(stats[0].item() - loss.item()) / loss.item() < 1e-4
    assert abs(stats[2].item() - n_ok) <= 1
    users_tab.close()


def _onehot_model(num_users, num_items, k, n_neg, seed=0, **kw):
    """A BPR model whose user rows are 0 and whose item rows are one-hot: a user's delta after one step is
    (lr / 2) * (n_live * e_i - sum_j e_j), so it spells out the negatives its positive was paired with
    (u = 0 gives x = 0, g = lr / 2, and leaves the item rows unchanged)."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    m = DeviceOnlineMF(num_users, num_items, k, learning_rate=0.5, negative_sample_rate=n_neg, seed=seed,
                       loss="bpr", **kw)
    return m


def _reset_onehot(m, num_items):
    m.users.zero_()
    m.items.local.zero_()
    m.items.local[:num_items, :num_items] = torch.eye(num_items, device=m.items.local.device)


def test_sampled_negatives_two_items_always_the_other(dev):
    n = 4096
    m = _onehot_model(n, 2, 4, n_neg=3)
    _reset_onehot(m, 2)
    users = torch.arange(n, device=dev, dtype=torch.int32)
    items = users % 2
    m.step(users, items, torch.ones(n, device=dev))
    torch.cuda.synchronize()
    want = torch.zeros(n, 4, device=dev)
    want[torch.arange(n), items.long()] = 0.75
    want[torch.arange(n), 1 - items.long()] = -0.75
    assert torch.equal(m.users, want)
    assert m.stats[1].item() == 3 * n
    m.close()


def test_sampled_negatives_spread_and_depend_on_the_seed(dev):
    n, ni, n_neg = 4096, 64, 3
    rows = []
    for seed in (1, 1, 2):
        m = _onehot_model(n, ni, ni, n_neg, seed=seed)
        _reset_onehot(m, ni)
        users = torch.arange(n, device=dev, dtype=torch.int32)
        items = users % ni
        m.step(users, items, torch.ones(n, device=dev))
        torch.cuda.synchronize()
        rows.append(m.users.clone())
        m.close()
    assert torch.equal(rows[0], rows[1])
    assert not torch.equal(rows[0], rows[2])
    r = rows[0]
    pos = (torch.arange(n, device=dev) % ni).long()
    assert torch.all(r[torch.arange(n), pos] == 0.25 * n_neg)           # no negative equals the positive
    counts = (-r / 0.25).round()
    counts[torch.arange(n), pos] = 0
    assert torch.all(counts >= 0) and torch.all(counts.sum(1) == n_neg)
    per_item = counts.sum(0)                                            # ~ uniform over the other items
    assert per_item.min() > 0.5 * per_item.mean() and per_item.max() < 1.5 * per_item.mean()


def test_user_memory_negatives_are_the_unseen_item_or_void(dev):
    M, n_users, n_neg = 8, 64, 4
    m = _onehot_model(n_users, M + 1, 16, n_neg, user_memory=M)
    users = torch.arange(n_users, device=dev, dtype=torch.int32)
    for t in range(M):                     # every user consumes items 0 .. M-1, one per step, in order
        m.step(users, torch.full_like(users, t), torch.ones(n_users, device=dev))
    _reset_onehot(m, M + 1)
    m.step(users, torch.zeros_like(users), torch.ones(n_users, device=dev))
    torch.cuda.synchronize()
    r = m.users[:, : M + 1]
    assert torch.all(r[:, 1:M] == 0)                 # never a seen item
    assert torch.equal(r[:, 0], -r[:, M])            # every live negative is item M
    assert r[:, 0].sum() > 0
    m.close()


def test_same_seed_models_end_bitwise_equal(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    out = []
    for _ in range(2):
        m = DeviceOnlineMF(64, 1000, 64, learning_rate=0.1, negative_sample_rate=3, seed=3, loss="bpr",
                           regularization=0.01, range_min=-0.3, range_max=0.3)
        g = torch.Generator().manual_seed(9)
        for _ in range(40):                # one positive per step: its triples are pushed in program order
            u = torch.randint(0, 64, (1,), generator=g, dtype=torch.int32).to(dev)
            i = torch.randint(0, 1000, (1,), generator=g, dtype=torch.int32).to(dev)
            m.step(u, i, torch.ones(1, device=dev))
        torch.cuda.synchronize()
        out.append((m.users.clone(), m.items.local.clone(), m.stats.clone()))
        m.close()
    for a, b in zip(*out):
        assert torch.equal(a, b)


def test_rows_outside_the_batch_stay_bitwise(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, b = 3000, 5000, 1000
    m = DeviceOnlineMF(nu, ni, 64, learning_rate=0.05, seed=2, loss="bpr", regularization=0.1,
                       range_min=-0.5, range_max=0.5)
    U0, V0 = m.users.clone(), m.items.local.clone()
    g = torch.Generator().manual_seed(4)
    users = torch.randint(0, nu // 2, (b,), generator=g).to(dev)
    items = torch.randint(0, ni // 2, (b,), generator=g).to(dev)
    negs = torch.randint(0, ni // 2, (b, 2), generator=g).to(dev)
    negs[::3, 1] = -1                                         # voided triples
    ratings = torch.ones(b, device=dev)
    ratings[1::4] = 0.0                                       # not positives: skipped whole
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
    # a negative equal to its positive is void as well
    assert m.stats[1].item() == int(((n >= 0) & (n != items[live][:, None])).sum())
    m.close()


def test_bpr_rejects_unsupported_combinations(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    m = DeviceOnlineMF(16, 16, 8, loss="bpr")
    u = torch.arange(4, device=dev, dtype=torch.int32)
    with pytest.raises(ValueError, match="negative_sample_rate"):
        m.step(u, u, torch.ones(4, device=dev))
    m.close()
    m = DeviceOnlineMF(16, 16, 8)
    with pytest.raises(ValueError, match="loss='bpr'"):
        m.step(u, u, torch.ones(4, device=dev), negatives=u[:, None].contiguous())
    m.close()
    m = DeviceOnlineMF(16, 16, 8, loss="bpr", item_cache=True)
    with pytest.raises(ValueError, match="replica"):
        m.step(u, u, torch.ones(4, device=dev), negatives=u[:, None].contiguous())
    m.close()


def test_bpr_quality_gate(dev):
    """Same data, same update budget as the sequential numpy run of tests/test_mf_bpr_host.py."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    tu, ti, eu, ei = Q.data()
    m = DeviceOnlineMF(Q.NUM_USERS, Q.NUM_ITEMS, Q.K, range_min=-Q.INIT, range_max=Q.INIT, learning_rate=Q.LR,
                       negative_sample_rate=1, seed=1, loss="bpr", regularization=Q.REG)
    du, di = tu.int().to(dev), ti.int().to(dev)
    ones = torch.ones(du.numel(), device=dev)
    for _ in range(Q.EPOCHS):
        for a in range(0, du.numel(), 128):
            m.step(du[a:a + 128], di[a:a + 128], ones[a:a + 128])
    torch.cuda.synchronize()
    m.check_finite()
    auc, recall = Q.metrics(m.users[:, :Q.K], m.items.local[:Q.NUM_ITEMS, :Q.K], (tu, ti), (eu, ei))
    assert auc >= Q.AUC_GATE and recall >= Q.RECALL_GATE, (auc, recall)
    m.close()


def test_ps_online_mf_device_bpr_returns_vectors(dev):
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.online import psOnlineMF

    tu, ti, _, _ = Q.data()
    recs = [Rating(int(u), int(i), 1.0) for u, i in zip(tu[:2000], ti[:2000])]
    def run(lr):
        return psOnlineMF(recs, numFactors=8, learningRate=lr, negativeSampleRate=2, backend="device",
                          loss="bpr", regularization=0.01, seed=1).collect()

    res, frozen = run(0.05), run(0.0)
    users = {r.value[0]: r.value[1] for r in res if r.is_left}
    items = {r.value[0]: r.value[1] for r in res if r.is_right}
    assert len(users) == len(set(tu[:2000].tolist())) and len(items) == 1 + int(ti[:2000].max())
    assert all(len(v) == 8 and all(abs(x) < 10 for x in v) for v in list(users.values()) + list(items.values()))
    users0 = {r.value[0]: r.value[1] for r in frozen if r.is_left}
    assert any((users[u] != users0[u]).any() for u in users)       # the BPR steps moved the vectors


def test_learner_and_generator_bpr_beats_an_untrained_model(dev):
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator

    tu, ti, _, _ = Q.data()
    recs = [Rating(int(u), int(i), 1.0, t) for t, (u, i) in enumerate(zip(tu.tolist(), ti.tolist()))]

    def hit_rate(lr):
        out = psOnlineLearnerAndGenerator(recs, numFactors=16, rangeMin=-0.1, rangeMax=0.1, learningRate=lr,
                                          negativeSampleRate=4, K=20, backend="device", loss="bpr",
                                          batch_size=256, seed=1)
        second = out[len(out) // 2:]
        return sum(item in {i for _, i in top} for _, item, _, top in second) / len(second)

    trained, frozen = hit_rate(0.2), hit_rate(0.0)
    assert trained > frozen + 0.01, (trained, frozen)


@pytest.mark.timeout(900)                  # torchrun children: their own 420 s limit applies first
def test_multi_rank_bpr():
    from tests.test_gpu_multi import _run

    _run("mp_bpr_check.py", 2, 29635, "MP_BPR_CHECK_OK")
