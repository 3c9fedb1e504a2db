"""Numerics of the hand-written sm_90a kernels vs plain PyTorch fp32 references."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def test_native_library_loaded(dev):
    from fps_b200.ops import native

    assert native.available(), "libfps_kernels.so must be built in-tree"
    native.lib()
    maps = open("/proc/self/maps").read()
    assert "libfps_kernels.so" in maps


@pytest.mark.parametrize("dim", [10, 16, 64, 300])
def test_init_rows_matches_philox_oracle(dev, dim):
    from fps_b200.store.sharded_table import ShardedTable
    from tests.philox_ref import init_rows_ref

    t = ShardedTable(1000, dim, seed=42, init_range=(-0.01, 0.01))
    ids = t.local_ids().cpu().numpy()
    ref = init_rows_ref(ids, dim, 42, -0.01, 0.01)
    got = t.local.cpu().numpy()
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-9)
    assert (got[:, dim:] == 0).all()
    t.close()


@pytest.mark.parametrize("dim,idt", [(10, torch.int64), (64, torch.int32), (128, torch.int64), (300, torch.int32)])
def test_pull_push_dot(dev, dim, idt):
    from fps_b200.store.sharded_table import ShardedTable

    n = 5000
    t = ShardedTable(n, dim, seed=3, init_range=(-1.0, 1.0), track_touched=True)
    table0 = t.local[:, :dim].clone()
    ids = torch.randint(0, n, (20000,), device=dev).to(idt)
    got = t.pull(ids)
    torch.testing.assert_close(got, table0[ids.long()], rtol=0, atol=0)
    delta = torch.randn(ids.numel(), dim, device=dev)
    t.push(ids, delta)
    ref = table0.clone().index_add_(0, ids.long(), delta)
    torch.testing.assert_close(t.local[:, :dim], ref, rtol=1e-5, atol=1e-5)
    loc = torch.randn(ids.numel(), dim, device=dev)
    s = t.pull_dot(ids, loc)
    torch.testing.assert_close(s, (ref[ids.long()] * loc).sum(1), rtol=1e-4, atol=1e-4)
    # touched bitmap == set of pulled ids
    dumped_ids, dumped = t.dump_local()
    assert set(dumped_ids.tolist()) == set(ids.long().unique().tolist())
    t.check_finite()
    t.push(ids[:1], torch.full((1, dim), float("nan"), device=dev))
    with pytest.raises(FloatingPointError):
        t.check_finite()
    t.close()


def _mf_reference(U, V, users, items, ratings, lr, err_mode):
    u = U[users]; v = V[items]
    resid = ratings - (u * v).sum(1)
    e = torch.sigmoid(resid) if err_mode == 0 else resid
    g = (lr * e)[:, None]
    U2 = U.clone().index_add_(0, users, g * v)
    V2 = V.clone().index_add_(0, items, g * u)
    return U2, V2, (resid ** 2).sum()


@pytest.mark.parametrize("kernel", ["tma", "reg"])
@pytest.mark.parametrize("k,idt,err_mode", [(64, torch.int32, 0), (64, torch.int64, 1), (10, torch.int32, 0),
                                            (16, torch.int32, 1), (128, torch.int64, 0), (300, torch.int32, 0),
                                            (4, torch.int32, 1), (1000, torch.int32, 0)])
def test_mf_sgd_fused_matches_reference(dev, k, idt, err_mode, kernel):
    """Unique (user, item) per batch => the async kernel is deterministic and must equal fp32 torch."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, b = 6000, 5000, 4000
    m = DeviceOnlineMF(nu, ni, k, range_min=-0.5, range_max=0.5, learning_rate=0.05, seed=5, err_mode=err_mode,
                       kernel=kernel)
    if k >= 1000:
        m.items.local.mul_(0.05); m.users.mul_(0.05)   # keep |u.v| moderate for the fp32 comparison
    U = m.users[:, :k].clone(); V = m.items.local[:, :k].clone()
    users = torch.randperm(nu, device=dev)[:b]
    items = torch.randperm(ni, device=dev)[:b]
    ratings = torch.rand(b, device=dev) * 2
    m.step(users.to(idt), items.to(idt), ratings)
    torch.cuda.synchronize()
    U2, V2, sq = _mf_reference(U, V, users, items, ratings, 0.05, err_mode)
    torch.testing.assert_close(m.users[:, :k], U2, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m.items.local[:, :k], V2, rtol=1e-5, atol=1e-6)
    s = m.stats.cpu()
    assert s[1].item() == b
    assert abs(s[0].item() - sq.item()) / sq.item() < 1e-4
    m.check_finite()
    m.close()


@pytest.mark.parametrize("kernel", ["tma", "reg"])
def test_mf_sgd_fused_duplicates_lose_no_update(dev, kernel):
    """Hot rows hammered by every lane-group: nothing corrupt, every update counted."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    k = 64
    m = DeviceOnlineMF(8, 4, k, range_min=0.1, range_max=0.2, learning_rate=0.0, seed=1, err_mode=1,
                       kernel=kernel)
    U = m.users[:, :k].clone(); V = m.items.local[:, :k].clone()
    users = torch.randint(0, 8, (10000,), device=dev, dtype=torch.int32)
    items = torch.randint(0, 4, (10000,), device=dev, dtype=torch.int32)
    m.step(users, items, torch.ones(10000, device=dev))
    torch.cuda.synchronize()
    torch.testing.assert_close(m.users[:, :k], U)  # lr = 0 -> nothing moves, nothing corrupt
    torch.testing.assert_close(m.items.local[:, :k], V)
    assert m.stats[1].item() == 10000
    m.close()


def test_mf_converges_rmse_gate(dev):
    """Model-quality gate mirroring PSOfflineMatrixFactorizationTest.scala:55-103 (RMSE <= 0.5)."""
    from fps_b200.models.mf.device import DeviceOnlineMF, ERR_PLAIN

    g = torch.Generator().manual_seed(47)
    nu, ni, k = 20, 15, 15
    users = torch.randint(0, nu, (100,), generator=g, dtype=torch.int32).cuda()
    items = torch.randint(0, ni, (100,), generator=g, dtype=torch.int32).cuda()
    ratings = torch.rand(100, generator=g).cuda()
    m = DeviceOnlineMF(nu, ni, k, range_min=0.0, range_max=1.0 / k ** 0.5, learning_rate=0.05, seed=47,
                       err_mode=ERR_PLAIN)
    for _ in range(200):
        m.step(users, items, ratings)
    pred = m.predict(users, items)
    rmse = ((pred - ratings) ** 2).mean().sqrt().item()
    assert rmse <= 0.5, rmse
    m.close()


@pytest.mark.parametrize("kernel", ["tma", "reg"])
def test_mf_negative_sampling_counts(dev, kernel):
    from fps_b200.models.mf.device import DeviceOnlineMF

    m = DeviceOnlineMF(1000, 500, 32, learning_rate=0.01, negative_sample_rate=3, seed=9, kernel=kernel)
    V0 = m.items.local.clone()
    users = torch.randint(0, 1000, (2048,), device=dev, dtype=torch.int32)
    items = torch.randint(0, 500, (2048,), device=dev, dtype=torch.int32)
    m.step(users, items, torch.ones(2048, device=dev))
    torch.cuda.synchronize()
    assert m.stats[1].item() == 2048 * 4
    changed = (m.items.local != V0).any(1).sum().item()
    assert changed > 400  # negatives touch (almost) every item
    m.check_finite()
    m.close()


def test_fit_stream_end_to_end(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    m = DeviceOnlineMF(5000, 3000, 64, learning_rate=0.01, seed=2)
    g = torch.Generator().manual_seed(1)
    batches = []
    for _ in range(7):
        batches.append((torch.randint(0, 5000, (4096,), generator=g, dtype=torch.int32).pin_memory(),
                        torch.randint(0, 3000, (4096,), generator=g, dtype=torch.int32).pin_memory(),
                        torch.rand(4096, generator=g).pin_memory()))
    res = list(m.fit_stream(iter(batches)))
    assert len(res) == 7
    assert all(c == 4096 for _, c in res)
    assert all(np.isfinite(s) for s, _ in res)
    m.close()


def test_packed64_records_equal_array_inputs(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.ops import native

    nu, ni, k, b = 50000, 30000, 64, 20000
    g = torch.Generator().manual_seed(3)
    users = torch.randperm(nu, generator=g)[:b].int()
    items = torch.randperm(ni, generator=g)[:b].int()
    ratings = torch.rand(b, generator=g).half().float()
    m1 = DeviceOnlineMF(nu, ni, k, learning_rate=0.05, seed=5, kernel="reg")
    m2 = DeviceOnlineMF(nu, ni, k, learning_rate=0.05, seed=5, kernel="reg")
    m1.step(users.cuda(), items.cuda(), ratings.cuda())
    m2.step(native.pack_ratings(users, items, ratings).cuda())
    torch.cuda.synchronize()
    assert torch.equal(m1.users, m2.users) and torch.equal(m1.items.local, m2.items.local)
    with pytest.raises(ValueError):
        native.pack_ratings(torch.tensor([1 << 26]), torch.tensor([0]), torch.tensor([1.0]))
    m1.close(); m2.close()


def test_generic_device_tier_batched_worker_logic(dev):
    """A user BatchedWorkerLogic on the device engine: word-count style pull -> push(+1) -> output."""
    from fps_b200.api import BatchedWorkerLogic
    from fps_b200.runtime.device_engine import transform_device
    from fps_b200.store.sharded_table import ShardedTable

    class CountLogic(BatchedWorkerLogic):
        def onRecvBatch(self, batch, ps):
            ps.pull(batch)

        def onPullRecvBatch(self, ids, values, ps):
            ps.output((int(ids.numel()), float(values.sum())))
            ps.push(ids, torch.ones(ids.numel(), 4, device=ids.device))

    table = ShardedTable(1000, 4, init="zeros", track_touched=True)
    batches = [torch.randint(0, 50, (200,), device=dev) for _ in range(6)]
    out = transform_device(batches, CountLogic(), table, pull_limit=64, worker_streams=2)
    counts = torch.bincount(torch.cat(batches), minlength=1000).float()
    model = dict((i, v) for i, v in out.ps_outputs())
    assert set(model) == set(torch.cat(batches).unique().tolist())
    for i, v in model.items():
        assert torch.allclose(v, torch.full((4,), counts[i].item()))
    assert sum(n for n, _ in out.worker_outputs()) == 1200
    assert max(n for n, _ in out.worker_outputs()) <= 64        # pull limiter chunks
    table.close()


def test_ps_online_mf_device_backend_through_reference_api(dev):
    import random

    import numpy as np

    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.offline import psOfflineMF

    r = random.Random(47)
    ratings = [Rating(r.randrange(20), r.randrange(15), r.random()) for _ in range(100)]
    out = psOfflineMF(ratings, numFactors=15, rangeMin=0.0, rangeMax=0.25, learningRate=0.05, iterations=150,
                      backend="device", seed=3, plain_residual=True, batch_size=64)
    users = dict(out.worker_outputs()); items = dict(out.ps_outputs())
    rmse = (sum((x.rating - float(np.dot(users[x.user], items[x.item]))) ** 2 for x in ratings) / len(ratings)) ** 0.5
    assert rmse <= 0.5, rmse
    out.model.close()


def test_cuda_graph_step_replays_fused_kernel(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.ops import native

    nu, ni, k, b = 5000, 3000, 64, 2048
    g = torch.Generator().manual_seed(9)
    m1 = DeviceOnlineMF(nu, ni, k, learning_rate=0.05, seed=5)
    m2 = DeviceOnlineMF(nu, ni, k, learning_rate=0.05, seed=5)
    static, replay = m2.make_graph_step(b, packed=True)
    m2.users.copy_(m1.users); m2.items.local.copy_(m1.items.local)      # undo the warm-up steps
    for _ in range(3):
        u = torch.randperm(nu, generator=g)[:b].int(); i = torch.randperm(ni, generator=g)[:b].int()
        r = torch.rand(b, generator=g).half().float()
        rec = native.pack_ratings(u, i, r).cuda()
        m1.step(rec)
        static[0].copy_(rec); replay()
    torch.cuda.synchronize()
    assert torch.equal(m1.users, m2.users) and torch.equal(m1.items.local, m2.items.local)
    assert m2.stats[1].item() == b
    m1.close(); m2.close()


def test_wide_rows_pull_push(dev):
    """dim > 1024 floats takes the (row, 4 KiB segment) kernel."""
    from fps_b200.store.sharded_table import ShardedTable

    n, dim = 37, 5000
    t = ShardedTable(n, dim, seed=3, init_range=(-1.0, 1.0))
    ref = t.local[:, :dim].clone()
    ids = torch.randint(0, n, (50,), device=dev)
    got = torch.empty((50, t.stride), device=dev)
    from fps_b200.ops import native
    native.pull_gather(t.table_c, ids, got)
    torch.testing.assert_close(got[:, :dim], ref[ids], rtol=0, atol=0)
    delta = torch.randn(50, t.stride, device=dev)
    native.push_add(t.table_c, ids, delta, scale=0.5)
    torch.testing.assert_close(t.local[:, :dim], ref.index_add_(0, ids, 0.5 * delta[:, :dim]), rtol=1e-5, atol=1e-5)
    t.close()


def test_item_cache_mode_single_gpu_matches_direct_mode(dev):
    """Item-cache mode (train a local replica, merge replica-base deltas) must give the direct-mode
    result for a conflict-free batch, and the master must equal the replica after every sync."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, k, b = 6000, 5000, 64, 3000
    m_direct = DeviceOnlineMF(nu, ni, k, range_min=-0.5, range_max=0.5, learning_rate=0.05, seed=5, item_cache=False)
    m_cache = DeviceOnlineMF(nu, ni, k, range_min=-0.5, range_max=0.5, learning_rate=0.05, seed=5, item_cache=True,
                             sync_every=2, replica_own_inplace=False)
    V0 = m_cache.items.local.clone()
    rep = m_cache.replica
    assert torch.equal(rep.cache[:ni], V0[:ni]) and torch.equal(rep.base, rep.cache)
    g = torch.Generator().manual_seed(1)
    for step in range(3):
        users = torch.randperm(nu, generator=g)[:b].int().cuda()
        items = torch.randperm(ni, generator=g)[:b].int().cuda()
        ratings = torch.rand(b, generator=g).cuda()
        m_direct.step(users, items, ratings); m_cache.step(users, items, ratings)
    m_cache.flush()
    torch.cuda.synchronize()
    torch.testing.assert_close(m_cache.users, m_direct.users, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m_cache.items.local, m_direct.items.local, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m_cache.replica.cache[:ni], m_cache.items.local[:ni], rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(m_cache.replica.base, m_cache.replica.cache, rtol=1e-6, atol=1e-7)
    m_direct.close(); m_cache.close()


def test_device_mf_checkpoint_resume(dev, tmp_path):
    from fps_b200.models.mf.device import DeviceOnlineMF

    g = torch.Generator().manual_seed(4)
    u = torch.randint(0, 3000, (8192,), generator=g, dtype=torch.int32).cuda()
    i = torch.randint(0, 2000, (8192,), generator=g, dtype=torch.int32).cuda()
    r = torch.rand(8192, generator=g).cuda()
    m = DeviceOnlineMF(3000, 2000, 32, learning_rate=0.05, seed=1)
    m.step(u, i, r)
    m.save(str(tmp_path))
    m2 = DeviceOnlineMF(3000, 2000, 32, learning_rate=0.05, seed=99)      # different init, then resume
    m2.load(str(tmp_path))
    assert torch.equal(m2.users, m.users) and torch.equal(m2.items.local, m.items.local) and m2.step_no == 1
    m.close(); m2.close()


@pytest.mark.parametrize("packed", [False, True])
def test_negative_sampler_respects_user_memory(dev, packed):
    """K5 contract (PSOnlineMatrixFactorizationWorker.scala:61-78): negatives are never one of the
    user's last `userMemory` items, the ring evicts the oldest item, positives pass through."""
    from fps_b200.ops import native

    n_users, n_items, mem, neg = 64, 48, 8, 3
    seen = torch.full((n_users, mem), -1, dtype=torch.int32, device=dev)
    pos = torch.zeros(n_users, dtype=torch.int32, device=dev)
    g = torch.Generator().manual_seed(5)
    history = {u: [] for u in range(n_users)}
    for step in range(12):
        users = torch.randperm(n_users, generator=g)[:40].to(torch.int32)       # distinct users per batch
        items = torch.randint(0, n_items, (40,), generator=g, dtype=torch.int32)
        ratings = torch.ones(40)
        for u, i in zip(users.tolist(), items.tolist()):
            history[u].append(i)
        if packed:
            rec = native.pack_ratings(users.cuda(), items.cuda(), ratings.cuda())
            ou, oi, orat = native.neg_sample(rec, None, None, neg, n_items, seen, pos, 1, seed=3, step=step)
        else:
            ou, oi, orat = native.neg_sample(users.cuda(), items.cuda(), ratings.cuda(), neg, n_items, seen,
                                             pos, 1, seed=3, step=step)
        ou, oi, orat = ou.cpu().view(40, 1 + neg), oi.cpu().view(40, 1 + neg), orat.cpu().view(40, 1 + neg)
        assert torch.equal(ou[:, 0], users) and torch.equal(oi[:, 0], items) and (orat[:, 0] == 1).all()
        assert (orat[:, 1:] == 0).all()
        for row, u in enumerate(users.tolist()):
            recent = set(history[u][-mem:])
            for j in range(1, 1 + neg):
                if ou[row, j] >= 0:
                    assert ou[row, j] == u and int(oi[row, j]) not in recent
        assert (ou[:, 1:] >= 0).float().mean() > 0.95     # 8 of 48 items excluded: a draw almost always succeeds
    for u in range(n_users):                              # ring content == last `mem` items of the user
        assert sorted(x for x in seen[u].cpu().tolist() if x >= 0) == sorted(history[u][-mem:])
    # a user who has seen everything gets voided negatives, which the fused kernel skips
    seen2 = torch.arange(16, dtype=torch.int32, device=dev).repeat(4, 1).contiguous()
    pos2 = torch.full((4,), 16, dtype=torch.int32, device=dev)
    ou, oi, orat = native.neg_sample(torch.arange(4, dtype=torch.int32, device=dev),
                                     torch.zeros(4, dtype=torch.int32, device=dev), torch.ones(4, device=dev),
                                     2, 16, seen2, pos2, 1)
    assert (ou.view(4, 3)[:, 1:] == -1).all()


def test_device_mf_with_user_memory_skips_voided_records(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    m = DeviceOnlineMF(200, 16, 16, learning_rate=0.05, negative_sample_rate=2, seed=2, user_memory=16)
    users = torch.arange(200, dtype=torch.int32, device=dev)
    for it in range(16):     # after 16 steps every user has all 16 items in memory: no negatives left
        m.stats.zero_()
        m.step(users, torch.full((200,), it, dtype=torch.int32, device=dev), torch.ones(200, device=dev))
    torch.cuda.synchronize()
    assert m.stats[1].item() == 200         # last step: positives only, voided negatives skipped
    m.stats.zero_()
    m2 = DeviceOnlineMF(200, 1000, 16, learning_rate=0.05, negative_sample_rate=2, seed=2, user_memory=16)
    m2.step(users, torch.zeros(200, dtype=torch.int32, device=dev), torch.ones(200, device=dev))
    torch.cuda.synchronize()
    assert m2.stats[1].item() == 600
    m.check_finite(); m.close(); m2.close()


def test_replica_flush_policy_count_timer_any_all_on_device(dev):
    """Count / timer / OR / AND flush conditions evaluated ON THE DEVICE per destination
    (CountLogic.scala:5-29, TimerLogic.scala:6-51, CombinationLogic.scala:12-33)."""
    import time
    from fps_b200.store.replica_cache import ReplicaCache
    from fps_b200.store.sharded_table import ShardedTable

    t = ShardedTable(500, 16, seed=1)
    rc = ReplicaCache(t, flush_count=300, stagger=False, own_inplace=False)       # count only: 100 messages per step
    for _ in range(7):
        rc.after_step(100)
    torch.cuda.synchronize()
    assert rc.flush_counts() == [2]                             # fired at 300 and 600 messages
    assert int(rc.pending[0]) == 100                            # 700 - 2 * 300
    rc = ReplicaCache(t, flush_count=10 ** 9, sync_interval_ms=20, stagger=False, own_inplace=False)   # timer only
    rc.after_step(1); torch.cuda.synchronize(); assert rc.flush_counts() == [0]
    time.sleep(0.03); rc.after_step(1); torch.cuda.synchronize(); assert rc.flush_counts() == [1]
    rc = ReplicaCache(t, flush_count=2, sync_interval_ms=250, require="all", stagger=False, own_inplace=False)
    rc.after_step(1); rc.after_step(1); torch.cuda.synchronize()
    assert rc.flush_counts() == [0]                             # count reached, deadline not yet
    time.sleep(0.3); rc.after_step(1); torch.cuda.synchronize(); assert rc.flush_counts() == [1]
    # a local update reaches the master on flush, and only then
    ids = torch.tensor([7], device=dev)
    before = t.pull(ids)[0, :16].clone()
    rc.cache[rc.row_index(ids)[0], :16] += 1.0
    torch.cuda.synchronize()
    torch.testing.assert_close(t.pull(ids)[0, :16], before)
    rc.flush(); torch.cuda.synchronize()
    torch.testing.assert_close(t.pull(ids)[0, :16], before + 1.0)
    torch.testing.assert_close(rc.rows(ids)[0], before + 1.0)
    assert torch.equal(rc.base, rc.cache)
    t.close()


@pytest.mark.parametrize("dim,n", [(64, 20011), (300, 1777), (3, 513)])
def test_replica_exchange_conserves_every_delta_single_rank(dev, dim, n):
    """Pushes into the replica while exchanges run on the side stream: afterwards the master holds
    init + every delta exactly once, replica == master == base (SimplePSLogic.scala:16-25 semantics
    through the batching path)."""
    from fps_b200.ops import native
    from fps_b200.store.replica_cache import ReplicaCache
    from fps_b200.store.sharded_table import ShardedTable

    t = ShardedTable(n, dim, seed=3, init_range=(-1, 1))
    all_ids = torch.arange(n, device=dev)
    init = t.pull(all_ids).clone()
    rc = ReplicaCache(t, sync_every=2, own_inplace=False)
    g = torch.Generator(device="cpu").manual_seed(dim)
    total = torch.zeros(n, dim, device=dev)
    for step in range(9):
        ids = torch.randint(0, n, (4000,), generator=g).to(dev)
        delta = torch.randn(4000, dim, generator=g).to(dev)
        rc.after_step(4000)                                     # exchange overlaps the push below
        native.push_add(rc.table_c, ids, delta)
        total.index_add_(0, ids, delta)
    rc.refresh(); torch.cuda.synchronize()
    torch.testing.assert_close(t.pull(all_ids), init + total, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(rc.rows(all_ids), init + total, rtol=1e-5, atol=1e-5)
    assert torch.equal(rc.base, rc.cache)
    t.close()


def test_bucket_by_replica_row_and_destination_feed(dev):
    """Owner-major bucketing: bucket = ((item % G) * rps + item // G) >> shift, and the histogram kernel
    feeds the per-destination message counters of the device-side flush policy."""
    from fps_b200.ops import native

    n, n_items, G, shift = 50_001, 6000, 4, 8
    rps = -(-n_items // G)
    g = torch.Generator().manual_seed(5)
    users = torch.randint(0, 1 << 20, (n,), generator=g, dtype=torch.int32).to(dev)
    items = torch.randint(0, n_items, (n,), generator=g, dtype=torch.int32).to(dev)
    ratings = torch.randint(0, 64, (n,), generator=g).float().to(dev)
    scratch = torch.zeros(2 * native.BUCKET_MAX, dtype=torch.int32, device=dev)
    pending = torch.zeros(G, dtype=torch.int64, device=dev)
    nb = -(-(rps * G) >> shift)
    rec = native.pack_ratings(users, items, ratings)
    out, _, _ = native.bucket_by_item(rec, None, None, shift, nb, scratch, num_shards=G,
                                      rows_per_shard=rps, pending=pending)
    assert torch.equal(torch.sort(out).values, torch.sort(rec).values)
    it = (out >> 16) & 0x3FFFFF
    b = ((it % G) * rps + it // G) >> shift
    assert (b[1:] >= b[:-1]).all()
    assert torch.equal(pending, torch.bincount(items.long() % G, minlength=G))


@pytest.mark.parametrize("packed", [False, True])
def test_bucket_by_item_is_a_grouping_permutation(dev, packed):
    from fps_b200.ops import native

    n, n_items, shift = 100_003, 5000, 9                      # 10 buckets of 512 items
    g = torch.Generator().manual_seed(11)
    users = torch.randint(0, 1 << 20, (n,), generator=g, dtype=torch.int32).to(dev)
    items = torch.randint(0, n_items, (n,), generator=g, dtype=torch.int32).to(dev)
    ratings = torch.randint(0, 64, (n,), generator=g).float().to(dev)        # exact in fp16
    scratch = torch.zeros(2 * native.BUCKET_MAX, dtype=torch.int32, device=dev)
    nb = -(-n_items >> shift)
    if packed:
        rec = native.pack_ratings(users, items, ratings)
        out, _, _ = native.bucket_by_item(rec, None, None, shift, nb, scratch)
        assert torch.equal(torch.sort(out).values, torch.sort(rec).values)          # a permutation
        b = ((out >> 16) & 0x3FFFFF) >> shift
    else:
        ou, oi, orat = native.bucket_by_item(users, items, ratings, shift, nb, scratch)
        key_in = (users.long() << 40) | (items.long() << 8) | ratings.long()
        key_out = (ou.long() << 40) | (oi.long() << 8) | orat.long()
        assert torch.equal(torch.sort(key_out).values, torch.sort(key_in).values)
        b = oi.long() >> shift
    assert (b[1:] >= b[:-1]).all()                                                   # grouped by bucket
    assert torch.equal(torch.bincount(b, minlength=nb), torch.bincount(items.long() >> shift, minlength=nb))


def test_item_blocking_changes_order_not_result(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    g = torch.Generator().manual_seed(12)
    nu, ni, n = 50_000, 20_000, 40_000
    users = torch.randperm(nu, generator=g)[:n].to(torch.int32).to(dev)      # distinct users
    items = torch.randint(0, ni, (n,), generator=g, dtype=torch.int32).to(dev)
    ratings = torch.rand(n, generator=g).to(dev)
    a = DeviceOnlineMF(nu, ni, 32, learning_rate=0.05, seed=5, item_blocking=False)
    b = DeviceOnlineMF(nu, ni, 32, learning_rate=0.05, seed=5, item_blocking=True, block_bytes=256 << 10)
    assert b.block_buckets > 4 and not a.item_blocking
    for m in (a, b):
        m.step(users, items, ratings)
        m.step(native_pack(users, items, ratings))
    torch.cuda.synchronize()
    # items are shared between ratings of one batch (asynchronous updates): order changes the result
    # only through which stale value a concurrent update reads -> compare loosely, users exactly-ish
    torch.testing.assert_close(b.items.local, a.items.local, rtol=0, atol=2e-3)
    torch.testing.assert_close(b.users, a.users, rtol=0, atol=2e-3)
    assert b.stats[1].item() == a.stats[1].item() == 2 * n
    a.close(); b.close()


def native_pack(u, i, r):
    from fps_b200.ops import native

    return native.pack_ratings(u, i, r)


def test_fp64_fused_mf_step_matches_float64_reference(dev):
    """The fp64 tier (reference precision, Vector.scala:8): one conflict-free micro-batch against torch float64."""
    from fps_b200.models.mf.device_f64 import DeviceOnlineMFf64
    from fps_b200.ops import native

    nu, ni, k, b, lr = 3000, 2000, 10, 1500, 0.05
    m = DeviceOnlineMFf64(nu, ni, k, range_min=-0.5, range_max=0.5, learning_rate=lr, seed=7)
    U0, V0 = m.users[:, :k].clone(), m.items_f64[:, :k].clone()
    assert U0.dtype == torch.float64 and float(U0.abs().max()) <= 0.5 and float(U0.std()) > 0.2
    g = torch.Generator().manual_seed(2)
    users = torch.randperm(nu, generator=g)[:b].int().to(dev)
    items = torch.randperm(ni, generator=g)[:b].int().to(dev)
    ratings = torch.rand(b, generator=g).to(dev)
    m.step(users, items, ratings)
    torch.cuda.synchronize()
    u, v = U0[users.long()], V0[items.long()]
    e = torch.sigmoid(ratings.double() - (u * v).sum(1))
    lr = float(torch.tensor(lr, dtype=torch.float32))        # the learning rate travels as an fp32 kernel argument
    U = U0.clone(); U[users.long()] += lr * e[:, None] * v
    V = V0.clone(); V[items.long()] += lr * e[:, None] * u
    torch.testing.assert_close(m.users[:, :k], U, rtol=1e-12, atol=1e-13)
    torch.testing.assert_close(m.items_f64[:, :k], V, rtol=1e-12, atol=1e-13)
    torch.testing.assert_close(m.predict(users, items), (U[users.long()] * V[items.long()]).sum(1),
                               rtol=1e-12, atol=1e-13)
    m.step(native.pack_ratings(users, items, ratings.half().float()))      # packed64 records: same kernel
    torch.cuda.synchronize()
    m.check_finite(); assert m.stats[1].item() == 2 * b
    m.close()
