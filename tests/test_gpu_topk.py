"""wgmma top-K scoring kernel vs fp32 PyTorch (TF32 tolerance) and brute-force top-K."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.mark.parametrize("nq,ni,k", [(128, 256, 64), (200, 1000, 64), (50, 333, 16), (300, 5000, 128), (130, 700, 10)])
def test_scores_match_fp32_matmul(dev, nq, ni, k):
    from fps_b200.models.mf.device_topk import DeviceTopK

    stride = (k + 3) // 4 * 4
    g = torch.Generator(device="cpu").manual_seed(nq + ni)
    items = torch.zeros(ni, stride); items[:, :k] = torch.randn(ni, k, generator=g)
    q = torch.zeros(nq, stride); q[:, :k] = torch.randn(nq, k, generator=g)
    items, q = items.to(dev), q.to(dev)
    got = DeviceTopK(items).scores(q_local=q)
    ref = q.double() @ items.double().T
    err = (got.double() - ref).abs().max().item()
    assert err < 2e-2 * (k ** 0.5), err          # TF32: 10-bit mantissa inputs, fp32 accumulate
    assert torch.allclose(got.double(), ref, rtol=5e-3, atol=5e-2)


def test_topk_equals_brute_force_with_pull_from_ps(dev):
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.store.sharded_table import ShardedTable

    k, nu, ni, K = 64, 3000, 20000, 100
    users = ShardedTable(nu, k, seed=1, init_range=(-1.0, 1.0))
    g = torch.Generator(device="cpu").manual_seed(0)
    scale = torch.rand(ni, 1, generator=g) * 2 + 0.1
    items = (torch.randn(ni, k, generator=g) * scale).to(dev).contiguous()
    q_ids = torch.randint(0, nu, (517,), generator=g).to(dev)
    tk = DeviceTopK(items)
    sc, rows = tk.topk(K, q_ids=q_ids, q_table=users)
    full = tk.scores(q_ids=q_ids, q_table=users)            # same TF32 arithmetic
    ref = torch.topk(full, K, dim=1)
    assert torch.equal(sc, ref.values)
    # item sets must agree wherever scores are distinct
    same = (rows == ref.indices) | (sc == torch.roll(sc, 1, 1)) | (sc == torch.roll(sc, -1, 1))
    assert same.all()
    # and against exact fp32: the exact top-10 must be inside the TF32 top-100
    u = users.pull(q_ids)
    exact = torch.topk(u @ items.T, 10, dim=1).indices
    hit = (exact[:, :, None] == rows[:, None, :]).any(-1).float().mean().item()
    assert hit > 0.999, hit
    sc2, rows2 = tk.topk(10, q_ids=q_ids, q_table=users, rescore=True)
    assert (sc2[:, :-1] >= sc2[:, 1:]).all()
    users.close()


def test_topk_small_item_table_and_k_larger_than_tiles(dev):
    from fps_b200.models.mf.device_topk import DeviceTopK, merge_partial_topk

    items = torch.randn(300, 32, device=dev)
    q = torch.randn(40, 32, device=dev)
    tk = DeviceTopK(items)
    sc, rows = tk.topk(50, q_local=q)
    ref = torch.topk(tk.scores(q_local=q), 50, dim=1)
    assert torch.equal(sc, ref.values)
    ms, mi = merge_partial_topk(torch.cat([sc, sc - 1000], 1), torch.cat([rows, rows], 1), 50)
    assert torch.equal(ms, sc) and torch.equal(mi, rows)


def test_length_sorted_pruning_is_exact_and_skips_short_tiles(dev):
    """LEMP LENGTH bound at tile granularity: skewed item lengths => only a prefix of the length-sorted
    table is scored, and the result equals the unpruned top-K (same TF32 scores, caller's row ids)."""
    from fps_b200.models.mf.device_topk import DeviceTopK

    k, ni, K = 64, 60000, 50
    g = torch.Generator(device="cpu").manual_seed(3)
    scale = torch.exp(torch.randn(ni, 1, generator=g) * 1.2)            # log-normal lengths (popularity skew)
    items = (torch.randn(ni, k, generator=g) * scale).to(dev).contiguous()
    q = torch.randn(700, k, generator=g).to(dev)
    plain, pruned = DeviceTopK(items), DeviceTopK(items, sort_by_length=True)
    sc0, rows0 = plain.topk(K, q_local=q)
    sc1, rows1 = pruned.topk(K, q_local=q)
    p1, p2 = pruned.last_tiles_scored
    assert p2 < pruned.n_tiles // 2 and p1 < pruned.n_tiles, (p1, p2, pruned.n_tiles)
    torch.testing.assert_close(sc1, sc0, rtol=0, atol=0)
    same = (rows1 == rows0) | (sc0 == torch.roll(sc0, 1, 1)) | (sc0 == torch.roll(sc0, -1, 1))
    assert same.all()
    # uniform lengths: nothing can be pruned, results still identical
    items2 = torch.nn.functional.normalize(torch.randn(5000, k, generator=g), dim=1).to(dev).contiguous()
    a, b = DeviceTopK(items2), DeviceTopK(items2, sort_by_length=True)
    s_a, r_a = a.topk(20, q_local=q[:130]); s_b, r_b = b.topk(20, q_local=q[:130])
    torch.testing.assert_close(s_b, s_a, rtol=0, atol=0)
    assert b.last_tiles_scored[1] == b.n_tiles


@pytest.mark.parametrize("n,L,K", [(37, 100, 1), (64, 7813, 100), (5, 50000, 257), (16, 1024, 1024), (9, 300, 50)])
def test_row_kth_largest_matches_torch(dev, n, L, K):
    from fps_b200.ops import native

    g = torch.Generator(device="cpu").manual_seed(n * L)
    x = (torch.randn(n, L, generator=g) * torch.exp(torch.randn(n, 1, generator=g) * 3)).to(dev)
    x[0, : L // 2] = x[0, 0]                                   # many equal values in one row
    if n > 2:
        x[1] = -x[1].abs()                                     # all negative
        x[2, ::3] = 0.0
    ref = torch.topk(x, K, dim=1).values[:, -1]
    assert torch.equal(native.row_kth_largest(x, K), ref)
    counts = torch.randint(0, L + 1, (n,), generator=g, dtype=torch.int32).to(dev)
    got = native.row_kth_largest(x, K, counts=counts)
    for r in range(n):
        c = int(counts[r])
        want = torch.topk(x[r, :c], K).values[-1].item() if c >= K else -3.0e38
        assert got[r].item() == pytest.approx(want, rel=0, abs=0) or (c < K and got[r].item() < -2.9e38)


@pytest.mark.parametrize("n,cap,K", [(33, 1024, 100), (7, 8192, 1000), (20, 300, 50), (4, 60000, 10), (12, 64, 64)])
def test_row_topk_sorted_matches_torch(dev, n, cap, K):
    from fps_b200.ops import native

    g = torch.Generator(device="cpu").manual_seed(cap + K)
    cs = torch.randn(n, cap, generator=g).to(dev)
    ci = torch.stack([torch.randperm(cap * 3, generator=g)[:cap] for _ in range(n)]).to(torch.int32).to(dev)
    ref = torch.topk(cs, K, dim=1)
    s, i = native.row_topk(cs, ci, K)
    assert torch.equal(s, ref.values) and torch.equal(i, torch.gather(ci, 1, ref.indices))
    counts = torch.randint(0, cap + 1, (n,), generator=g, dtype=torch.int32).to(dev)
    counts[0] = 0
    s, i = native.row_topk(cs, ci, K, counts=counts)
    for r in range(n):
        c = int(counts[r]); kk = min(K, c)
        want = torch.topk(cs[r, :c], kk)
        assert torch.equal(s[r, :kk], want.values) and torch.equal(i[r, :kk], ci[r, :c][want.indices])
        assert (s[r, kk:] < -2.9e38).all() and (i[r, kk:] == -1).all()
    # ties: equal scores come out by ascending item id
    cs2 = torch.full((3, 500), -1.0, device=dev); cs2[:, :7] = 1.0; cs2[:, 7:37] = 0.0
    ci2 = torch.arange(500, 0, -1, dtype=torch.int32, device=dev).repeat(3, 1).contiguous()
    s, i = native.row_topk(cs2, ci2, 20)
    assert (s[:, :7] == 1).all() and (s[:, 7:] == 0).all()
    assert torch.equal(i[0, :7], torch.arange(494, 501, dtype=torch.int32, device=dev))
    assert torch.equal(i[0, 7:], torch.arange(464, 477, dtype=torch.int32, device=dev))


def test_topk_degenerate_queries_fall_back_to_brute_force(dev):
    """An all-zero query ties every item at score 0: candidate segments overflow, theta cannot rise, and
    the row must be answered by the brute-force path; ordinary rows of the same batch stay exact."""
    from fps_b200.models.mf.device_topk import DeviceTopK

    g = torch.Generator(device="cpu").manual_seed(8)
    items = torch.randn(40000, 32, generator=g).to(dev)
    q = torch.randn(300, 32, generator=g).to(dev)
    q[7] = 0.0
    q[123] = 0.0
    for sort in (False, True):
        tk = DeviceTopK(items, sort_by_length=sort)
        sc, rows = tk.topk(25, q_local=q)
        ref = torch.topk(DeviceTopK(items).scores(q_local=q), 25, dim=1)
        assert torch.equal(sc, ref.values)
        assert (sc[7] == 0).all() and (sc[123] == 0).all()
        ok = torch.ones(300, dtype=torch.bool, device=dev); ok[7] = ok[123] = False
        same = (rows == ref.indices) | (sc == torch.roll(sc, 1, 1)) | (sc == torch.roll(sc, -1, 1))
        assert same[ok].all()
        assert rows.min() >= 0 and rows.max() < 40000 and len(set(rows[7].tolist())) == 25


def test_distributed_topk_single_rank_maps_to_global_ids(dev):
    from fps_b200.models.mf.device_topk import DistributedTopK
    from fps_b200.store.sharded_table import ShardedTable

    users = ShardedTable(2000, 32, seed=4, init_range=(-1, 1))
    g = torch.Generator(device="cpu").manual_seed(9)
    items = torch.randn(3000, 32, generator=g).to(dev)
    gids = (torch.arange(3000, device=dev) * 7 + 3)
    q = torch.randint(0, 2000, (150,), generator=g).to(dev)
    sc, ids = DistributedTopK(users, items, gids).topk(q, 15, workerK=15)
    exact = users.pull(q) @ items.T
    ref = torch.topk(exact, 15, dim=1)
    overlap = (ids[:, :, None] == gids[ref.indices][:, None, :]).any(-1).float().mean().item()
    assert overlap > 0.97 and ((ids - 3) % 7 == 0).all()
    torch.testing.assert_close(sc, ref.values, rtol=2e-2, atol=2e-2)
    users.close()


def test_ps_topk_generator_and_online_learner_device_backends(dev):
    """Reference-shaped entry points on the device tier: same lists as the host tier (LEMP scan) for a
    pre-trained model; unknown users get an empty list; the online learner is prequential."""
    import numpy as np

    from fps_b200.api import Left, Right
    from fps_b200.models.mf.common import Rating, attachLength
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator, psTopKGenerator

    rng = np.random.RandomState(0)
    k, n_items, n_users = 8, 300, 40
    items = {i: rng.randn(k) * (0.5 + rng.rand()) for i in range(n_items)}
    users = {u: rng.randn(k) for u in range(0, n_users, 2)}            # odd users are unknown
    model = [Left((i, attachLength(v))) for i, v in items.items()] + \
            [Right((u, attachLength(v))) for u, v in users.items()]
    queries = [Rating(int(u), int(rng.randint(n_items)), 1.0, t) for t, u in enumerate(rng.randint(0, n_users, 60))]
    host = psTopKGenerator(queries, model, K=10, workerK=10, workerParallelism=2, psParallelism=2,
                           iterationWaitTime=200)
    devr = psTopKGenerator(queries, model, K=10, workerK=10, backend="device")
    assert len(devr) == len(queries)
    by_ts = {ts: topk for (_item, ts, topk) in host}
    for (item, ts, topk), q in zip(devr, queries):
        assert item == q.item and ts == q.timestamp
        if q.user % 2 == 1:
            assert topk == []
            continue
        want = by_ts[ts]
        assert len(set(i for _, i in topk) & set(i for _, i in want)) >= 9          # same items (TF32 near-ties) ...
        np.testing.assert_allclose([s for s, _ in topk], [s for s, _ in want], rtol=5e-3, atol=5e-3)  # TF32 scores
    # online learner + generator: one list per rating, lists exclude nothing for memory 0, model trains
    ratings = [Rating(int(rng.randint(30)), int(rng.randint(50)), 1.0, t) for t in range(500)]
    out = psOnlineLearnerAndGenerator(ratings, numFactors=8, K=5, userMemory=0, backend="device",
                                      learningRate=0.1, rangeMin=0.05, rangeMax=0.3, batch_size=100,
                                      plain_residual=True)
    assert len(out) == 500 and all(len(t) == 5 for (_u, _i, _ts, t) in out)
    assert [(u, i, ts) for (u, i, ts, _t) in out] == [(r.user, r.item, r.timestamp) for r in ratings]
    pred = out.model.predict(torch.tensor([r.user for r in ratings[:100]], device=dev, dtype=torch.int32),
                             torch.tensor([r.item for r in ratings[:100]], device=dev, dtype=torch.int32))
    assert pred.mean().item() > 0.45                                   # trained towards rating 1 from ~0.25
    out.model.close()
