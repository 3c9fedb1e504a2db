"""Device top-K with per-query exclusion lists (the seen-item filter of the generators) against brute
force over the same TF32 scores, the select kernels' per-row arguments against torch, and the device
generators against ``_seen_filter`` applied to complete candidate lists."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _csr(lists, dev):
    off = np.zeros(len(lists) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(x) for x in lists])
    flat = np.concatenate([np.asarray(x, dtype=np.int64) for x in lists]) if off[-1] else np.zeros(0, np.int64)
    return torch.from_numpy(off).to(dev), torch.from_numpy(flat).to(dev)


def _masked(full, lists):
    """Scores with the excluded (in-range) columns of every row at -inf."""
    full = full.clone()
    for q, x in enumerate(lists):
        x = [i for i in x if 0 <= i < full.shape[1]]
        if x:
            full[q, torch.tensor(x, device=full.device)] = float("-inf")
    return full


def _assert_exact(sc, rows, masked, K):
    """``(sc, rows)`` is the top-K of ``masked``: same scores, same items wherever scores are distinct,
    ``(-3e38, -1)`` where fewer than K admissible items exist, no excluded item."""
    ref = torch.topk(masked, K, dim=1)
    valid = ref.values > float("-inf")
    assert torch.equal(sc, torch.where(valid, ref.values, torch.full_like(sc, -3.0e38)))
    assert (rows[~valid] == -1).all()
    same = (rows == ref.indices) | (sc == torch.roll(sc, 1, 1)) | (sc == torch.roll(sc, -1, 1))
    assert same[valid].all()
    got = torch.gather(masked, 1, rows.clamp_min(0))
    assert (got[valid] > float("-inf")).all()                                 # nothing excluded came back
    for r in range(rows.shape[0]):                                            # and no item twice
        v = rows[r][rows[r] >= 0]
        assert v.unique().numel() == v.numel()


def _exclusions(full, K, rng, n_items):
    """Mixed exclusion lists: exact top-3K of the query (adversarial), random ids with duplicates and
    out-of-range values, and empty rows."""
    top = torch.topk(full, 3 * K, dim=1).indices.cpu().numpy()
    lists = []
    for q in range(full.shape[0]):
        kind = q % 3
        if kind == 0:
            lists.append(rng.permutation(top[q]).tolist())
        elif kind == 1:
            x = rng.randint(-20, n_items + 20, rng.randint(0, 4 * K)).tolist()
            lists.append(x + x[: len(x) // 3])                                # duplicates
        else:
            lists.append([] if q % 2 else top[q, :2].tolist() * 2)
    return lists


@pytest.mark.parametrize("sort", [False, True])
def test_exclude_q_ids_sharded_table_matches_brute_force(dev, sort):
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.store.sharded_table import ShardedTable

    k, nu, ni, K = 64, 3000, 60000, 20
    users = ShardedTable(nu, k, seed=1, init_range=(-1.0, 1.0))
    g = torch.Generator(device="cpu").manual_seed(11)
    scale = torch.exp(torch.randn(ni, 1, generator=g) * 1.2)                  # skewed lengths: pruning bites
    items = (torch.randn(ni, k, generator=g) * scale).to(dev).contiguous()
    q_ids = torch.randint(0, nu, (301,), generator=g).to(dev)
    tk = DeviceTopK(items, sort_by_length=sort)
    full = tk.scores(q_ids=q_ids, q_table=users)
    lists = _exclusions(full, K, np.random.RandomState(1), ni)
    off, rows = _csr(lists, dev)
    sc, got = tk.topk(K, q_ids=q_ids, q_table=users, exclude=(off, rows))
    _assert_exact(sc, got, _masked(full, lists), K)
    if sort:
        assert tk.last_tiles_scored[1] < tk.n_tiles                          # the LENGTH bound still prunes
    # no exclusion at all == the plain call, and an all-out-of-range list too
    s0, r0 = tk.topk(K, q_ids=q_ids, q_table=users)
    empty = (torch.zeros(302, dtype=torch.int64, device=dev), torch.zeros(0, dtype=torch.int64, device=dev))
    s1, r1 = tk.topk(K, q_ids=q_ids, q_table=users, exclude=empty)
    assert torch.equal(s0, s1) and torch.equal(r0, r1)
    # rescore keeps the admissible set
    s2, r2 = tk.topk(K, q_ids=q_ids, q_table=users, exclude=(off, rows), rescore=True)
    assert (torch.gather(_masked(full, lists), 1, r2) > float("-inf")).all()
    assert (s2[:, :-1] >= s2[:, 1:]).all()
    # several query chunks (256 rows each): the exclusion CSR is sliced and rebased per chunk
    tk.max_batch_bytes = 1
    s3, r3 = tk.topk(K, q_ids=q_ids, q_table=users, exclude=(off, rows))
    _assert_exact(s3, r3, _masked(full, lists), K)
    assert torch.equal(s3, sc) and torch.equal(r3, got)
    users.close()


@pytest.mark.parametrize("sort", [False, True])
def test_exclude_q_local_short_rows_and_degenerate_query(dev, sort):
    from fps_b200.models.mf.device_topk import DeviceTopK

    g = torch.Generator(device="cpu").manual_seed(12)
    # small table: rows that exclude almost everything have fewer than K admissible items
    items = torch.randn(300, 32, generator=g).to(dev)
    q = torch.randn(40, 32, generator=g).to(dev)
    tk = DeviceTopK(items, sort_by_length=sort)
    full = tk.scores(q_local=q)
    rng = np.random.RandomState(2)
    lists = [rng.permutation(300)[: rng.randint(0, 300)].tolist() for _ in range(40)]
    lists[0] = list(range(300))                                               # nothing admissible
    lists[1] = list(range(290))                                               # 10 < K admissible
    lists[2] = []
    sc, rows = tk.topk(50, q_local=q, exclude=_csr(lists, dev))
    _assert_exact(sc, rows, _masked(full, lists), 50)
    assert (rows[0] == -1).all() and (rows[1, :10] >= 290).all() and (rows[1, 10:] == -1).all()
    # an all-zero query ties every item at 0: its candidate segments overflow whatever theta is, so it is
    # answered by the brute-force fallback, which must mask the excluded columns.  The exclusion lists stay
    # short (K + max E_q well below the tile count), so the candidate buffer keeps its usual size.
    items = torch.randn(40000, 32, generator=g).to(dev)
    q = torch.randn(300, 32, generator=g).to(dev)
    q[7] = 0.0
    q[280] = 0.0
    tk = DeviceTopK(items, sort_by_length=sort)
    full = tk.scores(q_local=q)
    lists = [rng.randint(0, 40000, 30).tolist() for _ in range(300)]
    lists[7] = list(range(30)) + [-1, 40000]                                  # the first 30 rows, out of range
    lists[280] = list(range(30, 60))
    for max_bytes in (512 << 20, 1):                                          # one chunk; chunks of 256 rows
        tk.max_batch_bytes = max_bytes
        sc, rows = tk.topk(25, q_local=q, exclude=_csr(lists, dev))
        assert tk.last_fallback_rows >= 2
        _assert_exact(sc, rows, _masked(full, lists), 25)
        assert (sc[7] == 0).all() and (rows[7] >= 30).all()
        assert (sc[280] == 0).all() and ((rows[280] < 30) | (rows[280] >= 60)).all()


@pytest.mark.parametrize("n,L", [(37, 100), (64, 7813), (5, 50000)])
def test_row_kth_largest_k_per_row(dev, n, L):
    from fps_b200.ops import native

    g = torch.Generator(device="cpu").manual_seed(n + L)
    x = (torch.randn(n, L, generator=g) * torch.exp(torch.randn(n, 1, generator=g) * 3)).to(dev)
    x[0, : L // 2] = x[0, 0]
    kpr = torch.randint(1, min(L, 400) + 1, (n,), generator=g, dtype=torch.int32)
    kpr[1] = L
    kpr[2] = L + 5                                                            # more than the row holds
    got = native.row_kth_largest(x, 7, k_per_row=kpr.to(dev))
    for r in range(n):
        k = int(kpr[r])
        want = torch.topk(x[r], k).values[-1].item() if k <= L else -3.0e38
        assert got[r].item() == want or (k > L and got[r].item() < -2.9e38)
    got_cols = native.row_kth_largest(x, 7, n_cols=L // 2, k_per_row=kpr.to(dev))
    for r in range(n):
        k = int(kpr[r])
        want = torch.topk(x[r, : L // 2], k).values[-1].item() if k <= L // 2 else -3.0e38
        assert got_cols[r].item() == want or (k > L // 2 and got_cols[r].item() < -2.9e38)
    with pytest.raises(ValueError):
        native.row_kth_largest(x, 7, k_per_row=kpr[:-1].to(dev))
    with pytest.raises(TypeError):
        native.row_kth_largest(x, 7, k_per_row=kpr.to(dev, torch.int64))


@pytest.mark.parametrize("n,cap,K", [(33, 1024, 100), (7, 8192, 1000), (20, 300, 50), (4, 60000, 10)])
def test_row_topk_exclude_matches_torch(dev, n, cap, K):
    from fps_b200.ops import native

    g = torch.Generator(device="cpu").manual_seed(cap * 3 + K)
    rng = np.random.RandomState(cap)
    cs = torch.randn(n, cap, generator=g)
    ci = torch.stack([torch.randperm(cap * 3, generator=g)[:cap] for _ in range(n)]).to(torch.int32)
    lists = []
    for r in range(n):
        present = ci[r, rng.permutation(cap)[: rng.randint(0, cap)]].tolist()
        absent = rng.randint(cap * 3, cap * 4, rng.randint(0, 20)).tolist()
        lists.append(sorted(set(present + absent)))
    lists[0] = sorted(ci[0].tolist())                                         # every candidate excluded
    lists[1] = sorted(ci[1].tolist())[: cap - K // 2]                         # fewer than K left
    off = torch.tensor(np.cumsum([0] + [len(x) for x in lists]), dtype=torch.int32)
    flat = torch.tensor([i for x in lists for i in x], dtype=torch.int32)
    s, i = native.row_topk(cs.to(dev), ci.to(dev), K, exclude=(off.to(dev), flat.to(dev)))
    s, i = s.cpu(), i.cpu()
    for r in range(n):
        keep = ~torch.isin(ci[r], torch.tensor(lists[r], dtype=torch.int32))
        adm_s, adm_i = cs[r][keep], ci[r][keep]
        kk = min(K, adm_s.numel())
        want = torch.topk(adm_s, kk)
        assert torch.equal(s[r, :kk], want.values) and torch.equal(i[r, :kk], adm_i[want.indices])
        assert (s[r, kk:] < -2.9e38).all() and (i[r, kk:] == -1).all()
    # empty exclusion lists: the plain result
    z = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    s2, i2 = native.row_topk(cs.to(dev), ci.to(dev), K, exclude=(z, torch.zeros(0, dtype=torch.int32, device=dev)))
    s3, i3 = native.row_topk(cs.to(dev), ci.to(dev), K)
    assert torch.equal(s2, s3) and torch.equal(i2, i3)
    with pytest.raises(ValueError):
        native.row_topk(cs.to(dev), ci.to(dev), K, exclude=(z[:-1], flat.to(dev)))


# --------------------------------------------------------------------------------------------------
# generators
# --------------------------------------------------------------------------------------------------
def _oracle(rows_full, K, memory):
    from fps_b200.models.mf.device_api import _seen_filter

    return _seen_filter(rows_full, K, memory)


def _assert_lists_equal(got, want):
    """Same scores; same items wherever neighbouring scores differ (TF32 ties may swap)."""
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert len(a) == len(b), (a, b)
        sa, sb = np.array([s for s, _ in a]), np.array([s for s, _ in b])
        np.testing.assert_allclose(sa, sb, rtol=1e-6, atol=1e-7)
        for j, ((s, i), (_s2, i2)) in enumerate(zip(a, b)):
            tie = any(abs(s - b[t][0]) <= 1e-6 * max(1.0, abs(s)) for t in (j - 1, j + 1) if 0 <= t < len(b))
            assert i == i2 or tie, (j, a, b)


def test_topk_generator_device_seen_items_are_excluded_exactly(dev):
    """A user who rates more of their own top items than any fixed over-fetch allows still gets K items."""
    from fps_b200.api import Left, Right
    from fps_b200.models.mf.common import Rating, attachLength
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.models.mf.topk import psTopKGenerator
    from fps_b200.store.sharded_table import ShardedTable

    rng = np.random.RandomState(4)
    k, n_items, n_users, K = 8, 3000, 30, 10
    item_vecs = rng.randn(n_items, k).astype(np.float32) * (0.3 + rng.rand(n_items, 1).astype(np.float32))
    user_vecs = rng.randn(n_users, k).astype(np.float32)
    model = [Left((i, attachLength(item_vecs[i]))) for i in range(n_items)] + \
            [Right((u, attachLength(user_vecs[u]))) for u in range(n_users)]
    # the TF32 scores the device computes: same table layout (flag column 1.0 on users, 0 on items)
    table = ShardedTable(n_users, k + 1, init="zeros")
    uv = torch.zeros((n_users, k + 1), device=dev)
    uv[:, :k] = torch.from_numpy(user_vecs).to(dev); uv[:, k] = 1.0
    table.load(torch.arange(n_users, device=dev), uv)
    local = torch.zeros((n_items, table.stride), device=dev)
    local[:, :k] = torch.from_numpy(item_vecs).to(dev)
    full = DeviceTopK(local).scores(q_ids=torch.arange(n_users, device=dev), q_table=table).cpu().numpy()
    table.close()
    order = np.lexsort((np.arange(n_items)[None, :].repeat(n_users, 0), -full), axis=1)
    # user 3 rates its own top-6K items in rank order, then everybody rates at random
    ratings, t = [], 0
    for i in order[3, : 6 * K]:
        ratings.append(Rating(3, int(i), 1.0, t)); t += 1
    for _ in range(200):
        u = int(rng.randint(n_users))
        i = int(order[u, rng.randint(3 * K)]) if rng.rand() < 0.5 else int(rng.randint(n_items))
        ratings.append(Rating(u, i, 1.0, t)); t += 1
    for memory in (-1, 50, 5):
        got = psTopKGenerator(ratings, model, K=K, workerK=K, userMemory=memory, backend="device", batch_size=64)
        rows_full = [(r.user, r.item, r.timestamp, [(float(full[r.user, j]), int(j)) for j in order[r.user]])
                     for r in ratings]
        want = _oracle(rows_full, K, memory)
        assert [(i, ts) for i, ts, _ in got] == [(r.item, r.timestamp) for r in ratings]
        _assert_lists_equal([x for _, _, x in got], [x for _, _, _, x in want])
        assert all(len(x) == K for _, _, x in got)


@pytest.mark.parametrize("memory", [3, -1])
@pytest.mark.parametrize("batch_size", [1, 50])
def test_online_learner_device_without_learning_matches_seen_filter(dev, memory, batch_size):
    """learningRate=0 keeps the Philox initialisation, so brute force over the final model is exact."""
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator

    rng = np.random.RandomState(5)
    n_users, n_items, K = 20, 300, 10
    # a first pass only to read the initial model (the stream does not change it)
    kw = dict(numFactors=16, K=K, learningRate=0.0, rangeMin=-1.0, rangeMax=1.0, seed=3, backend="device",
              numUsers=n_users, numItems=n_items, plain_residual=True)
    probe = psOnlineLearnerAndGenerator([Rating(0, 0, 1.0, 0)], userMemory=0, **kw)
    users_all = torch.arange(n_users, device=dev)
    full = DeviceTopK(probe.items[: probe.n_items]).scores(q_ids=users_all, q_table=probe.users).cpu().numpy()
    probe.model.close()
    order = np.lexsort((np.arange(n_items)[None, :].repeat(n_users, 0), -full), axis=1)
    ratings, t = [], 0
    for i in order[2, : 3 * K]:                                               # user 2 rates its own top-3K
        ratings.append(Rating(2, int(i), 1.0, t)); t += 1
    for _ in range(150):
        u = int(rng.randint(n_users))
        i = int(order[u, rng.randint(2 * K)]) if rng.rand() < 0.6 else int(rng.randint(n_items))
        ratings.append(Rating(u, i, 1.0, t)); t += 1
    out = psOnlineLearnerAndGenerator(ratings, userMemory=memory, batch_size=batch_size, **kw)
    after = DeviceTopK(out.items[: out.n_items]).scores(q_ids=users_all, q_table=out.users).cpu().numpy()
    assert np.array_equal(after, full)                                        # nothing was learned
    rows_full = [(r.user, r.item, r.timestamp, [(float(full[r.user, j]), int(j)) for j in order[r.user]])
                 for r in ratings]
    want = _oracle(rows_full, K, memory)
    assert [(u, i, ts) for (u, i, ts, _) in out] == [(r.user, r.item, r.timestamp) for r in ratings]
    _assert_lists_equal([x for *_, x in out], [x for *_, x in want])
    assert all(len(x) == K for *_, x in out)
    out.model.close()


@pytest.mark.timeout(900)               # the torchrun children have their own 420 s limit
def test_multi_rank_distributed_topk_exclude():
    from tests.test_gpu_multi import _run

    _run("mp_topk_exclude_check.py", 2, 29631, "MP_TOPK_EXCLUDE_CHECK_OK")
