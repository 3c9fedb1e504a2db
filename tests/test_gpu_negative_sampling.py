"""Negatives from the items each worker has seen (``negative_sampling="seen"``) and skip-gram's unigram noise on
the device: the registry against the numpy reference, the domain each record draws from, counts, uniformity,
determinism, training numerics against fp32 torch, untouched rows and the multi-rank split."""
from collections import deque

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models.mf.common import SeenRegistryOracle
from fps_b200.ops import native

pytestmark = pytest.mark.gpu


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _first_occurrence(items):
    _, idx = np.unique(np.asarray(items), return_index=True)
    return np.asarray(items)[np.sort(idx)]


def _records(fmt, users, items, ratings):
    if fmt == "packed64":
        return (native.pack_ratings(users, items, ratings),)
    idt = torch.int32 if fmt == "int32" else torch.int64
    return users.to(idt), items.to(idt), ratings


@pytest.mark.parametrize("fmt", ["int32", "int64", "packed64"])
def test_seen_items_is_the_first_occurrence_order(dev, fmt):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni = 3000, 5000
    m = DeviceOnlineMF(nu, ni, 16, negative_sample_rate=2, user_memory=8, negative_sampling="seen", seed=3)
    g = torch.Generator().manual_seed(11)
    stream = []
    for n in (700, 1, 2500, 1200):
        users = torch.randint(0, nu, (n,), generator=g)
        items = torch.randint(0, ni // 4, (n,), generator=g)    # repeats inside and across micro-batches
        stream.append(items)
        m.step(*_records(fmt, users.to(dev), items.to(dev), torch.ones(n, device=dev)))
    want = _first_occurrence(torch.cat(stream).numpy())
    np.testing.assert_array_equal(m.seen_items().cpu().numpy(), want)
    m.check_finite()
    m.close()


def _sample(users, items, neg_rate, registry, memory, n_users, step, seed=5):
    seen = seen_pos = None
    if memory:
        seen = torch.full((n_users, memory), -1, dtype=torch.int32, device=users.device)
        seen_pos = torch.zeros(n_users, dtype=torch.int32, device=users.device)
    return native.neg_sample_seen(users, items, torch.ones(users.numel(), device=users.device), neg_rate, registry,
                                  seen, seen_pos, seed=seed, step=step), (seen, seen_pos)


def test_every_negative_is_in_its_domain_and_outside_the_ring(dev):
    nu, ni, m_neg, memory = 64, 400, 3, 4
    reg = native.seen_registry(ni, dev)
    oracle = SeenRegistryOracle(ni, nu, m_neg, memory)
    seen = torch.full((nu, memory), -1, dtype=torch.int32, device=dev)
    seen_pos = torch.zeros(nu, dtype=torch.int32, device=dev)
    rings = {}
    g = torch.Generator().manual_seed(2)
    for step in range(6):
        users = torch.randperm(nu, generator=g)[:48]                          # distinct users per batch
        items = torch.randint(0, ni // 2, (48,), generator=g)
        dom, _, k = oracle.batch(users.numpy(), items.numpy())
        order = oracle.order
        ou, oi, orat = native.neg_sample_seen(users.int().to(dev), items.int().to(dev), torch.ones(48, device=dev),
                                              m_neg, reg, seen, seen_pos, seed=9, step=step)
        ou, oi, orat = (t.view(48, 1 + m_neg).cpu().numpy() for t in (ou, oi, orat))
        np.testing.assert_array_equal(ou[:, 0], users.numpy())
        np.testing.assert_array_equal(oi[:, 0], items.numpy())
        assert (orat[:, 1:] == 0).all()
        for p in range(48):
            u, it = int(users[p]), int(items[p])
            ring = rings.setdefault(u, deque(maxlen=memory))
            ring.append(it)
            domain = set(order[:dom[p]].tolist())
            drawn = [int(x) for x, uu in zip(oi[p, 1:], ou[p, 1:]) if uu >= 0]
            assert (ou[p, 1 + k[p]:] == -1).all()
            for x in drawn:
                assert x in domain and x not in ring and x != it, (step, p, x)
        np.testing.assert_array_equal(reg[0][:int(reg[1].item())].cpu().numpy(), oracle.order)


def test_only_admissible_item_is_drawn(dev):
    """The user rated 3, the registry holds 3 and 4: with a one-item ring the only admissible item is 4."""
    reg = native.seen_registry(10, dev)
    seen = torch.full((2, 1), -1, dtype=torch.int32, device=dev)
    seen_pos = torch.zeros(2, dtype=torch.int32, device=dev)
    one = torch.ones(2, device=dev)
    native.neg_sample_seen(torch.tensor([0, 1], device=dev, dtype=torch.int32),
                           torch.tensor([3, 4], device=dev, dtype=torch.int32), one, 1, reg, seen, seen_pos, step=0)
    ou, oi, _ = native.neg_sample_seen(torch.tensor([0], device=dev, dtype=torch.int32),
                                       torch.tensor([3], device=dev, dtype=torch.int32), one[:1], 1, reg, seen,
                                       seen_pos, step=1)
    assert ou.tolist() == [0, 0] and oi.tolist() == [3, 4]


def test_first_record_is_void_and_own_first_item_joins_from_the_next_record(dev):
    reg = native.seen_registry(100, dev)
    users = torch.tensor([0, 1, 2], device=dev, dtype=torch.int32)
    items = torch.tensor([10, 11, 12], device=dev, dtype=torch.int32)
    (ou, oi, _), _ = _sample(users, items, 2, reg, 0, 3, step=0)
    ou, oi = ou.view(3, 3).tolist(), oi.view(3, 3).tolist()
    assert ou[0] == [0, -1, -1]                  # empty domain
    assert ou[1] == [1, 1, -1] and oi[1][1] == 10   # D_1 = [10]: 11 is not in it yet
    assert ou[2][1:] == [2, 2] and set(oi[2][1:]) <= {10, 11} and 12 not in oi[2][1:]


def test_stats_count_the_oracle_negatives(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, neg, memory = 4000, 1000, 2, 2
    m = DeviceOnlineMF(nu, ni, 16, negative_sample_rate=neg, user_memory=memory, negative_sampling="seen",
                       seed=1, step_window=0)
    oracle = SeenRegistryOracle(ni, nu, neg, memory)
    g = torch.Generator().manual_seed(4)
    users = torch.randperm(nu, generator=g)[:500]
    items = torch.randperm(ni, generator=g)[:500]            # first batch: 500 distinct new items
    batches = [(users, items)]
    for _ in range(4):
        batches.append((torch.randperm(nu, generator=g)[:800], torch.randint(0, 600, (800,), generator=g)))
    want = 0
    for u, i in batches:
        want += u.numel() + int(oracle.batch(u.numpy(), i.numpy())[2].sum())
        m.step(u.int().to(dev), i.int().to(dev), torch.rand(u.numel(), device=dev))
    assert int(m.stats[1].item()) == want
    m.close()


def test_draws_are_uniform_over_the_domain(dev):
    from scipy.stats import chisquare

    reg = native.seen_registry(1000, dev)
    known = torch.randperm(1000, generator=torch.Generator().manual_seed(1))[:50].int().to(dev)
    native.neg_sample_seen(torch.arange(50, device=dev, dtype=torch.int32), known, torch.ones(50, device=dev), 1, reg)
    n, m_neg = 20000, 4
    pos = known[torch.randint(0, 50, (n,), device=dev)]
    ou, oi, _ = native.neg_sample_seen(torch.randint(0, 10**6, (n,), device=dev, dtype=torch.int32), pos,
                                       torch.ones(n, device=dev), m_neg, reg, seed=3, step=1)
    ou, oi = ou.view(n, -1)[:, 1:], oi.view(n, -1)[:, 1:]
    assert (ou >= 0).all()
    slot = {int(x): s for s, x in enumerate(known.tolist())}
    got = np.bincount([slot[int(x)] for x in oi.reshape(-1).tolist()], minlength=50)
    # rejection of the positive: every other domain item is equally likely
    hits = np.bincount([slot[int(x)] for x in pos.tolist()], minlength=50)
    expected = m_neg * (n - hits) / 49.0
    assert chisquare(got, expected).pvalue > 1e-3


def test_unigram_noise_follows_counts_to_the_power(dev):
    from scipy.stats import chisquare

    from fps_b200.models.w2v import DeviceSkipGram

    V = 64
    counts = np.random.default_rng(3).integers(1, 500, size=V).astype(np.float64)
    counts[[5, 17, 40]] = 0
    m = DeviceSkipGram(V, 8, negative=5, seed=2, noise_counts=counts, noise_power=0.75)
    n = 30000
    ctx = torch.randint(0, V, (n,), device=dev, dtype=torch.int32)
    ou, oi, orat = native.neg_sample_noise(torch.zeros(n, device=dev, dtype=torch.int32), ctx,
                                           torch.ones(n, device=dev), 5, m._noise_cdf, m._noise_last, seed=2, step=0)
    ou, oi = ou.view(n, 6)[:, 1:].reshape(-1), oi.view(n, 6)[:, 1:].reshape(-1)
    assert (ou >= 0).all() and (orat.view(n, 6)[:, 1:] == 0).all()
    got = np.bincount(oi.cpu().numpy(), minlength=V)
    assert got[[5, 17, 40]].sum() == 0
    w = counts ** 0.75
    w[counts == 0] = 0
    pos_hits = np.bincount(ctx.cpu().numpy(), minlength=V)
    # P(x | positive c) = w_x / (W - w_c) for x != c
    per_pos = w[None, :] / (w.sum() - w[:, None])
    np.fill_diagonal(per_pos, 0)
    expected = 5 * (pos_hits[:, None] * per_pos).sum(0)
    live = w > 0
    assert chisquare(got[live], expected[live] * got.sum() / expected[live].sum()).pvalue > 1e-3
    m.close()


@pytest.mark.parametrize("memory", [0, 16])
def test_same_seed_same_stream_same_records(dev, memory):
    """With a ring, each micro-batch holds a user once: the ring cursor of a user repeated inside a batch is
    taken in whatever order the warps reach it, as in fps_neg_sample.  Without one, users may repeat."""
    g = torch.Generator().manual_seed(8)
    users = (lambda: torch.randperm(5000, generator=g)[:3000]) if memory else \
        (lambda: torch.randint(0, 500, (3000,), generator=g))
    batches = [(users(), torch.randint(0, 900, (3000,), generator=g)) for _ in range(3)]
    outs = []
    for _ in range(2):
        reg = native.seen_registry(900, dev)
        seen = torch.full((5000, memory), -1, dtype=torch.int32, device=dev) if memory else None
        seen_pos = torch.zeros(5000, dtype=torch.int32, device=dev) if memory else None
        run = []
        for step, (u, i) in enumerate(batches):
            run.append(native.neg_sample_seen(u.to(dev), i.to(dev), torch.ones(3000, device=dev), 3, reg, seen,
                                              seen_pos, seed=77, step=step))
        outs.append(run)
    for a, b in zip(*outs):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def _clone_sampler_state(m):
    reg = tuple(t.clone() for t in m._registry)
    ring = (m.seen.clone(), m.seen_pos.clone()) if m.user_memory > 0 else (None, None)
    return reg, ring


def _mf_pointwise_reference(U, V, users, items, ratings, lr):
    keep = users >= 0
    users, items, ratings = users[keep].long(), items[keep].long(), ratings[keep]
    u, v = U[users], V[items]
    e = torch.sigmoid(ratings - (u * v).sum(1))[:, None]
    return U.clone().index_add_(0, users, lr * e * v), V.clone().index_add_(0, items, lr * e * u)


@pytest.mark.parametrize("memory", [0, 8])
def test_pointwise_seen_step_matches_fp32_reference(dev, memory):
    """Distinct users and positive items per batch.  A user's positive and negative records, and negatives
    shared between records, meet in one launch; with rows of +-0.01 and lr = 0.01 the order they are applied in
    moves the result by < 3e-7, so the reference applies every expanded record to the initial rows."""
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, k, lr = 3000, 4000, 16, 0.01
    m = DeviceOnlineMF(nu, ni, k, learning_rate=lr, negative_sample_rate=2, user_memory=memory,
                       negative_sampling="seen", seed=6)
    g = torch.Generator().manual_seed(5)
    for step in range(3):
        users = torch.randperm(nu, generator=g)[:1500].int().to(dev)
        items = torch.randperm(ni, generator=g)[:1500].int().to(dev)
        ratings = torch.rand(1500, generator=g).to(dev)
        U, V = m.users[:, :k].clone(), m.items.local[:ni, :k].clone()
        reg, (seen, seen_pos) = _clone_sampler_state(m)
        ou, oi, orat = native.neg_sample_seen(users, items, ratings, 2, reg, seen, seen_pos, m.world, seed=m.seed,
                                              step=m.step_no)
        m.step(users, items, ratings)
        torch.cuda.synchronize()
        U2, V2 = _mf_pointwise_reference(U, V, ou, oi, orat, lr)
        torch.testing.assert_close(m.users[:, :k], U2, rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(m.items.local[:ni, :k], V2, rtol=1e-4, atol=1e-6)
        if step:
            assert (ou.view(1500, 3)[:, 1:] >= 0).all()
    m.close()


def test_bpr_seen_step_matches_fp32_reference(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, k, lr = 3000, 4000, 16, 0.01
    m = DeviceOnlineMF(nu, ni, k, learning_rate=lr, negative_sample_rate=1, user_memory=8, negative_sampling="seen",
                       loss="bpr", seed=6)
    g = torch.Generator().manual_seed(7)
    triples = 0
    for step in range(3):
        users = torch.randperm(nu, generator=g)[:1500].int().to(dev)
        items = torch.randperm(ni, generator=g)[:1500].int().to(dev)
        ratings = torch.rand(1500, generator=g).to(dev) + 0.5
        U, V = m.users[:, :k].clone(), m.items.local[:ni, :k].clone()
        reg, (seen, seen_pos) = _clone_sampler_state(m)
        ou, oi, _ = native.neg_sample_seen(users, items, ratings, 1, reg, seen, seen_pos, m.world, seed=m.seed,
                                           step=m.step_no)
        m.step(users, items, ratings)
        torch.cuda.synchronize()
        ou, oi = ou.view(1500, 2), oi.view(1500, 2)
        keep = ou[:, 1] >= 0
        u, i, j = users[keep].long(), items[keep].long(), oi[keep, 1].long()
        uu, vi, vj = U[u], V[i], V[j]
        x = (uu * (vi - vj)).sum(1)
        gg = (lr * torch.sigmoid(-x))[:, None]
        U2 = U.clone().index_add_(0, u, gg * (vi - vj))
        V2 = V.clone().index_add_(0, i, gg * uu).index_add_(0, j, -gg * uu)
        torch.testing.assert_close(m.users[:, :k], U2, rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(m.items.local[:ni, :k], V2, rtol=1e-4, atol=1e-6)
        triples += int(keep.sum().item())
        assert int(m.stats[1].item()) == triples
    m.close()


def test_skipgram_unigram_step_matches_fp32_reference(dev):
    from fps_b200.models.w2v import DeviceSkipGram

    V, D, lr, neg = 4000, 300, 0.005, 5
    counts = np.random.default_rng(1).integers(1, 100, size=V).astype(np.float64)
    counts[::7] = 0
    m = DeviceSkipGram(V, D, learning_rate=lr, negative=neg, seed=1, noise_counts=counts)
    m.w_out.local.uniform_(-0.05, 0.05)
    Win, Wout = m.w_in.local[:V, :D].clone(), m.w_out.local[:V, :D].clone()
    c = torch.randperm(V, device=dev)[:500].int(); o = torch.randperm(V, device=dev)[:500].int()
    ec, eo, el = native.neg_sample_noise(c, o, torch.ones(500, device=dev), neg, m._noise_cdf, m._noise_last,
                                         seed=m.seed, step=m.step_no)
    m.step(c, o)
    torch.cuda.synchronize()
    assert (ec >= 0).all() and not np.isin(eo.view(500, -1)[:, 1:].cpu().numpy(), np.arange(0, V, 7)).any()
    ec, eo = ec.long(), eo.long()
    u, v = Win[ec], Wout[eo]
    g = (lr * (el - torch.sigmoid((u * v).sum(1))))[:, None]
    torch.testing.assert_close(m.w_in.local[:V, :D], Win.clone().index_add_(0, ec, g * v), rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(m.w_out.local[:V, :D], Wout.clone().index_add_(0, eo, g * u), rtol=1e-4, atol=1e-6)
    m.close()


@pytest.mark.parametrize("mode", ["seen", "uniform"])
def test_never_rated_item_rows_keep_their_init(dev, mode):
    """A stream that rates a quarter of the catalogue: with "seen" no negative reaches the other rows."""
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.models.mf.online import psOnlineMF

    nu, ni, k = 500, 2000, 8
    rng = np.random.default_rng(0)
    recs = [Rating(int(u), int(i), float(r)) for u, i, r in
            zip(rng.integers(0, nu, 20000), rng.integers(0, ni // 4, 20000) * 4, rng.random(20000))]
    rs = psOnlineMF(recs, numFactors=k, learningRate=0.05, negativeSampleRate=3, seed=3, backend="device",
                    numUsers=nu, numItems=ni, batch_size=4096, negativeSampling=mode)
    rated = np.zeros(ni, dtype=bool)
    rated[np.arange(0, ni, 4)] = True
    fresh = DeviceOnlineMF(nu, ni, k, seed=3)
    init = fresh.items.local[:ni, :k].cpu()
    got = rs.model.items.local[:ni, :k].cpu()
    never = torch.from_numpy(~rated)
    if mode == "seen":
        assert torch.equal(got[never], init[never])
        np.testing.assert_array_equal(np.sort(rs.model.seen_items().cpu().numpy()), np.arange(0, ni, 4))
    else:
        assert (got[never] != init[never]).any(dim=1).sum() > 100
    assert (got[~never] != init[~never]).any(dim=1).all()
    fresh.close()


def test_seen_sampling_refusals(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    with pytest.raises(ValueError, match="negative_sample_rate >= 1"):
        DeviceOnlineMF(10, 10, 4, negative_sampling="seen")
    with pytest.raises(ValueError, match="'uniform' or 'seen'"):
        DeviceOnlineMF(10, 10, 4, negative_sample_rate=1, negative_sampling="popular")
    m = DeviceOnlineMF(10, 10, 4, negative_sample_rate=1, negative_sampling="seen", loss="bpr")
    one = torch.ones(2, device=dev)
    ids = torch.tensor([1, 2], device=dev, dtype=torch.int32)
    with pytest.raises(ValueError, match="without negatives="):
        m.step(ids, ids, one, negatives=ids[:, None].contiguous())
    m.close()
    u = DeviceOnlineMF(10, 10, 4, negative_sample_rate=1)
    with pytest.raises(ValueError, match="negative_sampling='seen'"):
        u.seen_items()
    u.close()


@pytest.mark.timeout(900)                  # torchrun children: their own 420 s limit applies first
def test_multi_rank_seen_registry():
    from tests.test_gpu_multi import _run

    _run("mp_negative_check.py", 2, 29643, "MP_NEGATIVE_CHECK_OK")
