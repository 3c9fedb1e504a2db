"""Device top-K on rows wider than 128 floats (the K-streamed scoring kernel, up to 512): raw scores
against fp64, the top-K pipeline against torch.topk of the kernel's own scores, the device generators
at 128+ factors, and word2vec nearest-neighbour queries (``DeviceSkipGram.most_similar``)."""
import numpy as np
import pytest
import torch

from tests.test_gpu_topk_exclude import _assert_exact, _csr, _masked

pytestmark = pytest.mark.gpu

# 132..320 run 128 query rows per CTA, 324 and 512 run 64 (the resident query block must leave room
# for 3 item stages)
WIDE_STRIDES = [132, 160, 256, 300, 320, 324, 512]


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _same_items(sc, rows, ref):
    """Item sets agree wherever the scores are distinct (ties may come in any order)."""
    return ((rows == ref.indices) | (sc == torch.roll(sc, 1, 1)) | (sc == torch.roll(sc, -1, 1))).all()


@pytest.mark.parametrize("stride", WIDE_STRIDES)
@pytest.mark.parametrize("nq", [1, 63, 64, 65, 129, 517])
def test_wide_scores_match_fp64_matmul(dev, stride, nq):
    from fps_b200.models.mf.device_topk import DeviceTopK

    ni = 1000 + stride % 97                        # never a multiple of the 128-item tile
    g = torch.Generator(device="cpu").manual_seed(stride * 1000 + nq)
    items = torch.randn(ni, stride, generator=g).to(dev)
    q = torch.randn(nq, stride, generator=g).to(dev)
    got = DeviceTopK(items).scores(q_local=q)
    ref = q.double() @ items.double().T
    err = (got.double() - ref).abs().max().item()
    assert err < 2e-2 * (stride ** 0.5), err        # TF32: 10-bit mantissa inputs, fp32 accumulate
    assert torch.allclose(got.double(), ref, rtol=5e-3, atol=5e-2 * (stride / 128) ** 0.5)


@pytest.mark.parametrize("dim", [300, 512])
def test_wide_topk_pull_from_ps_equals_brute_force(dev, dim):
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.store.sharded_table import ShardedTable

    nu, ni, K = 3000, 20000 + 37, 100
    users = ShardedTable(nu, dim, seed=1, init_range=(-1.0, 1.0))
    g = torch.Generator(device="cpu").manual_seed(dim)
    scale = torch.rand(ni, 1, generator=g) * 2 + 0.1
    items = (torch.randn(ni, dim, generator=g) * scale).to(dev).contiguous()
    q_ids = torch.randint(0, nu, (517,), generator=g).to(dev)
    tk = DeviceTopK(items)
    sc, rows = tk.topk(K, q_ids=q_ids, q_table=users)
    full = tk.scores(q_ids=q_ids, q_table=users)            # same TF32 arithmetic
    ref = torch.topk(full, K, dim=1)
    assert torch.equal(sc, ref.values)
    assert _same_items(sc, rows, ref)
    assert tk.last_fallback_rows == 0
    # the queries pulled by the kernel are the table's rows
    torch.testing.assert_close(full, DeviceTopK(items).scores(q_local=users.pull(q_ids)), rtol=0, atol=0)
    users.close()


@pytest.mark.parametrize("stride", [300, 512])
def test_wide_topk_q_local_and_pass1_fraction(dev, stride):
    from fps_b200.models.mf.device_topk import DeviceTopK

    g = torch.Generator(device="cpu").manual_seed(5 + stride)
    ni = 70000 + 11                                          # >= 512 tiles: pass 1 defaults to 1/8 of them
    items = torch.randn(ni, stride, generator=g).to(dev)
    q = torch.randn(200, stride, generator=g).to(dev)
    full = DeviceTopK(items).scores(q_local=q)
    ref = torch.topk(full, 50, dim=1)
    for frac in (0.0, 0.125, 0.5):
        tk = DeviceTopK(items, pass1_fraction=frac)
        sc, rows = tk.topk(50, q_local=q)
        assert torch.equal(sc, ref.values), frac
        assert _same_items(sc, rows, ref), frac


@pytest.mark.parametrize("stride", [256, 300, 324])
def test_wide_length_sorted_pruning_is_exact_and_prunes(dev, stride):
    from fps_b200.models.mf.device_topk import DeviceTopK

    ni, K = 60000, 50
    g = torch.Generator(device="cpu").manual_seed(3)
    scale = torch.exp(torch.randn(ni, 1, generator=g) * 1.2)            # log-normal lengths
    items = (torch.randn(ni, stride, generator=g) * scale).to(dev).contiguous()
    q = torch.randn(300, stride, generator=g).to(dev)
    plain, pruned = DeviceTopK(items), DeviceTopK(items, sort_by_length=True)
    sc0, rows0 = plain.topk(K, q_local=q)
    sc1, rows1 = pruned.topk(K, q_local=q)
    p1, p2 = pruned.last_tiles_scored
    # the LENGTH bound loosens as the dimension grows (random directions score ~|q||i|/sqrt(dim)),
    # but a skewed table still loses its short tail
    assert p2 < 0.75 * pruned.n_tiles and p1 < pruned.n_tiles, (p1, p2, pruned.n_tiles)
    torch.testing.assert_close(sc1, sc0, rtol=0, atol=0)
    ref = torch.topk(plain.scores(q_local=q), K, dim=1)
    assert torch.equal(sc0, ref.values)
    assert _same_items(sc1, rows1, ref)


@pytest.mark.parametrize("stride", [132, 512])
def test_wide_k_larger_than_tiles(dev, stride):
    from fps_b200.models.mf.device_topk import DeviceTopK

    g = torch.Generator(device="cpu").manual_seed(stride)
    items = torch.randn(300, stride, generator=g).to(dev)              # 3 tiles, K = 50
    q = torch.randn(70, stride, generator=g).to(dev)
    tk = DeviceTopK(items)
    sc, rows = tk.topk(50, q_local=q)
    ref = torch.topk(tk.scores(q_local=q), 50, dim=1)
    assert torch.equal(sc, ref.values)
    assert _same_items(sc, rows, ref)


@pytest.mark.parametrize("stride,sort", [(300, False), (300, True), (512, False)])
def test_wide_exclude_matches_masked_brute_force(dev, stride, sort):
    from fps_b200.models.mf.device_topk import DeviceTopK

    ni, K = 30000, 20
    g = torch.Generator(device="cpu").manual_seed(21)
    scale = torch.exp(torch.randn(ni, 1, generator=g))
    items = (torch.randn(ni, stride, generator=g) * scale).to(dev).contiguous()
    q = torch.randn(150, stride, generator=g).to(dev)
    tk = DeviceTopK(items, sort_by_length=sort)
    full = tk.scores(q_local=q)
    rng = np.random.RandomState(4)
    top = torch.topk(full, 3 * K, dim=1).indices.cpu().numpy()
    lists = [rng.permutation(top[r]).tolist() if r % 2 == 0 else rng.randint(0, ni, 2 * K).tolist()
             for r in range(q.shape[0])]
    sc, rows = tk.topk(K, q_local=q, exclude=_csr(lists, dev))
    _assert_exact(sc, rows, _masked(full, lists), K)


def _model(rng, k, n_items, n_users):
    from fps_b200.api import Left, Right
    from fps_b200.models.mf.common import attachLength

    items = {i: rng.randn(k) * (0.5 + rng.rand()) for i in range(n_items)}
    users = {u: rng.randn(k) for u in range(0, n_users, 2)}            # odd users are unknown
    return [Left((i, attachLength(v))) for i, v in items.items()] + \
           [Right((u, attachLength(v))) for u, v in users.items()]


@pytest.mark.parametrize("k", [128, 200])
def test_ps_topk_generator_device_wide_factors(dev, k):
    """128 factors + the "loaded" column = stride 132: the K-streamed kernel serves the generator."""
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.topk import psTopKGenerator

    rng = np.random.RandomState(k)
    n_items, n_users = 300, 40
    model = _model(rng, k, n_items, n_users)
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
        assert len(set(i for _, i in topk) & set(i for _, i in want)) >= 9
        np.testing.assert_allclose([s for s, _ in topk], [s for s, _ in want], rtol=5e-3, atol=5e-3)


def test_online_learner_device_256_factors(dev):
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator

    rng = np.random.RandomState(1)
    ratings = [Rating(int(rng.randint(30)), int(rng.randint(50)), 1.0, t) for t in range(500)]
    out = psOnlineLearnerAndGenerator(ratings, numFactors=256, K=5, userMemory=0, backend="device",
                                      learningRate=0.1, rangeMin=0.01, rangeMax=0.05, batch_size=100,
                                      plain_residual=True)
    assert len(out) == 500 and all(len(t) == 5 for (_u, _i, _ts, t) in out)
    assert [(u, i, ts) for (u, i, ts, _t) in out] == [(r.user, r.item, r.timestamp) for r in ratings]
    u = torch.tensor([r.user for r in ratings[:100]], device=dev, dtype=torch.int32)
    i = torch.tensor([r.item for r in ratings[:100]], device=dev, dtype=torch.int32)
    # initial u.v is about 256 * 0.03^2 = 0.23; training moves it towards the rating 1
    assert out.model.predict(u, i).mean().item() > 0.45
    out.model.close()


def _cosine_topk(w, words, K):
    """fp32 brute force: cosine of every word against the vocabulary, the word itself masked."""
    wn = torch.nn.functional.normalize(w, dim=1)
    cos = wn[words] @ wn.T
    cos[torch.arange(words.numel(), device=w.device), words] = float("-inf")
    return cos, torch.topk(cos, K, dim=1)


def _check_neighbours(sg, words, K):
    sc, ids = sg.most_similar(words, K)
    assert sc.shape == ids.shape == (words.numel(), K)
    w = sg.w_in.pull(torch.arange(sg.vocab, device=words.device))
    cos, ref = _cosine_topk(w, words, K)
    assert (ids != words[:, None]).all()                                 # never the query word itself
    assert (ids >= 0).all() and (sc[:, :-1] >= sc[:, 1:]).all()
    exact = torch.gather(cos, 1, ids)                                    # fp32 cosine of what came back
    torch.testing.assert_close(sc, exact, rtol=0, atol=3e-3)             # TF32 scores of unit vectors
    # a valid top-K up to TF32 near-ties: nothing left out beats the K-th returned by more than that
    assert (ref.values[:, -1] <= exact[:, -1] + 6e-3).all()
    overlap = (ids[:, :, None] == ref.indices[:, None, :]).any(-1).float().mean().item()
    assert overlap > 0.9, overlap
    return ids


def test_most_similar_matches_cosine_brute_force_and_follows_training(dev):
    from fps_b200.models.w2v import DeviceSkipGram

    vocab, K = 6000, 10
    sg = DeviceSkipGram(vocab, dim=300, learning_rate=0.05, negative=5, seed=3)
    g = torch.Generator(device=dev).manual_seed(0)
    # correlated pairs (word w with w +- 1 .. 3): neighbourhoods become structured
    def train(steps):
        for _ in range(steps):
            c = torch.randint(0, vocab, (8192,), generator=g, device=dev, dtype=torch.int32)
            off = torch.randint(1, 4, (8192,), generator=g, device=dev, dtype=torch.int32)
            sg.step(c, (c + off) % vocab)
    train(20)
    words = torch.randint(0, vocab, (300,), generator=g, device=dev)
    words[:3] = torch.tensor([0, vocab - 1, 17], device=dev)
    ids1 = _check_neighbours(sg, words, K)
    ids1b = _check_neighbours(sg, words, K)                              # cached snapshot: same answer
    assert torch.equal(ids1, ids1b)
    train(40)                                                            # invalidates the snapshot
    ids2 = _check_neighbours(sg, words, K)
    assert not torch.equal(ids1, ids2)
    # int32 words, and K beyond the vocabulary: the lists end in (-3e38, -1)
    small = DeviceSkipGram(40, dim=300, seed=1)
    sc, ids = small.most_similar(torch.arange(5, device=dev, dtype=torch.int32), K=45)
    assert ids.shape == (5, 45) and (ids[:, :39] >= 0).all() and (ids[:, 39:] == -1).all() and (sc[:, 39:] < -1e38).all()
    for r in range(5):
        assert sorted(ids[r, :39].tolist()) == [i for i in range(40) if i != r]
    small.close()
    sg.close()


@pytest.mark.timeout(900)               # the torchrun children have their own 420 s limit
def test_multi_rank_most_similar():
    from tests.test_gpu_multi import _run

    _run("mp_w2v_neighbours_check.py", 2, 29633, "MP_W2V_NEIGHBOURS_CHECK_OK")
