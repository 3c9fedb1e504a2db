"""Row-wise AdaGrad on the device (``optimizer="adagrad"``): the fused pointwise, skip-gram and BPR kernels against
a torch fp32 oracle of the rule in ``models/mf/common.py::rowwise_adagrad``, what they leave alone, checkpoints,
refusals, quality over a learning-rate grid and the 2-rank direct mode."""
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import native
from tests import bpr_quality as Q

pytestmark = pytest.mark.gpu

EPS = 1e-8


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _model(nu, ni, k, lr, **kw):
    from fps_b200.models.mf.device import DeviceOnlineMF

    kw.setdefault("range_min", -0.5)
    kw.setdefault("range_max", 0.5)
    return DeviceOnlineMF(nu, ni, k, learning_rate=lr, seed=5, optimizer="adagrad", step_window=0, **kw)


def _apply(T, G, rows, delta, lr, k):
    """The rule for distinct rows: s = |delta|^2 / k, T[row] += lr * delta / (sqrt(G + s) + eps), G += s."""
    s = (delta * delta).sum(1) / k
    T = T.clone().index_add_(0, rows, lr * delta / (torch.sqrt(G[rows] + s) + EPS)[:, None])
    return T, G.clone().index_add_(0, rows, s)


def _pointwise_oracle(U, V, Gu, Gv, users, items, ratings, lr, k, err_mode):
    u, v = U[users], V[items]
    d = (u * v).sum(1)
    resid = ratings - d
    e = (torch.sigmoid(resid) if err_mode == 0 else resid)[:, None]
    U2, Gu2 = _apply(U, Gu, users, e * v, lr, k)
    V2, Gv2 = _apply(V, Gv, items, e * u, lr, k)
    return U2, V2, Gu2, Gv2, (resid * resid).sum()


def _ratings(U, V, users, items, gen):
    """Ratings whose residual against the current rows is at least 0.1 away from 0.  Near e = 0 the step
    lr * e * v / (|e| |v| / sqrt(k) + eps) turns on the last bits of e, which a different summation order of
    u.v changes, so an fp32 oracle could not be held to 1e-5 there."""
    d = (U[users] * V[items]).sum(1)
    n = users.numel()
    sign = torch.where(torch.rand(n, generator=gen, device=d.device) < 0.5, -1.0, 1.0)
    return d + sign * (0.1 + torch.rand(n, generator=gen, device=d.device))


def _state(m, k):
    gu, gv = m.accumulators
    return m.users[:, :k].clone(), m.items.local[:, :k].clone(), gu.clone(), gv.clone()


def _check(m, k, want):
    U2, V2, Gu2, Gv2 = want
    gu, gv = m.accumulators
    torch.testing.assert_close(m.users[:, :k], U2, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(m.items.local[:, :k], V2, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(gu, Gu2, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(gv, Gv2, rtol=1e-5, atol=1e-6)


def _step(m, users, items, ratings, fmt):
    if fmt == "packed64":
        m.step(native.pack_ratings(users, items, ratings))
    else:
        idt = torch.int32 if fmt == "int32" else torch.int64
        m.step(users.to(idt), items.to(idt), ratings)


@pytest.mark.parametrize("err_mode", [0, 1])
@pytest.mark.parametrize("fmt", ["int32", "int64", "packed64"])
@pytest.mark.parametrize("k", [10, 64, 128, 300])
def test_pointwise_conflict_free_matches_oracle(dev, k, fmt, err_mode):
    nu, ni, b, lr = 6000, 9000, 4000, 0.05
    m = _model(nu, ni, k, lr, err_mode=err_mode)
    U, V, Gu, Gv = _state(m, k)
    gen = torch.Generator(device=dev).manual_seed(k)
    users = torch.randperm(nu, generator=gen, device=dev)[:b]
    items = torch.randperm(ni, generator=gen, device=dev)[:b]
    ratings = _ratings(U, V, users, items, gen)
    if fmt == "packed64":      # the record holds the rating as fp16
        ratings = ratings.half().float()
    _step(m, users, items, ratings, fmt)
    torch.cuda.synchronize()
    *want, sq = _pointwise_oracle(U, V, Gu, Gv, users, items, ratings, lr, k, err_mode)
    _check(m, k, want)
    s = m.stats.cpu()
    assert s[1].item() == b
    assert abs(s[0].item() - sq.item()) / sq.item() < 1e-4
    m.check_finite()
    m.close()


def test_accumulators_compound_over_steps(dev):
    """Two steps over the same rows: the second step is scaled by the G the first one left."""
    nu, ni, k, b, lr = 3000, 3000, 64, 2000, 0.1
    m = _model(nu, ni, k, lr, err_mode=1)
    U, V, Gu, Gv = _state(m, k)
    gen = torch.Generator(device=dev).manual_seed(2)
    users = torch.randperm(nu, generator=gen, device=dev)[:b]
    items = torch.randperm(ni, generator=gen, device=dev)[:b]
    for t in range(2):
        ratings = _ratings(U, V, users, items, gen)
        _step(m, users, items, ratings, "int32")
        U, V, Gu, Gv, _ = _pointwise_oracle(U, V, Gu, Gv, users, items, ratings, lr, k, 1)
    torch.cuda.synchronize()
    assert Gu[users].min() > 0
    _check(m, k, (U, V, Gu, Gv))
    m.close()


def _bpr_oracle(U, V, Gu, Gv, users, items, negs, lr, reg, k):
    u, vi, vj = U[users], V[items], V[negs]
    x = (u * (vi - vj)).sum(1)
    g = torch.sigmoid(-x)[:, None]
    U2, Gu2 = _apply(U, Gu, users, g * (vi - vj) - reg * u, lr, k)
    V2, Gv2 = _apply(V, Gv, items, g * u - reg * vi, lr, k)
    V2, Gv2 = _apply(V2, Gv2, negs, -g * u - reg * vj, lr, k)
    return U2, V2, Gu2, Gv2


@pytest.mark.parametrize("reg", [0.0, 0.01])
@pytest.mark.parametrize("k", [10, 64, 128])
def test_bpr_conflict_free_matches_oracle(dev, k, reg):
    nu, ni, b, lr = 6000, 9000, 4000, 0.05
    m = _model(nu, ni, k, lr, loss="bpr", regularization=reg)
    U, V, Gu, Gv = _state(m, k)
    users = torch.randperm(nu, device=dev)[:b]
    ij = torch.randperm(ni, device=dev)[:2 * b]
    items, negs = ij[:b], ij[b:]
    m.step(users.int(), items.int(), torch.ones(b, device=dev), negatives=negs.int()[:, None].contiguous())
    torch.cuda.synchronize()
    _check(m, k, _bpr_oracle(U, V, Gu, Gv, users, items, negs, lr, reg, k))
    assert m.stats[1].item() == b
    m.check_finite()
    m.close()


@pytest.mark.parametrize("user_memory", [0, 8])
def test_bpr_sampled_touches_exactly_its_rows(dev, user_memory):
    nu, ni, k, b = 4000, 500, 32, 1000
    m = _model(nu, ni, k, 0.1, loss="bpr", negative_sample_rate=3, user_memory=user_memory)
    users = torch.randperm(nu, device=dev)[:b].int()
    items = torch.randint(0, ni, (b,), device=dev, dtype=torch.int32)
    V0 = m.items.local[:ni, :k].clone()
    for _ in range(3):
        m.step(users, items, torch.ones(b, device=dev))
    torch.cuda.synchronize()
    gu, gv = m.accumulators
    assert torch.isfinite(m.users).all() and torch.isfinite(m.items.local).all()
    touched_u = torch.zeros(gu.numel(), dtype=torch.bool, device=dev)
    touched_u[users.long()] = True
    assert (gu[touched_u] > 0).all() and (gu[~touched_u] == 0).all()
    moved = (m.items.local[:ni, :k] != V0).any(1)          # every item row updated: positives and negatives
    assert ((gv[:ni] > 0) == moved).all()
    assert moved[items.long()].all()
    m.check_finite()
    m.close()


def test_skipgram_matches_oracle_and_trains(dev):
    from fps_b200.models.w2v import DeviceSkipGram

    vocab, dim, b, lr = 5000, 100, 2000, 0.05
    sg = DeviceSkipGram(vocab, dim, learning_rate=lr, negative=0, optimizer="adagrad")
    W_in, W_out = sg.w_in.local[:vocab, :dim].clone(), sg.w_out.local[:vocab, :dim].clone()
    W_out.uniform_(-0.1, 0.1)
    sg.w_out.local[:vocab, :dim] = W_out           # non-zero W_out, so both tables move
    G = torch.zeros(vocab, device=dev)
    ids = torch.randperm(vocab, device=dev)[:2 * b]
    c, x = ids[:b], ids[b:]
    sg.step(c.int(), x.int())
    torch.cuda.synchronize()
    u, v = W_in[c], W_out[x]
    e = (1.0 - torch.sigmoid((u * v).sum(1)))[:, None]
    want_in, g_in = _apply(W_in, G, c, e * v, lr, dim)
    want_out, g_out = _apply(W_out, G, x, e * u, lr, dim)
    torch.testing.assert_close(sg.w_in.local[:vocab, :dim], want_in, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(sg.w_out.local[:vocab, :dim], want_out, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(sg.acc_in.local[:vocab], g_in, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(sg.acc_out.local[:vocab], g_out, rtol=1e-5, atol=1e-6)
    sg.close()

    sg = DeviceSkipGram(vocab, dim, learning_rate=0.05, negative=5, optimizer="adagrad")
    g = torch.Generator(device=dev).manual_seed(1)
    centers = torch.randint(0, vocab, (4096,), generator=g, device=dev, dtype=torch.int32)
    contexts = (centers + 1) % vocab
    losses = []                        # -log sigmoid(W_in[c] . W_out[x]) of the positive pairs
    for _ in range(20):
        losses.append(float(-torch.log(sg.score(centers.long(), contexts.long())).mean()))
        sg.step(centers, contexts)
    losses.append(float(-torch.log(sg.score(centers.long(), contexts.long())).mean()))
    sg.check_finite()
    assert all(l == l for l in losses) and losses[-1] < 0.9 * losses[0], losses
    sg.close()


def test_rows_outside_the_batch_unchanged_and_sgd_allocates_nothing(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, k, b = 5000, 5000, 64, 1000
    m = _model(nu, ni, k, 0.1)
    U0, V0 = m.users.clone(), m.items.local.clone()
    users = torch.randperm(nu, device=dev)[:b]
    items = torch.randperm(ni, device=dev)[:b]
    m.step(users.int(), items.int(), torch.rand(b, device=dev))
    torch.cuda.synchronize()
    gu, gv = m.accumulators
    ou = torch.ones(m.users.shape[0], dtype=torch.bool, device=dev); ou[users] = False
    oi = torch.ones(m.items.local.shape[0], dtype=torch.bool, device=dev); oi[items] = False
    assert torch.equal(m.users[ou], U0[ou]) and torch.equal(m.items.local[oi], V0[oi])
    assert (gu[ou] == 0).all() and (gv[oi] == 0).all()
    assert torch.equal(m.users[:, k:], U0[:, k:])        # the padding columns stay zero
    m.close()
    s = DeviceOnlineMF(nu, ni, k)
    assert s.accumulators is None and s._user_acc is None and s._item_acc is None
    s.close()


def test_save_load_resumes_bitwise(dev, tmp_path):
    nu, ni, k, b = 4000, 3000, 64, 1500
    g = torch.Generator(device=dev).manual_seed(3)
    batches = [(torch.randperm(nu, generator=g, device=dev)[:b].int(),
                torch.randperm(ni, generator=g, device=dev)[:b].int(),
                torch.rand(b, generator=g, device=dev)) for _ in range(3)]
    a = _model(nu, ni, k, 0.05)
    for bt in batches[:2]:
        a.step(*bt)
    a.save(str(tmp_path))
    a.step(*batches[2])
    torch.cuda.synchronize()
    c = _model(nu, ni, k, 0.05)
    c.load(str(tmp_path))
    c.step(*batches[2])
    torch.cuda.synchronize()
    assert torch.equal(a.users, c.users) and torch.equal(a.items.local, c.items.local)
    assert all(torch.equal(x, y) for x, y in zip(a.accumulators, c.accumulators))
    a.close(); c.close()


def test_checkpoint_without_accumulators_loads_zeros(dev, tmp_path):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, k = 1000, 800, 16
    s = DeviceOnlineMF(nu, ni, k, seed=5)
    s.step(torch.arange(100, device=dev, dtype=torch.int32), torch.arange(100, device=dev, dtype=torch.int32),
           torch.ones(100, device=dev))
    s.save(str(tmp_path))
    m = _model(nu, ni, k, 0.05)
    m.step(torch.arange(100, device=dev, dtype=torch.int32), torch.arange(100, device=dev, dtype=torch.int32),
           torch.ones(100, device=dev))
    m.load(str(tmp_path))
    gu, gv = m.accumulators
    assert (gu == 0).all() and (gv == 0).all()
    assert torch.equal(m.users[:, :k], s.users[:, :k])
    s.close(); m.close()


@pytest.mark.parametrize("kw, fix", [
    (dict(output_ring=object()), "output_ring=None"),
    (dict(kernel="tma"), "kernel=None"),
    (dict(item_cache=True), "item_cache=False"),
])
def test_refusals(dev, kw, fix):
    from fps_b200.models.mf.device import DeviceOnlineMF

    with pytest.raises(ValueError, match=fix):
        DeviceOnlineMF(100, 100, 8, optimizer="adagrad", **kw)


def test_refusals_unknown_and_skipgram_replica(dev):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.models.w2v import DeviceSkipGram

    with pytest.raises(ValueError, match="'sgd' or 'adagrad'"):
        DeviceOnlineMF(100, 100, 8, optimizer="adam")
    with pytest.raises(ValueError, match="replica_cache=False"):
        DeviceSkipGram(100, 8, optimizer="adagrad", replica_cache=True)
    with pytest.raises(ValueError, match="'sgd' or 'adagrad'"):
        DeviceSkipGram(100, 8, optimizer="adam")


def test_ps_online_mf_device_adagrad(dev):
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.online import psOnlineMF

    recs = [Rating(u, (7 * u) % 50, 1.0) for u in range(200)]
    out = psOnlineMF(recs, numFactors=8, learningRate=0.1, backend="device", optimizer="adagrad")
    gu, gv = out.model.accumulators
    assert (gu[:200] > 0).all() and (gv[:50] > 0).all()
    out.model.close()


# ---- quality over a learning-rate grid ------------------------------------------------------------------
LR_GRID = [0.02, 0.1, 0.4]            # 20x


def _pointwise_rmse(opt, lr, dev):
    from fps_b200.models.mf.device import DeviceOnlineMF, ERR_PLAIN
    from fps_b200.utils.synthetic import lowrank_ratings

    nu, ni, k, batch, steps = 20000, 5000, 16, 1 << 15, 600        # ~1000 updates per user
    m = DeviceOnlineMF(nu, ni, k, range_min=-0.05, range_max=0.05, learning_rate=lr, seed=1, err_mode=ERR_PLAIN,
                       optimizer=opt, step_window=0)
    gh = torch.Generator(device=dev).manual_seed(99991)
    hu = torch.randint(0, nu, (1 << 18,), generator=gh, device=dev, dtype=torch.int32)
    hi = torch.randint(0, ni, (1 << 18,), generator=gh, device=dev, dtype=torch.int32)
    hr = lowrank_ratings(hu, hi)
    untrained = float(((hr - m.predict(hu, hi)) ** 2).mean().sqrt())
    for s in range(steps):
        g = torch.Generator(device=dev).manual_seed(7919 * s + 1)
        u = torch.randint(0, nu, (batch,), generator=g, device=dev, dtype=torch.int32)
        i = torch.randint(0, ni, (batch,), generator=g, device=dev, dtype=torch.int32)
        m.step(u, i, lowrank_ratings(u, i))
    rmse = float(((hr - m.predict(hu, hi)) ** 2).mean().sqrt())
    m.close()
    return rmse, untrained


def test_quality_pointwise_lr_grid(dev):
    res = {opt: [_pointwise_rmse(opt, lr, dev) for lr in LR_GRID] for opt in ("sgd", "adagrad")}
    print("\nADAGRAD_QUALITY pointwise held-out RMSE (lr: sgd / adagrad, untrained):")
    for j, lr in enumerate(LR_GRID):
        print(f"  lr={lr}: {res['sgd'][j][0]:.4f} / {res['adagrad'][j][0]:.4f}, {res['adagrad'][j][1]:.4f}")
    for rmse, untrained in res["adagrad"]:
        assert rmse == rmse and rmse < 0.95 * untrained, res      # finite, and it has learned


def _bpr_quality(opt, lr, dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    tu, ti, eu, ei = Q.data()
    m = DeviceOnlineMF(Q.NUM_USERS, Q.NUM_ITEMS, Q.K, range_min=-Q.INIT, range_max=Q.INIT, learning_rate=lr,
                       negative_sample_rate=1, seed=1, loss="bpr", regularization=Q.REG, optimizer=opt)
    before = Q.metrics(m.users[:, :Q.K], m.items.local[:Q.NUM_ITEMS, :Q.K], (tu, ti), (eu, ei))
    u, i = tu.int().to(dev), ti.int().to(dev)
    perm = torch.Generator().manual_seed(0)
    for _ in range(Q.EPOCHS):
        p = torch.randperm(u.numel(), generator=perm).to(dev)
        for a in range(0, u.numel(), 128):
            sel = p[a:a + 128]
            m.step(u[sel], i[sel], torch.ones(sel.numel(), device=dev))
    torch.cuda.synchronize()
    m.check_finite()
    after = Q.metrics(m.users[:, :Q.K], m.items.local[:Q.NUM_ITEMS, :Q.K], (tu, ti), (eu, ei))
    m.close()
    return after, before


def test_quality_bpr_lr(dev):
    res = {(opt, lr): _bpr_quality(opt, lr, dev) for opt in ("sgd", "adagrad") for lr in (0.05, 0.2)}
    print("\nADAGRAD_QUALITY bpr held-out (auc, recall@10) [untrained]:")
    for (opt, lr), (after, before) in res.items():
        print(f"  {opt} lr={lr}: auc={after[0]:.3f} recall@10={after[1]:.3f} [auc {before[0]:.3f}]")
    for lr in (0.05, 0.2):
        (auc, _), (auc0, _) = res[("adagrad", lr)]
        assert auc == auc and auc > auc0 + 0.05, res


def test_multi_rank_direct_adagrad():
    from tests.test_gpu_multi import _run

    _run("mp_adagrad_check.py", 2, 29641, "MP_ADAGRAD_CHECK_OK")
