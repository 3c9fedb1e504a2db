"""Skip-gram from a token stream on the device: the subsample kernel against the numpy replay, the fused
center-window kernel against an fp32 oracle, what it leaves alone, its counters, that ``train_tokens`` never
synchronises with the host, the quality it reaches and the 2-rank check."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models import w2v_ref as R
from fps_b200.ops import native
from tests.philox_ref import philox4x32 as PH

pytestmark = pytest.mark.gpu


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("n", [1, 37, 256, 1000, 70000, 400000])
def test_subsample_matches_numpy_replay(dev, dtype, n):
    vocab = 500
    rng = np.random.default_rng(n)
    tok = rng.integers(0, vocab, size=n)
    tok[rng.random(n) < 0.05] = -1
    tok[rng.random(n) < 0.01] = vocab + 3                # invalid ids: boundaries, counted as dropped
    counts = np.bincount(tok[(tok >= 0) & (tok < vocab)], minlength=vocab).astype(np.float64) + 1.0
    p = R.keep_probabilities(counts ** 2, 1e-3)         # a skewed table: many words dropped
    ts = torch.zeros(4, dtype=torch.int64, device=dev)
    seq, pos, n_comp = native.w2v_subsample(torch.from_numpy(tok).to(dev, dtype), vocab,
                                            torch.from_numpy(p).to(dev), seed=5, step=3, token_stats=ts)
    rs, rp, kept, dropped = R.compact(tok, vocab, p, 3, 5, PH)
    m = int(n_comp.item())
    assert m == len(rs)
    assert np.array_equal(seq[:m].cpu().numpy(), rs) and np.array_equal(pos[:m].cpu().numpy(), rp)
    assert ts.tolist() == [n, kept, 0, dropped]
    assert kept == int(R.keep_mask(tok, p, 3, 5, PH).sum())


def _replay(tokens, vocab, window, neg, step, seed, cdf=None, last=0):
    """Per kept center: (center word, [[(word, label)] per context])."""
    seq, pos, _, _ = R.compact(tokens, vocab, None, step, seed, PH)
    out = []
    for e, ctx in R.windows(seq, pos, window, step, seed, PH):
        out.append((int(seq[e]), R.center_targets(int(pos[e]), seq[ctx], neg, vocab, step, seed, PH, cdf=cdf,
                                                  last_nonzero=last)))
    return out


def _collision_free_corpus(vocab, n_sent, neg, window, seed, cdf=None, last=0):
    """Two-word sentences of distinct words; sentences whose replayed W_out rows meet another center's are
    turned into boundaries until no row is read by two centers."""
    g = np.random.default_rng(seed)
    words = g.permutation(vocab)[: 2 * n_sent]
    tok = np.full(3 * n_sent, -1, dtype=np.int64)
    tok[0::3], tok[1::3] = words[0::2], words[1::2]
    while True:
        rep = _replay(tok, vocab, window, neg, 0, seed, cdf, last)
        readers = {}
        for c, tg in rep:
            for w in {t for ctx in tg for t, _ in ctx if t >= 0}:
                readers.setdefault(w, set()).add(c)
        shared = {w for w, cs in readers.items() if len(cs) > 1}
        bad = {c for c, tg in rep if any(t in shared for ctx in tg for t, _ in ctx)}
        if not bad:
            return tok, rep
        for s in range(n_sent):
            if tok[3 * s] in bad or tok[3 * s + 1] in bad:
                tok[3 * s:3 * s + 2] = -1


def _model(vocab, dim, neg, lr, noise=None, seed=4):
    from fps_b200.models.w2v import DeviceSkipGram

    m = DeviceSkipGram(vocab, dim, learning_rate=lr, negative=neg, seed=seed, noise_counts=noise, sample=0.0)
    m.w_out.local.uniform_(-0.05, 0.05)
    return m


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("dim", [32, 100, 300, 512])
def test_fused_kernel_matches_fp32_oracle(dev, dim, noise):
    vocab, neg, lr, window = 60000, 5, 0.05, 5
    counts = None
    if noise:
        counts = np.random.default_rng(2).integers(0, 50, size=vocab).astype(np.float64)
    m = _model(vocab, dim, neg, lr, counts)
    cdf = m._noise_cdf.cpu().numpy() if noise else None
    tok, rep = _collision_free_corpus(vocab, 200, neg, window, m.seed, cdf, m._noise_last)
    assert sum(len(ctx) for _, tg in rep for ctx in tg) > 1000   # targets left after the filter
    reads = [c for c, _ in rep] + [t for _, tg in rep for ctx in tg for t, _ in ctx]
    Win, Wout = m.w_in.local[:vocab, :dim].cpu().numpy(), m.w_out.local[:vocab, :dim].cpu().numpy()
    W_in, W_out = Win.copy(), Wout.copy()
    loss = 0.0
    for c, tg in rep:
        D, lsum = R.center_update(Win[c].copy(), W_out, tg, lr, block=R.target_block(dim))
        W_in[c] += D
        loss += lsum
    m.train_tokens(torch.from_numpy(tok).to(dev), window=window)
    torch.cuda.synchronize()
    got_in, got_out = m.w_in.local[:vocab, :dim].cpu().numpy(), m.w_out.local[:vocab, :dim].cpu().numpy()
    np.testing.assert_allclose(got_in, W_in, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got_out, W_out, rtol=1e-5, atol=1e-7)
    untouched = np.setdiff1d(np.arange(vocab), np.array(reads))
    assert np.array_equal(got_in[untouched], Win[untouched]) and np.array_equal(got_out[untouched], Wout[untouched])
    n_tgt = sum(t >= 0 for _, tg in rep for ctx in tg for t, _ in ctx)
    st, ts = m.stats.cpu(), m.token_stats.cpu()
    assert st[1].item() == n_tgt and abs(st[0].item() - loss) < 1e-4 * loss
    assert ts.tolist() == [len(tok), int((tok >= 0).sum()), sum(len(tg) for _, tg in rep), 0]
    assert int(m.nan_flag.item()) == 0
    m.close()


def test_multi_context_windows_match_sequential_reference(dev):
    """Sentences of 8 words and radii up to 4: a center's contexts read its earlier pushes.  Rows shared between
    centers are applied Hogwild-style; with rows of +-0.05 and lr = 0.002 the order moves a value by < 1e-6, so the
    reference applies the centers one after the other."""
    vocab, dim, neg, lr = 20000, 64, 3, 0.002
    m = _model(vocab, dim, neg, lr)
    g = np.random.default_rng(9)
    tok = np.full((300, 9), -1, dtype=np.int64)
    tok[:, :8] = g.permutation(vocab)[:2400].reshape(300, 8)
    tok = tok.reshape(-1)
    Win, W_out = m.w_in.local[:vocab, :dim].cpu().numpy(), m.w_out.local[:vocab, :dim].cpu().numpy()
    W_in = Win.copy()
    st = R.train_call(W_in, W_out, tok, lr=lr, window=4, negative_count=neg, step=0, seed=m.seed, philox=PH)
    m.train_tokens(torch.from_numpy(tok).to(dev), window=4)
    torch.cuda.synchronize()
    np.testing.assert_allclose(m.w_in.local[:vocab, :dim].cpu().numpy(), W_in, rtol=0, atol=1e-6)
    np.testing.assert_allclose(m.w_out.local[:vocab, :dim].cpu().numpy(), W_out, rtol=0, atol=1e-6)
    assert m.token_stats.tolist() == [st["tokens"], st["kept"], st["contexts"], st["dropped"]]
    assert m.stats[1].item() == st["targets"]
    m.close()


def test_same_seed_same_tables(dev):
    vocab, dim = 30000, 100
    tok, _ = _collision_free_corpus(vocab, 150, 5, 5, 4)
    out = []
    for _ in range(2):
        m = _model(vocab, dim, 5, 0.05)
        torch.manual_seed(0)
        m.w_out.local.uniform_(-0.05, 0.05)
        m.train_tokens(torch.from_numpy(tok).to(dev), window=5)
        out.append((m.w_in.local.clone(), m.w_out.local.clone()))
        m.close()
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def test_non_finite_dot_sets_nan_flag(dev):
    m = _model(1000, 32, 2, 0.05)
    m.w_out.local[:1000] = float("inf")
    m.train_tokens(torch.tensor([1, 2, 3, -1], device=dev), window=2)
    assert int(m.nan_flag.item()) == 1
    m.close()


def test_train_tokens_never_syncs_with_the_host(dev):
    from fps_b200.models.w2v import DeviceSkipGram

    vocab = 5000
    tok = torch.randint(-1, vocab, (100000,), device=dev)
    counts = torch.bincount(tok[tok >= 0], minlength=vocab).double()
    m = DeviceSkipGram(vocab, 64, negative=5, noise_counts=counts.cpu().numpy(), sample=1e-3)
    m.train_tokens(tok)                                  # first call: scratch allocation
    torch.cuda.synchronize()
    before = native.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            m.train_tokens(tok, window=5)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert native.launch_count() - before == 6
    assert m.step_no == 4
    ts = m.token_stats.cpu()
    assert ts[0].item() == 4 * 100000 and 0 < ts[1].item() < 4 * 100000 and ts[2].item() > 0
    m.close()


def test_model_refusals(dev):
    from fps_b200.models.w2v import DeviceSkipGram

    m = DeviceSkipGram(100, 8, optimizer="adagrad", sample=0.0)
    with pytest.raises(ValueError, match="optimizer='sgd'"):
        m.train_tokens(torch.zeros(4, dtype=torch.int64, device=dev))
    m.close()
    m = DeviceSkipGram(100, 8)
    with pytest.raises(ValueError, match="pass word_counts"):
        m.train_tokens(torch.zeros(4, dtype=torch.int64, device=dev))
    m.close()
    m = DeviceSkipGram(100, 8, sample=0.0)
    with pytest.raises(ValueError, match="window must be"):
        m.train_tokens(torch.zeros(4, dtype=torch.int64, device=dev), window=0)
    with pytest.raises(ValueError, match="int32 or int64"):
        m.train_tokens(torch.zeros(4, device=dev))
    m.close()


def test_quality_gate_through_fit_tokens(dev):
    from fps_b200.models.w2v import DeviceSkipGram
    from fps_b200.utils.synthetic import topic_corpus

    vocab, topics = 2000, 40
    tok = topic_corpus(vocab, topics, 10, 40000, seed=2)
    counts = np.bincount(tok[tok >= 0].numpy(), minlength=vocab).astype(np.float64)
    m = DeviceSkipGram(vocab, 64, learning_rate=0.025, negative=5, seed=3, word_counts=counts, noise_counts=counts,
                       sample=1e-3)
    m.fit_tokens(tok.pin_memory(), epochs=3, batch_tokens=1 << 17, window=5)
    m.check_finite()
    words = torch.arange(vocab, device=dev)
    _, ids = m.most_similar(words, 10)
    prec = float(((ids % topics) == (words % topics)[:, None]).float().mean())
    chance = (vocab / topics - 1) / (vocab - 1)
    print(f"w2v token quality: precision@10 {prec:.3f}, chance {chance:.3f}")
    assert prec > 0.9, (prec, chance)     # measured 1.000 on an H100
    m.close()


@pytest.mark.timeout(900)               # the torchrun children have their own 420 s limit
def test_multi_rank_train_tokens():
    from tests.test_gpu_multi import _run

    _run("mp_w2v_tokens_check.py", 2, 29647, "MP_W2V_TOKENS_CHECK_OK")
