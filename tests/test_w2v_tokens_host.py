"""Skip-gram from a token stream on the host: the numpy reference of ``DeviceSkipGram.train_tokens`` (keep
probabilities, Philox draws, compaction, windows, the center update), its quality on a topic corpus, and the
refusals."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models import w2v_ref as R
from fps_b200.models.w2v import check_sample, check_token_call, expected_records
from fps_b200.utils.synthetic import topic_corpus
from tests.philox_ref import philox4x32 as PH


def test_keep_probabilities_follow_word2vec_rule():
    c = np.array([0, 1, 10, 1000, 100000, 5], dtype=np.float64)
    s = 1e-3
    p = R.keep_probabilities(c, s)
    f = c / c.sum()
    for w in range(len(c)):
        want = 1.0 if c[w] == 0 else min(1.0, (np.sqrt(f[w] / s) + 1) * s / f[w])
        assert p[w] == want
    assert (R.keep_probabilities(c, 0.0) == 1).all()
    assert p[4] < 0.2 and p[1] == 1.0


def test_keep_draws_match_their_probability():
    n = 40000
    p = np.array([0.25, 1.0, 0.6])
    tokens = np.arange(n) % 3
    kept = R.keep_mask(tokens, p, step=3, seed=9, philox=PH)
    for w in range(3):
        frac = kept[tokens == w].mean()
        assert abs(frac - p[w]) < 4 * np.sqrt(p[w] * (1 - p[w]) / (n / 3)) + 1e-12
    # a 53-bit uniform keyed (i, 0, 0, step; seed)
    r = PH(np.uint32(7), np.uint32(0), np.uint32(0), np.uint32(3), 9, 0)
    u = (((int(r[0]) << 32) | int(r[1])) >> 11) * 2.0 ** -53
    assert kept[7] == (u < p[tokens[7]])


def test_window_radii_are_uniform():
    from scipy.stats import chisquare

    r = R.radii(np.arange(60000), 5, step=1, seed=4, philox=PH)
    assert r.min() == 1 and r.max() == 5
    assert chisquare(np.bincount(r, minlength=6)[1:]).pvalue > 1e-3


def test_windows_stop_at_boundaries_and_dropped_tokens_close_gaps():
    vocab = 10
    p = np.ones(vocab)
    p[3] = 0.0                                          # word 3 is never kept
    tokens = np.array([1, 3, 2, 4, -1, 5, 6, 77, 7, 3, 8])
    seq, pos, kept, dropped = R.compact(tokens, vocab, p, 0, 0, PH)
    assert seq.tolist() == [1, 2, 4, -1, 5, 6, -1, 7, 8]
    assert pos.tolist() == [0, 2, 3, 4, 5, 6, 7, 8, 10]
    assert kept == 7 and dropped == 1
    wins = dict(R.windows(seq, pos, 50, 0, 0, PH))    # radius >= every sentence: the whole sentence
    assert wins[0] == [1, 2] and wins[1] == [0, 2] and wins[4] == [5] and wins[7] == [8] and wins[8] == [7]
    assert 3 not in wins and 6 not in wins
    r = R.radii(pos, 2, 0, 0, PH)
    for e, ctx in R.windows(seq, pos, 2, 0, 0, PH):
        assert all(abs(q - e) <= r[e] for q in ctx) and ctx == sorted(ctx)


def test_invalid_ids_are_boundaries_and_counted():
    seq, pos, kept, dropped = R.compact(np.array([0, 12, -5, 1, -1, 2]), 10, None, 0, 0, PH)
    assert seq.tolist() == [0, -1, -1, 1, -1, 2] and kept == 3 and dropped == 2


def test_negatives_reject_the_context_word():
    cdf = np.cumsum([0.0, 5.0, 0.0, 1.0])                 # only words 1 and 3 can be drawn
    got = [R.negative(i, 0, 0, 1, 4, 0, 0, PH, cdf=cdf, last_nonzero=3) for i in range(200)]
    assert set(got) - {-1} == {3}
    assert R.negative(0, 0, 0, 0, 1, 0, 0, PH) == -1    # vocab of one: every draw is the context word
    u = [R.negative(i, 1, 2, 5, 7, 0, 0, PH) for i in range(300)]
    assert 5 not in u and set(u) == {0, 1, 2, 3, 4, 6}


def test_center_update_is_a_gradient_step():
    """One context: D and the W_out deltas are -lr times the gradient of the SGNS loss of its targets."""
    rng = np.random.default_rng(0)
    dim, lr = 7, 0.1
    u = rng.normal(size=dim)
    W = rng.normal(size=(5, dim)) * 0.5
    targets = [[(2, 1.0), (0, 0.0), (4, 0.0)]]

    def loss(u, W):
        return sum(np.logaddexp(0, -np.dot(u, W[t]) if lab else np.dot(u, W[t])) for t, lab in targets[0])

    W2 = W.copy()
    D, L = R.center_update(u.copy(), W2, targets, lr)
    assert np.isclose(L, loss(u, W))
    eps = 1e-6
    gu = np.array([(loss(u + eps * np.eye(dim)[k], W) - loss(u - eps * np.eye(dim)[k], W)) / (2 * eps)
                   for k in range(dim)])
    np.testing.assert_allclose(D, -lr * gu, rtol=1e-6, atol=1e-9)
    for t in (2, 0, 4):
        gv = np.array([(loss(u, W + eps * np.outer(np.eye(5)[t], np.eye(dim)[k])) -
                        loss(u, W - eps * np.outer(np.eye(5)[t], np.eye(dim)[k]))) / (2 * eps) for k in range(dim)])
        np.testing.assert_allclose(W2[t] - W[t], -lr * gv, rtol=1e-6, atol=1e-9)
    assert (W2[[1, 3]] == W[[1, 3]]).all()


def test_later_contexts_read_the_earlier_updates():
    rng = np.random.default_rng(1)
    u, W = rng.normal(size=4).astype(np.float32), rng.normal(size=(3, 4)).astype(np.float32)
    W2 = W.copy()
    D, _ = R.center_update(u, W2, [[(0, 1.0)], [(0, 1.0)]], 0.5)
    g1 = 0.5 * (1 - 1 / (1 + np.exp(-np.dot(u, W[0]))))
    v1 = W[0] + g1 * u
    w2 = u + g1 * W[0]
    g2 = 0.5 * (1 - 1 / (1 + np.exp(-np.dot(w2, v1))))
    np.testing.assert_allclose(D, g1 * W[0] + g2 * v1, rtol=1e-5)
    np.testing.assert_allclose(W2[0], v1 + g2 * w2, rtol=1e-5)


def _one_context_in_blocks(u, W, blocks, lr):
    """One context trained block by block: all rows of a block pulled, then each target's update."""
    e = np.zeros_like(u)
    for blk in blocks:
        vs = [W[t].copy() for t, _ in blk]
        for (t, label), v in zip(blk, vs):
            g = lr * (label - 1.0 / (1.0 + np.exp(-np.dot(u, v))))
            e += g * v
            W[t] += g * u
    return e


def test_void_draw_keeps_its_target_slot():
    """Blocks are made of target slots 0 .. negative: a voided draw keeps its slot, so the next block starts at
    slot 8 whether or not a draw before it was voided.  Sentence ``0 1`` of a 3-word vocabulary, one try per draw:
    the center 0 trains [1, 2, 2] and then [2, 2, 0, 0], not [1, 2, 2, 2, 2, 0, 0] in one block."""
    tg = R.center_targets(0, [1], 12, 3, step=0, seed=4, philox=PH, max_tries=1)
    assert tg == [[(1, 1.0)] + [(-1, 0.0)] * 5 + [(2, 0.0)] * 4 + [(-1, 0.0)] + [(0, 0.0)] * 2]
    rng = np.random.default_rng(3)
    u, W0 = rng.uniform(-0.5, 0.5, 8), rng.uniform(-0.5, 0.5, (3, 8))
    W = W0.copy()
    D, _ = R.center_update(u, W, tg, 0.1, block=8)
    by_slot = W0.copy()
    e = _one_context_in_blocks(u, by_slot, [[(1, 1.0), (2, 0.0), (2, 0.0)],
                                            [(2, 0.0), (2, 0.0), (0, 0.0), (0, 0.0)]], 0.1)
    np.testing.assert_allclose(W, by_slot, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(D, e, rtol=1e-13, atol=1e-15)
    compacted = W0.copy()
    e_c = _one_context_in_blocks(u, compacted, [[(1, 1.0)] + [(2, 0.0)] * 4 + [(0, 0.0)] * 2], 0.1)
    assert np.abs(compacted - W).max() > 1e-3 and np.abs(e_c - D).max() > 1e-3
    # counters leave the voids out
    w_in, w_out = rng.uniform(-0.5, 0.5, (3, 8)), rng.uniform(-0.5, 0.5, (3, 8))
    st = R.train_call(w_in, w_out, np.array([0, 1]), lr=0.1, window=1, negative_count=12, step=0, seed=4,
                      philox=PH, max_tries=1)
    tg1 = R.center_targets(1, [0], 12, 3, step=0, seed=4, philox=PH, max_tries=1)
    assert st["contexts"] == 2 and st["targets"] == 7 + sum(t >= 0 for t, _ in tg1[0])


def _replay_in_blocks(w_in, w_out, tokens, block, *, lr, neg, seed):
    seq, pos, _, _ = R.compact(tokens, len(w_in), None, 0, seed, PH)
    for e, ctx in R.windows(seq, pos, 1, 0, seed, PH):
        tg = R.center_targets(int(pos[e]), seq[ctx], neg, len(w_in), 0, seed, PH)
        D, _ = R.center_update(w_in[seq[e]].copy(), w_out, tg, lr, block)
        w_in[seq[e]] += D


@pytest.mark.parametrize("width,block", [(388, 6), (384, 8)])
def test_train_call_takes_the_target_block_from_the_row_width(width, block):
    """Rows over 384 floats are pulled 6 target slots at a time.  With seed 0, word 0 sits in slots 1, 2 and 6 of
    the center 0's targets: a block of 6 reads it in slot 6 with the earlier pushes applied, a block of 8 as it
    was before the block."""
    vocab, neg, lr, seed = 4, 7, 0.1, 0
    tokens = np.array([0, 1])
    assert [t for t, _ in R.center_targets(0, [1], neg, vocab, 0, seed, PH)[0]] == [1, 0, 0, 2, 3, 2, 0, 2]
    assert R.target_block(width) == block
    rng = np.random.default_rng(1)
    w_in, w_out = rng.uniform(-0.5, 0.5, (vocab, width)), rng.uniform(-0.5, 0.5, (vocab, width))
    got_in, got_out = w_in.copy(), w_out.copy()
    R.train_call(got_in, got_out, tokens, lr=lr, window=1, negative_count=neg, step=0, seed=seed, philox=PH)
    res = {}
    for b in (6, 8):
        a, o = w_in.copy(), w_out.copy()
        _replay_in_blocks(a, o, tokens, b, lr=lr, neg=neg, seed=seed)
        res[b] = a, o
    assert np.array_equal(got_in, res[block][0]) and np.array_equal(got_out, res[block][1])
    assert np.abs(res[6][1] - res[8][1]).max() > 1e-3 and np.abs(res[6][0] - res[8][0]).max() > 1e-3


def test_topic_corpus_is_seeded_and_topical():
    a, b = topic_corpus(100, 5, 8, 50, seed=3), topic_corpus(100, 5, 8, 50, seed=3)
    assert torch.equal(a, b) and a.dtype == torch.int64 and a.numel() == 50 * 9
    s = a.view(50, 9)
    assert (s[:, -1] == -1).all() and ((s[:, :-1] % 5) == (s[:, :1] % 5)).all()
    c = np.bincount(a[a >= 0].numpy(), minlength=100)
    assert c[:5].sum() > 5 * c[50:55].sum()               # Zipf: low ranks dominate


def _precision_at_10(W, topics):
    Wn = W / np.maximum(np.linalg.norm(W, axis=1, keepdims=True), 1e-30)
    S = Wn @ Wn.T
    np.fill_diagonal(S, -np.inf)
    nb = np.argsort(-S, axis=1)[:, :10]
    return float(((nb % topics) == (np.arange(len(W)) % topics)[:, None]).mean())


def test_numpy_quality_gate_on_topic_corpus():
    """Sequential numpy reference, 3 calls of ~3.6k tokens.  Measured precision@10: 0.90 (chance 0.076)."""
    vocab, topics, dim = 120, 12, 16
    tokens = topic_corpus(vocab, topics, 8, 1200, seed=5).numpy()
    counts = np.bincount(tokens[tokens >= 0], minlength=vocab).astype(np.float64)
    rng = np.random.default_rng(0)
    w_in = ((rng.random((vocab, dim)) - 0.5) / dim).astype(np.float32)
    w_out = np.zeros((vocab, dim), dtype=np.float32)
    p = R.keep_probabilities(counts, 1e-2)
    calls = np.array_split(tokens, 3)
    for step, t in enumerate(calls):
        st = R.train_call(w_in, w_out, t, lr=0.05, window=3, negative_count=4, step=step, seed=1, philox=PH, p=p)
        assert st["kept"] < (t >= 0).sum()             # subsampling dropped frequent words
    prec = _precision_at_10(w_in, topics)
    chance = (vocab / topics - 1) / (vocab - 1)
    assert prec > 0.7, (prec, chance)


def test_refusals_name_the_fix():
    t = torch.zeros(4, dtype=torch.int64)
    with pytest.raises(ValueError, match="optimizer='sgd'"):
        check_token_call(t, 5, "adagrad", 0.0, False)
    with pytest.raises(ValueError, match="window must be an integer >= 1"):
        check_token_call(t, 0, "sgd", 0.0, False)
    with pytest.raises(ValueError, match="pass word_counts"):
        check_token_call(t, 5, "sgd", 1e-3, False)
    for bad in (t.float(), t.numpy(), t.view(2, 2)):
        with pytest.raises(ValueError, match="int32 or int64"):
            check_token_call(bad, 5, "sgd", 0.0, True)
    check_token_call(t.int(), 5, "sgd", 1e-3, True)
    for s in (-1e-3, float("nan")):
        with pytest.raises(ValueError, match="sample must be a finite number >= 0"):
            check_sample(s)
    assert expected_records(1000, 5, 5) == 1000 * 6 * 6


def test_model_refuses_bad_sample_and_counts_before_allocating():
    from fps_b200.models.w2v import DeviceSkipGram

    with pytest.raises(ValueError, match="sample must be"):
        DeviceSkipGram(10, 8, sample=-1.0)
    with pytest.raises(ValueError, match="word_counts must hold one count per word"):
        DeviceSkipGram(10, 8, word_counts=np.ones(3))
