"""CBOW from a token stream on the host: the numpy reference of ``DeviceSkipGram.train_tokens(cbow=True)``
(``models/w2v_ref.py``: the mean of the context rows, the center's targets, the unscaled error pushed to every
context), its counters, its quality on a topic corpus, and the refusals."""
import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models import w2v_ref as R
from fps_b200.models.w2v import check_token_call, expected_records
from fps_b200.ops import native
from fps_b200.utils.synthetic import topic_corpus
from tests.philox_ref import philox4x32 as PH


def _sgns_loss(h, W, targets):
    return sum(np.logaddexp(0, -np.dot(h, W[t]) if lab else np.dot(h, W[t])) for t, lab in targets if t >= 0)


def test_cbow_update_moves_contexts_by_cw_times_the_gradient():
    """word2vec.c's rule, kept on purpose: the W_out deltas are -lr times the gradient of the SGNS loss of h, and
    every context row moves by e = -lr times the gradient with respect to h, which is -lr * cw times the gradient
    with respect to that row (mean in, unscaled error out), not -lr times it."""
    rng = np.random.default_rng(0)
    dim, lr = 7, 0.1
    W_in, W = rng.normal(size=(6, dim)), rng.normal(size=(5, dim)) * 0.5
    ctx = [0, 3, 5]
    targets = [(2, 1.0), (0, 0.0), (4, 0.0)]
    h = W_in[ctx].mean(axis=0)
    a, b = W_in.copy(), W.copy()
    e, L = R.cbow_update(a, b, ctx, targets, lr, block=8)
    assert np.isclose(L, _sgns_loss(h, W, targets))
    eps = 1e-6
    eye = np.eye(dim)
    gh = np.array([(_sgns_loss(h + eps * eye[k], W, targets) - _sgns_loss(h - eps * eye[k], W, targets)) / (2 * eps)
                   for k in range(dim)])
    np.testing.assert_allclose(e, -lr * gh, rtol=1e-6, atol=1e-9)
    def loss_of_rows(X):
        return _sgns_loss(X[ctx].mean(axis=0), W, targets)

    for c in ctx:
        gx = np.array([(loss_of_rows(W_in + eps * np.outer(np.eye(6)[c], eye[k])) -
                        loss_of_rows(W_in - eps * np.outer(np.eye(6)[c], eye[k]))) / (2 * eps) for k in range(dim)])
        np.testing.assert_allclose(gx * len(ctx), gh, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(a[c] - W_in[c], -lr * len(ctx) * gx, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(a[c] - W_in[c], e, rtol=1e-12, atol=1e-15)
    for t in (2, 0, 4):
        gv = np.array([(_sgns_loss(h, W + eps * np.outer(np.eye(5)[t], eye[k]), targets) -
                        _sgns_loss(h, W - eps * np.outer(np.eye(5)[t], eye[k]), targets)) / (2 * eps)
                       for k in range(dim)])
        np.testing.assert_allclose(b[t] - W[t], -lr * gv, rtol=1e-6, atol=1e-9)
    assert (a[[1, 2, 4]] == W_in[[1, 2, 4]]).all() and (b[[1, 3]] == W[[1, 3]]).all()


def test_h_is_the_mean_and_a_repeated_context_counts_twice():
    rng = np.random.default_rng(1)
    W_in, W = rng.normal(size=(6, 5)), rng.normal(size=(6, 5))
    a, b = W_in.copy(), W.copy()
    e, _ = R.cbow_update(a, b, [2, 5, 2], [(1, 1.0), (4, 0.0)], 0.2)
    h = (2 * W_in[2] + W_in[5]) / 3
    g1 = 0.2 * (1 - 1 / (1 + np.exp(-np.dot(h, W[1]))))
    g4 = 0.2 * (0 - 1 / (1 + np.exp(-np.dot(h, W[4]))))
    np.testing.assert_allclose(e, g1 * W[1] + g4 * W[4], rtol=1e-12)
    np.testing.assert_allclose(b[1], W[1] + g1 * h, rtol=1e-12)
    np.testing.assert_allclose(b[4], W[4] + g4 * h, rtol=1e-12)
    np.testing.assert_allclose(a[2], W_in[2] + 2 * e, rtol=1e-12)    # pushed once per occurrence
    np.testing.assert_allclose(a[5], W_in[5] + e, rtol=1e-12)
    assert (a[[0, 1, 3, 4]] == W_in[[0, 1, 3, 4]]).all()


def test_negatives_are_keyed_on_slot_0_and_reject_the_center_word():
    """Sentence ``0 1`` of a 2-word vocabulary: the noise words of center 0 are drawn from the counters of context
    slot 0 and may be its context word 1, never the center word 0; a draw that keeps hitting 0 is void."""
    vocab, neg = 2, 20
    tg = R.center_targets(0, [0], neg, vocab, 0, 4, PH)[0]
    assert tg[0] == (0, 1.0) and {t for t, _ in tg[1:]} <= {1, -1} and (1, 0.0) in tg[1:]
    assert [t for t, _ in tg[1:]] == [R.negative(0, 0, j, 0, vocab, 0, 4, PH) for j in range(neg)]
    rng = np.random.default_rng(2)
    w_in, w_out = rng.uniform(-0.5, 0.5, (vocab, 8)), rng.uniform(-0.5, 0.5, (vocab, 8))
    a, b = w_in.copy(), w_out.copy()
    st = R.train_call(a, b, np.array([0, 1]), lr=0.1, window=1, negative_count=neg, step=0, seed=4, philox=PH,
                      cbow=True)
    a2, b2 = w_in.copy(), w_out.copy()
    tg1 = R.center_targets(1, [1], neg, vocab, 0, 4, PH)[0]
    R.cbow_update(a2, b2, [1], tg, 0.1)
    R.cbow_update(a2, b2, [0], tg1, 0.1)
    assert np.array_equal(a, a2) and np.array_equal(b, b2)
    assert st["targets"] == sum(t >= 0 for t, _ in tg + tg1) and st["contexts"] == 2
    # skip-gram rejects the context word instead: the same counters give different words
    sg = R.center_targets(0, [1], neg, vocab, 0, 4, PH)[0]
    assert {t for t, _ in sg[1:]} <= {0, -1}


def test_void_draw_keeps_its_target_slot():
    """The slot list of the skip-gram void test, trained on h: blocks are slots 0-7 and 8-12 whatever was voided."""
    tg = [(1, 1.0)] + [(-1, 0.0)] * 5 + [(2, 0.0)] * 4 + [(-1, 0.0)] + [(0, 0.0)] * 2
    rng = np.random.default_rng(3)
    W_in, W0 = rng.uniform(-0.5, 0.5, (4, 8)), rng.uniform(-0.5, 0.5, (3, 8))
    h = (W_in[0] + W_in[3]) / 2

    def blocked(blocks):
        W, e = W0.copy(), np.zeros(8)
        for blk in blocks:
            vs = [W[t].copy() for t, _ in blk]
            for (t, label), v in zip(blk, vs):
                g = 0.1 * (label - 1.0 / (1.0 + np.exp(-np.dot(h, v))))
                e += g * v
                W[t] += g * h
        return W, e

    a, b = W_in.copy(), W0.copy()
    e, _ = R.cbow_update(a, b, [0, 3], tg, 0.1, block=8)
    W, e_slot = blocked([[(1, 1.0), (2, 0.0), (2, 0.0)], [(2, 0.0), (2, 0.0), (0, 0.0), (0, 0.0)]])
    np.testing.assert_allclose(b, W, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(e, e_slot, rtol=1e-13, atol=1e-15)
    Wc, ec = blocked([[(1, 1.0)] + [(2, 0.0)] * 4 + [(0, 0.0)] * 2])
    assert np.abs(Wc - b).max() > 1e-4 and np.abs(ec - e).max() > 1e-4


def test_centers_without_contexts_train_and_count_nothing():
    rng = np.random.default_rng(4)
    w_in, w_out = rng.uniform(-0.5, 0.5, (10, 8)), rng.uniform(-0.5, 0.5, (10, 8))
    a, b = w_in.copy(), w_out.copy()
    st = R.train_call(a, b, np.array([5, -1, 7, -1, 12, 3]), lr=0.1, window=5, negative_count=5, step=0, seed=1,
                      philox=PH, cbow=True)
    assert np.array_equal(a, w_in) and np.array_equal(b, w_out)
    assert st == dict(tokens=6, kept=3, contexts=0, dropped=1, loss=0.0, targets=0)
    e, loss = R.cbow_update(a, b, [], [(5, 1.0)], 0.1)
    assert not e.any() and loss == 0.0 and np.array_equal(a, w_in) and np.array_equal(b, w_out)


def test_train_call_counters():
    vocab, neg, window, seed = 50, 3, 3, 6
    tok = np.random.default_rng(5).integers(-1, vocab + 2, size=300)
    tok[100:103] = tok[200:203] = [-1, 9, -1]             # one-word sentences
    rng = np.random.default_rng(6)
    w_in, w_out = rng.uniform(-0.1, 0.1, (vocab, 12)), rng.uniform(-0.1, 0.1, (vocab, 12))
    st = R.train_call(w_in.copy(), w_out.copy(), tok, lr=0.05, window=window, negative_count=neg, step=2,
                      seed=seed, philox=PH, cbow=True, max_tries=1)
    seq, pos, kept, dropped = R.compact(tok, vocab, None, 2, seed, PH)
    wins = R.windows(seq, pos, window, 2, seed, PH)
    live = [(e, c) for e, c in wins if c]
    n_tgt = sum(t >= 0 for e, _ in live
                for t, _ in R.center_targets(int(pos[e]), [seq[e]], neg, vocab, 2, seed, PH, max_tries=1)[0])
    assert len(live) < len(wins)                         # some kept words have no context
    assert st["tokens"] == 300 and st["kept"] == kept and st["dropped"] == dropped > 0
    assert st["contexts"] == sum(len(c) for _, c in wins) and st["targets"] == n_tgt < len(live) * (1 + neg)
    assert st["loss"] > 0


def test_reverse_order_replay_applies_the_same_centers():
    vocab = 30
    tok = np.random.default_rng(7).integers(0, vocab, size=40)
    rng = np.random.default_rng(8)
    w_in, w_out = rng.uniform(-0.5, 0.5, (vocab, 8)), rng.uniform(-0.5, 0.5, (vocab, 8))
    f = R.train_call(w_in.copy(), w_out.copy(), tok, lr=0.1, window=3, negative_count=2, step=0, seed=1,
                     philox=PH, cbow=True)
    r = R.train_call(w_in.copy(), w_out.copy(), tok, lr=0.1, window=3, negative_count=2, step=0, seed=1,
                     philox=PH, cbow=True, order="reverse")
    assert {k: f[k] for k in ("tokens", "kept", "contexts", "dropped", "targets")} == \
        {k: r[k] for k in ("tokens", "kept", "contexts", "dropped", "targets")}


def test_expected_records():
    assert expected_records(1000, 5, 5, cbow=True) == 1000 * ((1 + 5) + (5 + 1))
    assert expected_records(1000, 5, 5) == expected_records(1000, 5, 5, cbow=False) == 1000 * 6 * 6
    assert expected_records(0, 5, 5, cbow=True) == 1


def test_refusals_name_the_fix():
    t = torch.zeros(4, dtype=torch.int64)
    for bad in (1, 0, "yes", None, np.bool_(True)):
        with pytest.raises(ValueError, match="cbow must be True"):
            check_token_call(t, 5, "sgd", 0.0, True, bad)
    with pytest.raises(ValueError, match="optimizer='sgd'"):
        check_token_call(t, 5, "adagrad", 0.0, True, True)
    with pytest.raises(ValueError, match="window must be an integer >= 1"):
        check_token_call(t, 0, "sgd", 0.0, True, True)
    with pytest.raises(ValueError, match="pass word_counts"):
        check_token_call(t, 5, "sgd", 1e-3, False, True)
    with pytest.raises(ValueError, match="int32 or int64"):
        check_token_call(t.float(), 5, "sgd", 0.0, True, True)
    check_token_call(t, 5, "sgd", 1e-3, True, True)
    with pytest.raises(ValueError, match="cbow must be True or False"):   # refused before any argument is read
        native.w2v_window_fused(None, None, None, None, None, 0.1, vocab=1, cbow=1)


def _precision_at_10(W, topics):
    Wn = W / np.maximum(np.linalg.norm(W, axis=1, keepdims=True), 1e-30)
    S = Wn @ Wn.T
    np.fill_diagonal(S, -np.inf)
    nb = np.argsort(-S, axis=1)[:, :10]
    return float(((nb % topics) == (np.arange(len(W)) % topics)[:, None]).mean())


def test_numpy_quality_gate_on_topic_corpus():
    """The skip-gram gate's corpus and schedule, trained with CBOW at word2vec.c's CBOW rate 0.05.  Measured
    precision@10: 0.897 (chance 0.076)."""
    vocab, topics, dim = 120, 12, 16
    tokens = topic_corpus(vocab, topics, 8, 1200, seed=5).numpy()
    counts = np.bincount(tokens[tokens >= 0], minlength=vocab).astype(np.float64)
    rng = np.random.default_rng(0)
    w_in = ((rng.random((vocab, dim)) - 0.5) / dim).astype(np.float32)
    w_out = np.zeros((vocab, dim), dtype=np.float32)
    p = R.keep_probabilities(counts, 1e-2)
    for step, t in enumerate(np.array_split(tokens, 3)):
        st = R.train_call(w_in, w_out, t, lr=0.05, window=3, negative_count=4, step=step, seed=1, philox=PH, p=p,
                          cbow=True)
        assert st["kept"] < (t >= 0).sum() and st["targets"] > 0
    prec = _precision_at_10(w_in, topics)
    chance = (vocab / topics - 1) / (vocab - 1)
    print(f"cbow numpy quality: precision@10 {prec:.3f}, chance {chance:.3f}")
    assert prec > 0.7, (prec, chance)
