"""The fused CBOW kernel (``fps_w2v_cbow_kernel``, ``train_tokens(cbow=True)``) against the fp64 replay of
``models/w2v_ref.py``, every Philox draw replayed by ``tests/philox_ref.py``: every dispatch rung and noise path,
the mean over up to ``2 * window`` contexts, repeated and voided rows, a realistic corpus, grid-stride rounds, the
ends of a call, the counters, no host sync, the quality it reaches and the 2-rank check."""
import functools

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models import w2v_ref as R
from fps_b200.ops import native
from tests.philox_ref import philox4x32 as PH

pytestmark = pytest.mark.gpu

SEED = 4

# The dispatch ladder is the skip-gram kernel's (tests/test_gpu_w2v_window_edges.py): dim -> (LPR, VPL, TB).
RUNGS = {3: (1, 1, 8), 4: (1, 1, 8), 8: (2, 1, 8), 13: (4, 1, 8), 16: (4, 1, 8), 24: (8, 1, 8), 36: (16, 1, 8),
         100: (32, 1, 8), 136: (32, 2, 8), 256: (32, 2, 8), 300: (32, 3, 8), 387: (32, 4, 6), 388: (32, 4, 6),
         512: (32, 4, 6)}
SWEEP = [(dim, neg) for dim, (lpr, _, _) in RUNGS.items() for neg in sorted({0, 1, lpr, lpr + 1, 7, 8, 20})]

# The fp32 kernel against the fp64 replay: the tolerance of the skip-gram edge tests.
RTOL, ATOL_OF_MAX = 2e-5, 1e-5


def _close(got, want, what):
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=ATOL_OF_MAX * float(np.abs(want).max()), err_msg=what)


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def test_sweep_reaches_every_rung_and_noise_path():
    assert {RUNGS[d][:2] for d, _ in SWEEP} == {(1, 1), (2, 1), (4, 1), (8, 1), (16, 1), (32, 1), (32, 2), (32, 3),
                                               (32, 4)}
    paths = {("shuffled" if n <= RUNGS[d][0] else "serial", "one block" if 1 + n <= RUNGS[d][2] else "several")
             for d, n in SWEEP}
    assert paths == {(a, b) for a in ("shuffled", "serial") for b in ("one block", "several")}


def _tables(vocab, dim, scale, seed, dev):
    """W_in and W_out ``[vocab, stride]`` fp32, uniform on +-scale, padding columns 0."""
    g = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for _ in range(2):
        t = torch.zeros(vocab, (dim + 3) // 4 * 4, device=dev)
        t[:, :dim] = (torch.rand(vocab, dim, generator=g, device=dev) * 2 - 1) * scale
        out.append(t)
    return out


def _fused(W_in, W_out, dim, tokens, vocab, *, lr, window, neg, step=0, max_tries=32, cdf=None, last=0,
           keep_p=None, reserve=0):
    """One CBOW call through native.w2v_subsample + native.w2v_window_fused(cbow=True); returns (stats,
    token_stats, nan_flag)."""
    dev = W_in.device
    st = torch.zeros(2, dtype=torch.float32, device=dev)
    ts = torch.zeros(4, dtype=torch.int64, device=dev)
    nan = torch.zeros(1, dtype=torch.int32, device=dev)
    seq, pos, n_comp = native.w2v_subsample(tokens, vocab, keep_p, seed=SEED, step=step, token_stats=ts)
    native.w2v_window_fused(seq, pos, n_comp, native.local_table(W_in, dim), native.local_table(W_out, dim), lr,
                            window=window, negative=neg, vocab=vocab, seed=SEED, step=step, cdf=cdf,
                            last_nonzero=last, max_tries=max_tries, stats=st, token_stats=ts, nan_flag=nan,
                            reserve_total=reserve, cbow=True)
    torch.cuda.synchronize()
    return st.cpu(), ts.cpu(), int(nan.item())


def _plan(tok, vocab, window, neg, step=0, **noise):
    seq, pos, _, _ = R.compact(tok, vocab, None, step, SEED, PH)
    return R.cbow_centers(seq, pos, window, neg, vocab, step, SEED, PH, **noise)


def _replay(W_in, W_out, dim, plan, lr, order=None):
    """The fp64 replay of ``plan`` (:func:`R.cbow_centers`) on the rows it touches: (rows_in, w_in, rows_out,
    w_out, loss), the rows sorted by word."""
    rin = sorted({c for ctx, _ in plan for c in ctx})
    rout = sorted({t for _, tg in plan for t, _ in tg if t >= 0})
    ai, ao = {w: k for k, w in enumerate(rin)}, {w: k for k, w in enumerate(rout)}
    w_in = W_in[rin, :dim].double().cpu().numpy()
    w_out = W_out[rout, :dim].double().cpu().numpy()
    loss = 0.0
    for ctx, tg in (plan[::-1] if order == "reverse" else plan):
        _, lsum = R.cbow_update(w_in, w_out, [ai[c] for c in ctx], [(ao[t] if t >= 0 else -1, lab) for t, lab in tg],
                                lr, R.target_block(dim))
        loss += lsum
    return rin, w_in, rout, w_out, loss


def _untouched_equal(got, before, rows, vocab):
    keep = torch.ones(vocab, dtype=torch.bool, device=got.device)
    keep[list(rows)] = False
    return torch.equal(got[:vocab][keep], before[:vocab][keep])


# ---- every rung x every noise path: sentences `x y`, no row read by two centers --------------------------------

VOCAB = 100_000


@functools.lru_cache(maxsize=None)
def _noise(kind):
    """(counts, cdf, last_nonzero) of the unigram noise: 30% of the words and the last 1000 have weight 0."""
    if kind == "uniform":
        return None, None, 0
    g = np.random.default_rng(11)
    c = g.integers(1, 50, size=VOCAB).astype(np.float64)
    c[g.random(VOCAB) < 0.3] = 0.0
    c[-1000:] = 0.0
    cdf = native.noise_cdf(torch.from_numpy(c).cuda(), 0.75).cpu().numpy()
    return c, cdf, int(np.flatnonzero(c)[-1])


@functools.lru_cache(maxsize=None)
def _pair_corpus(neg, kind, n_sent=16):
    """Sentences ``x y -1`` whose centers pull pairwise disjoint W_out rows.  The center x reads only W_in[y], which
    only x pushes to (after its pull), so nothing depends on the order the lane-groups run in.  A candidate
    sentence that would read a row another center reads is replaced by a boundary."""
    _, cdf, last = _noise(kind)
    words = iter(np.random.default_rng(100 + neg).permutation(VOCAB).tolist())
    tok, used, n_ok = [], set(), 0
    while n_ok < n_sent:
        x, y = next(words), next(words)
        i = len(tok)
        tx = R.center_targets(i, [x], neg, VOCAB, 0, SEED, PH, cdf=cdf, last_nonzero=last)[0]
        ty = R.center_targets(i + 1, [y], neg, VOCAB, 0, SEED, PH, cdf=cdf, last_nonzero=last)[0]
        rx, ry = {t for t, _ in tx}, {t for t, _ in ty}
        if rx & ry or (rx | ry) & used or -1 in rx | ry or len(rx) + len(ry) < len(tx) + len(ty):
            tok.append(-1)
            continue
        used |= rx | ry
        tok += [x, y, -1]
        n_ok += 1
    return np.array(tok, dtype=np.int64)


@pytest.mark.parametrize("noise", ["uniform", "unigram"])
@pytest.mark.parametrize("dim,neg", SWEEP)
def test_cbow_kernel_matches_fp64_replay_at_every_rung(dev, dim, neg, noise):
    from fps_b200.models.w2v import DeviceSkipGram

    lr = 0.1
    counts, cdf, last = _noise(noise)
    tok = _pair_corpus(neg, noise)
    plan = _plan(tok, VOCAB, 5, neg, cdf=cdf, last_nonzero=last)
    m = DeviceSkipGram(VOCAB, dim, learning_rate=lr, negative=neg, seed=SEED, noise_counts=counts, sample=0.0)
    try:
        W_in, W_out = _tables(VOCAB, dim, dim ** -0.25, dim + neg, dev)
        m.w_in.local.copy_(W_in)
        m.w_out.local.copy_(W_out)
        rin, w_in, rout, w_out, loss = _replay(W_in, W_out, dim, plan, lr)
        m.train_tokens(torch.from_numpy(tok).to(dev), window=5, cbow=True)
        torch.cuda.synchronize()
        got_in, got_out = m.w_in.local, m.w_out.local
        _close(got_in[rin, :dim].cpu().numpy(), w_in, "W_in")
        _close(got_out[rout, :dim].cpu().numpy(), w_out, "W_out")
        assert _untouched_equal(got_in, W_in, rin, VOCAB) and _untouched_equal(got_out, W_out, rout, VOCAB)
        assert not got_in[:, dim:].any() and not got_out[:, dim:].any()
        n_centers = int((tok >= 0).sum())
        assert len(plan) == n_centers and len(rout) == n_centers * (1 + neg)
        st, ts = m.stats.cpu(), m.token_stats.cpu()
        assert st[1].item() == n_centers * (1 + neg)
        assert abs(st[0].item() - loss) <= 1e-5 * loss
        assert ts.tolist() == [len(tok), n_centers, n_centers, 0]
        assert int(m.nan_flag.item()) == 0
    finally:
        m.close()


# ---- the mean over up to 2 * window contexts, exactly ----------------------------------------------------------

def _long_corpus(neg, window, sent_len, n_sent, seed):
    """Sentences of ``sent_len`` distinct words; every W_out row is a target of at most one center (sentences that
    would break this become boundaries).  Returns (tokens, plan, designated) where ``designated`` holds, per
    sentence, the index into ``plan`` of its center with the most contexts."""
    words = iter(np.random.default_rng(seed).permutation(VOCAB).tolist())
    tok, used, chosen = [], set(), []
    while len(chosen) < n_sent:
        sent = [next(words) for _ in range(sent_len)]
        cand = tok + sent + [-1]
        plan = _plan(np.array(cand), VOCAB, window, neg)
        new = plan[len(_plan(np.array(tok), VOCAB, window, neg)) if tok else 0:]
        rows = [t for _, tg in new for t, _ in tg]
        if -1 in rows or len(set(rows)) < len(rows) or set(rows) & used:
            tok.append(-1)
            continue
        used |= set(rows)
        start = len(plan) - len(new)
        chosen.append(start + max(range(len(new)), key=lambda k: len(new[k][0])))
        tok = cand
    return np.array(tok, dtype=np.int64), _plan(np.array(tok), VOCAB, window, neg), chosen


@pytest.mark.parametrize("dim,neg", [(4, 5), (36, 5), (100, 8), (300, 5), (512, 7)])
def test_mean_over_many_contexts_matches_replay_exactly(dev, dim, neg):
    """Only the designated center of each sentence has non-zero W_out rows.  Every other center reads zero rows,
    so its e is 0 exactly and it pushes zeros to W_in: the final W_in and the designated centers' target rows do not
    depend on the order.  The other centers push g h with g = lr (label - 1/2) whatever h is, and h sees the
    designated center's push to a shared context row or not, so their W_out rows lie between the replay run
    forward and the replay run backward."""
    window, lr = 5, 0.1
    tok, plan, chosen = _long_corpus(neg, window, 14, 6, dim + neg)
    assert max(len(plan[k][0]) for k in chosen) == 2 * window
    W_in, _ = _tables(VOCAB, dim, 0.5, dim, dev)
    W_out = torch.zeros_like(W_in)
    hot = sorted({t for k in chosen for t, _ in plan[k][1]})
    W_out[hot, :dim] = (torch.rand(len(hot), dim, device=dev) * 2 - 1) * 0.5
    rin, w_in, rout, w_out, loss = _replay(W_in, W_out, dim, plan, lr)
    _, w_in_r, _, w_out_r, _ = _replay(W_in, W_out, dim, plan, lr, order="reverse")
    np.testing.assert_allclose(w_in_r, w_in, rtol=1e-12, atol=1e-15)
    a, b = W_in.clone(), W_out.clone()
    st, ts, nan = _fused(a, b, dim, torch.from_numpy(tok).to(dev), VOCAB, lr=lr, window=window, neg=neg)
    _close(a[rin, :dim].cpu().numpy(), w_in, "W_in")
    got_out = b[rout, :dim].cpu().numpy()
    is_hot = np.isin(rout, hot)
    _close(got_out[is_hot], w_out[is_hot], "designated W_out")
    lo, hi = np.minimum(w_out, w_out_r)[~is_hot], np.maximum(w_out, w_out_r)[~is_hot]
    tol = RTOL * np.abs(hi) + ATOL_OF_MAX * float(np.abs(w_out).max())
    assert ((got_out[~is_hot] >= lo - tol) & (got_out[~is_hot] <= hi + tol)).all(), "other W_out"
    assert _untouched_equal(a, W_in, rin, VOCAB) and _untouched_equal(b, W_out, rout, VOCAB)
    n_ctx = sum(len(c) for c, _ in plan)
    assert st[1].item() == len(plan) * (1 + neg) and abs(st[0].item() - loss) <= 1e-5 * loss
    assert ts.tolist() == [len(tok), int((tok >= 0).sum()), n_ctx, 0] and nan == 0


# ---- voided and repeated targets: one sentence `x y` per call on a tiny vocabulary ------------------------------

@pytest.mark.parametrize("noise", ["uniform", "on the center"])
@pytest.mark.parametrize("max_tries", [1, 2])
@pytest.mark.parametrize("dim,neg", [(16, 12), (100, 12), (512, 12), (4, 255), (512, 255)])
def test_void_and_repeated_targets_match_fp64_replay(dev, dim, neg, max_tries, noise):
    """With W_in[y] = 0 the center x has h = 0 (only x pushes to W_in[y], after its pull), so it pushes g * 0 to
    every W_out row: W_out and W_in[x] = the center y's update do not depend on the order.  W_in[y] = e of x reads
    rows y pushes to, before or after; it is held to the bound that leaves."""
    lr = 0.1
    if noise == "uniform":
        vocab, x, y, cdf, last = 3, 0, 1, None, 0
    else:   # words 0 and 4 have weight 0; 12 / 14 of the draws are word 3, the center y
        vocab, x, y, last = 5, 1, 3, 3
        cdf = np.cumsum([0.0, 1.0, 1.0, 12.0, 0.0])
    cdf_d = torch.from_numpy(cdf).to(dev) if cdf is not None else None
    tokens = torch.tensor([x, y], device=dev)
    noise_kw = dict(cdf=cdf, last_nonzero=last, max_tries=max_tries)
    seen = set()
    for step in range(2 if neg == 255 else 6):
        W_in, W_out = _tables(vocab, dim, 0.5, step, dev)
        W_in[y] = 0.0
        in0 = W_in.cpu().numpy()
        w_in, w_out = W_in[:, :dim].double().cpu().numpy(), W_out[:, :dim].double().cpu().numpy()
        h_y = w_in[x].copy()
        want = R.train_call(w_in, w_out, [x, y], lr=lr, window=5, negative_count=neg, step=step, seed=SEED,
                            philox=PH, cbow=True, **noise_kw)
        st, ts, nan = _fused(W_in, W_out, dim, tokens, vocab, lr=lr, window=5, neg=neg, step=step,
                             max_tries=max_tries, cdf=cdf_d, last=last)
        got_in, got_out = W_in.cpu().numpy(), W_out.cpu().numpy()
        _close(got_out[:, :dim], w_out, f"W_out, step {step}")
        _close(got_in[x, :dim], w_in[x], f"W_in[x], step {step}")
        sx = [t for t, _ in R.center_targets(0, [x], neg, vocab, step, SEED, PH, **noise_kw)[0]]
        sy = [t for t, _ in R.center_targets(1, [y], neg, vocab, step, SEED, PH, **noise_kw)[0]]
        assert x not in sx[1:] and y not in sy[1:]
        bound = 0.5 * lr * lr * np.abs(h_y) * sum(sy.count(t) for t in sx if t >= 0)
        tol = bound + RTOL * np.abs(w_in[y]) + ATOL_OF_MAX * np.abs(w_in[y]).max()
        assert (np.abs(got_in[y, :dim] - w_in[y]) <= tol).all(), f"W_in[y], step {step}"
        others = [w for w in range(vocab) if w not in (x, y)]
        assert np.array_equal(got_in[others], in0[others])
        assert not got_in[:, dim:].any() and not got_out[:, dim:].any()
        assert st[1].item() == want["targets"] == sum(t >= 0 for t in sx + sy)
        assert abs(st[0].item() - want["loss"]) <= 1e-5 * want["loss"]
        assert ts.tolist() == [2, 2, 2, 0] and want["contexts"] == 2 and nan == 0
        tb = RUNGS[dim][2]
        live = [[t for t in sy[b:b + tb] if t >= 0] for b in range(0, len(sy), tb)]
        if any(len(b) != len(set(b)) for b in live):
            seen.add("repeat inside a block")
        if any(set(a) & set(b) for k, a in enumerate(live) for b in live[k + 1:]):
            seen.add("repeat in a later block")
        if any(-1 in sy[b:b + tb] for b in range(0, len(sy) - tb, tb)):
            seen.add("void before a block boundary")
    assert seen == {"repeat inside a block", "repeat in a later block", "void before a block boundary"}


# ---- repeated context words and a context equal to the center word ---------------------------------------------

def _order_tolerance(W_in, W_out, dim, plan, lr, factor):
    """(forward replay, tolerance): ``factor`` times the largest difference between the replay run forward and run
    backward, plus the fp32 tolerance."""
    fwd = _replay(W_in, W_out, dim, plan, lr)
    rev = _replay(W_in, W_out, dim, plan, lr, order="reverse")
    spread = max(np.abs(fwd[1] - rev[1]).max(), np.abs(fwd[3] - rev[3]).max())
    scale = max(np.abs(fwd[1]).max(), np.abs(fwd[3]).max())
    return fwd, factor * spread + ATOL_OF_MAX * scale


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_repeated_context_and_context_equal_to_center(dev, dtype):
    """Sentences ``a b a c`` and ``d d`` of fresh words, radius up to 3: b has the context a twice, the first a has
    itself as a context, d's only context is d.  The centers of one sentence share rows, applied Hogwild-style;
    lr = 2e-3 keeps the order's effect (bounded by 4x the forward/backward spread of the replay) far below that of
    pushing a repeated context once, or of h summed rather than averaged."""
    vocab, dim, neg, lr, window = 50000, 64, 3, 2e-3, 3
    words = np.random.default_rng(21).permutation(vocab)
    tok = []
    for s in range(60):
        a, b, c, d = words[4 * s:4 * s + 4]
        tok += [a, b, a, c, -1, d, d, -1]
    tok = np.array(tok, dtype=np.int64)
    plan = _plan(tok, vocab, window, neg)
    assert any(ctx.count(ctx[0]) > 1 for ctx, _ in plan)
    W_in, W_out = _tables(vocab, dim, 0.5, 3, dev)
    (rin, w_in, rout, w_out, loss), tol = _order_tolerance(W_in, W_out, dim, plan, lr, 4.0)
    a_, b_ = W_in.clone(), W_out.clone()
    st, ts, nan = _fused(a_, b_, dim, torch.from_numpy(tok).to(dtype).to(dev), vocab, lr=lr, window=window, neg=neg)
    gi, go = a_[rin, :dim].cpu().numpy(), b_[rout, :dim].cpu().numpy()
    assert np.abs(gi - w_in).max() <= tol and np.abs(go - w_out).max() <= tol
    # the effect of a wrong update is far above the tolerance
    once = [(sorted(set(c)), tg) for c, tg in plan]
    _, w_in_once, _, _, _ = _replay(W_in, W_out, dim, once, lr)
    assert np.abs(w_in_once - w_in).max() > 20 * tol
    # the loss reads rows the other centers of the sentence push: held to 2e-3 (5e-4 measured on an H100)
    assert st[1].item() == sum(t >= 0 for _, tg in plan for t, _ in tg) and abs(st[0].item() - loss) <= 2e-3 * loss
    assert ts.tolist() == [len(tok), int((tok >= 0).sum()), sum(len(c) for c, _ in plan), 0] and nan == 0


# ---- a realistic corpus ----------------------------------------------------------------------------------------

def test_topic_corpus_call_matches_sequential_replay(dev):
    """One call of a Zipf topic corpus with unigram noise, subsampling and radii up to 5, where frequent words are
    read and pushed by many centers at once.  The tolerance is 4x the largest difference between the replay run
    forward and backward (plus the fp32 tolerance); it stays at least 20x below the effect of e divided by cw
    (about 50x in the numpy replay at lr = 0.002)."""
    from fps_b200.utils.synthetic import topic_corpus

    vocab, dim, neg, lr, window = 2000, 64, 5, 0.002, 5
    tok = topic_corpus(vocab, 40, 10, 300, seed=3).numpy()
    counts = np.bincount(tok[tok >= 0], minlength=vocab).astype(np.float64)
    cdf = native.noise_cdf(torch.from_numpy(counts).to(dev), 0.75)
    last = int(np.flatnonzero(counts)[-1])
    p = R.keep_probabilities(counts, 1e-3)
    seq, pos, kept, dropped = R.compact(tok, vocab, p, 0, SEED, PH)
    plan = R.cbow_centers(seq, pos, window, neg, vocab, 0, SEED, PH, cdf=cdf.cpu().numpy(), last_nonzero=last)
    assert kept < (tok >= 0).sum()
    W_in, W_out = _tables(vocab, dim, 0.5 / dim ** 0.5, 8, dev)
    (rin, w_in, rout, w_out, loss), tol = _order_tolerance(W_in, W_out, dim, plan, lr, 4.0)
    a, b = W_in.clone(), W_out.clone()
    st, ts, nan = _fused(a, b, dim, torch.from_numpy(tok).to(dev), vocab, lr=lr, window=window, neg=neg, cdf=cdf,
                         last=last, keep_p=torch.from_numpy(p).to(dev))
    gi, go = a[rin, :dim].cpu().numpy(), b[rout, :dim].cpu().numpy()
    assert np.abs(gi - w_in).max() <= tol and np.abs(go - w_out).max() <= tol
    orig = R.cbow_update

    def divided(w_in_, w_out_, ctx, tg, lr_, block=8):   # e / cw pushed to the contexts
        before = w_in_[ctx].copy()
        e, lsum = orig(w_in_, w_out_, ctx, tg, lr_, block)
        w_in_[ctx] = before + e / len(ctx)
        return e, lsum

    R.cbow_update = divided
    try:
        _, w_in_div, _, _, _ = _replay(W_in, W_out, dim, plan, lr)
    finally:
        R.cbow_update = orig
    assert np.abs(w_in_div - w_in).max() > 20 * tol
    assert st[1].item() == sum(t >= 0 for _, tg in plan for t, _ in tg) and abs(st[0].item() - loss) <= 1e-4 * loss
    assert ts.tolist() == [len(tok), kept, sum(len(c) for c, _ in plan), dropped] and nan == 0


# ---- grid-stride rounds ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [4, 100])   # LPR 1 and LPR 32
def test_grid_stride_rounds_match_replay_and_default_grid(dev, dim):
    """Sentences ``x y -1`` of distinct words with no negatives: x reads W_in[y] and W_out[x], which no other center
    reads, so the tables are deterministic at any size.  1.5 entries per lane-group of a grid of one CTA per SM:
    the default grid takes them in one round, the grid a large reserve_total shrinks in two."""
    lr = 0.1
    groups = native.sm_count(0) * 256 // RUNGS[dim][0]
    n_sent = groups // 2 + 1
    vocab = 2 * n_sent
    tok = np.full((n_sent, 3), -1, dtype=np.int64)
    tok[:, :2] = np.random.default_rng(dim).permutation(vocab).reshape(n_sent, 2)
    tok = tok.reshape(-1)
    assert len(tok) > groups
    W_in, W_out = _tables(vocab, dim, dim ** -0.25, 7, dev)
    w_in, w_out = W_in[:, :dim].double().cpu().numpy(), W_out[:, :dim].double().cpu().numpy()
    want = R.train_call(w_in, w_out, tok, lr=lr, window=5, negative_count=0, step=0, seed=SEED, philox=PH, cbow=True)
    tokens = torch.from_numpy(tok).to(dev)
    runs = []
    for reserve in (0, 1 << 20):
        a, b = W_in.clone(), W_out.clone()
        st, ts, nan = _fused(a, b, dim, tokens, vocab, lr=lr, window=5, neg=0, reserve=reserve)
        _close(a[:, :dim].cpu().numpy(), w_in, f"W_in, reserve {reserve}")
        _close(b[:, :dim].cpu().numpy(), w_out, f"W_out, reserve {reserve}")
        assert st[1].item() == want["targets"] == 2 * n_sent
        assert abs(st[0].item() - want["loss"]) <= 1e-5 * want["loss"]
        assert ts.tolist() == [len(tok), 2 * n_sent, 2 * n_sent, 0] and nan == 0
        runs.append((a, b))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


# ---- the ends of a call ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_sentence_cut_by_both_ends_of_the_call(dev, dtype):
    """One 9-word sentence with no boundary token, radii up to 5: most windows stop at the start or the end of the
    call.  The centers share rows Hogwild-style; at rows of +-0.05 and lr = 2e-4 the order moves a value by about
    1e-9, far inside the tolerance of 5e-7, while one context more or less moves rows by ~1e-6."""
    vocab, dim, neg, lr, window = 20000, 64, 3, 2e-4, 5
    tok = np.random.default_rng(3).permutation(vocab)[:9]
    W_in, W_out = _tables(vocab, dim, 0.05, 5, dev)
    w_in, w_out = W_in[:, :dim].double().cpu().numpy(), W_out[:, :dim].double().cpu().numpy()
    want = R.train_call(w_in, w_out, tok, lr=lr, window=window, negative_count=neg, step=0, seed=SEED, philox=PH,
                        cbow=True)
    seq, pos, _, _ = R.compact(tok, vocab, None, 0, SEED, PH)
    r = R.radii(pos, window, 0, SEED, PH)
    assert sum(e - r[e] < 0 for e in range(9)) >= 2 and sum(e + r[e] > 8 for e in range(9)) >= 2
    st, ts, nan = _fused(W_in, W_out, dim, torch.from_numpy(tok).to(dev, dtype), vocab, lr=lr, window=window, neg=neg)
    _close(W_in[:vocab, :dim].cpu().numpy(), w_in, "W_in")
    _close(W_out[:vocab, :dim].cpu().numpy(), w_out, "W_out")
    assert st[1].item() == want["targets"] and abs(st[0].item() - want["loss"]) <= 1e-5 * want["loss"]
    assert ts.tolist() == [9, 9, want["contexts"], 0] and nan == 0


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("case", ["boundaries and dropped ids", "all subsampled away", "one-word sentences",
                                  "one token"])
def test_call_without_contexts_leaves_tables_and_stats_alone(dev, case, dtype):
    vocab, dim = 50, 36
    keep_p = None
    if case == "boundaries and dropped ids":
        tok = np.array([-1, 50, -1, -7, 1 << 20, -1, 51])
    elif case == "all subsampled away":   # no entry at all: n_comp = 0
        tok = np.arange(40) % vocab
        keep_p = np.zeros(vocab)
    elif case == "one-word sentences":    # kept centers with no context
        tok = np.array([3, -1, 4, 60, 5, -1, 6])
    else:
        tok = np.array([17])
    W_in, W_out = _tables(vocab, dim, 0.5, 1, dev)
    in0, out0 = W_in.clone(), W_out.clone()
    st, ts, nan = _fused(W_in, W_out, dim, torch.from_numpy(tok).to(dev, dtype), vocab, lr=0.1, window=5, neg=5,
                         keep_p=torch.from_numpy(keep_p).to(dev) if keep_p is not None else None)
    _, _, kept, dropped = R.compact(tok, vocab, keep_p, 0, SEED, PH)
    assert torch.equal(W_in, in0) and torch.equal(W_out, out0)
    assert st.tolist() == [0.0, 0.0] and nan == 0
    assert ts.tolist() == [len(tok), kept, 0, dropped]
    assert (kept, dropped) == {"boundaries and dropped ids": (0, 4), "all subsampled away": (0, 0),
                               "one-word sentences": (4, 1), "one token": (1, 0)}[case]


# ---- counters and control --------------------------------------------------------------------------------------

def _model(vocab, dim, neg, lr, noise=None, seed=4, sample=0.0):
    from fps_b200.models.w2v import DeviceSkipGram

    m = DeviceSkipGram(vocab, dim, learning_rate=lr, negative=neg, seed=seed, noise_counts=noise, sample=sample)
    m.w_out.local.uniform_(-0.05, 0.05)
    return m


def test_same_seed_same_tables_and_skip_gram_unchanged(dev):
    vocab, dim = VOCAB, 100
    tok = torch.from_numpy(_pair_corpus(5, "uniform")).to(dev)
    out = []
    for cbow in (True, True, False):
        m = _model(vocab, dim, 5, 0.05)
        torch.manual_seed(0)
        m.w_out.local.uniform_(-0.05, 0.05)
        m.train_tokens(tok, window=5, cbow=cbow)
        out.append((m.w_in.local.clone(), m.w_out.local.clone()))
        m.close()
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    assert not torch.equal(out[0][0], out[2][0])


def test_non_finite_dot_sets_nan_flag(dev):
    m = _model(1000, 32, 2, 0.05)
    m.w_out.local[:1000] = float("inf")
    m.train_tokens(torch.tensor([1, 2, 3, -1], device=dev), window=2, cbow=True)
    assert int(m.nan_flag.item()) == 1
    m.close()


def test_train_tokens_cbow_never_syncs_with_the_host(dev):
    from fps_b200.models.w2v import DeviceSkipGram

    vocab = 5000
    tok = torch.randint(-1, vocab, (100000,), device=dev)
    counts = torch.bincount(tok[tok >= 0], minlength=vocab).double()
    m = DeviceSkipGram(vocab, 64, negative=5, noise_counts=counts.cpu().numpy(), sample=1e-3)
    m.train_tokens(tok, cbow=True)                       # first call: scratch allocation
    torch.cuda.synchronize()
    before = native.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            m.train_tokens(tok, window=5, cbow=True)
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
        m.train_tokens(torch.zeros(4, dtype=torch.int64, device=dev), cbow=True)
    m.close()
    m = DeviceSkipGram(100, 8, sample=0.0)
    for bad in (1, "true", None):
        with pytest.raises(ValueError, match="cbow must be True"):
            m.train_tokens(torch.zeros(4, dtype=torch.int64, device=dev), cbow=bad)
        with pytest.raises(ValueError, match="cbow must be True"):
            m.fit_tokens(torch.zeros(4, dtype=torch.int64, device=dev), cbow=bad)
    with pytest.raises(ValueError, match="window must be"):
        m.train_tokens(torch.zeros(4, dtype=torch.int64, device=dev), window=0, cbow=True)
    assert m.step_no == 0 and not m.token_stats.any()
    m.close()


def test_quality_gate_through_fit_tokens(dev):
    """The corpus, schedule and bar of the skip-gram gate (test_gpu_w2v_tokens.py), trained with CBOW at
    word2vec.c's CBOW rate 0.05.  Measured precision@10: 1.000 on an H100 (skip-gram's gate: 1.000)."""
    from fps_b200.models.w2v import DeviceSkipGram
    from fps_b200.utils.synthetic import topic_corpus

    vocab, topics = 2000, 40
    tok = topic_corpus(vocab, topics, 10, 40000, seed=2)
    counts = np.bincount(tok[tok >= 0].numpy(), minlength=vocab).astype(np.float64)
    m = DeviceSkipGram(vocab, 64, learning_rate=0.05, negative=5, seed=3, word_counts=counts, noise_counts=counts,
                       sample=1e-3)
    m.fit_tokens(tok.pin_memory(), epochs=3, batch_tokens=1 << 17, window=5, cbow=True)
    m.check_finite()
    words = torch.arange(vocab, device=dev)
    _, ids = m.most_similar(words, 10)
    prec = float(((ids % topics) == (words % topics)[:, None]).float().mean())
    chance = (vocab / topics - 1) / (vocab - 1)
    print(f"w2v cbow quality: precision@10 {prec:.3f}, chance {chance:.3f}")
    assert prec > 0.9, (prec, chance)     # measured 1.000 on an H100
    m.close()


@pytest.mark.timeout(900)               # the torchrun children have their own 420 s limit
def test_multi_rank_train_tokens_cbow():
    from tests.test_gpu_multi import _run

    _run("mp_w2v_cbow_check.py", 2, 29649, "MP_W2V_CBOW_CHECK_OK")
