"""The fused window kernel's skip-gram (``fps_w2v_kernel<false, ...>``) against the fp64 replay of
``models/w2v_ref.py``, every Philox draw replayed by ``tests/philox_ref.py``: every dispatch rung and the four ways a
context's noise words are drawn and blocked, uniform and unigram noise, voided and repeated targets, grid-stride
rounds, the ends of a call, and the counters."""
import functools

import numpy as np
import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.models import w2v_ref as R
from fps_b200.ops import native
from tests.philox_ref import philox4x32 as PH
from tests.w2v_cases import ATOL_OF_MAX, RTOL, RUNGS, SEED, SWEEP, VOCAB, close, fused, noise_dist, tables

pytestmark = pytest.mark.gpu

def _path(neg, lpr, tb):
    """How the kernel gets a context's noise words: lane j of the group draws word j and the others read it with a
    shuffle (negative <= LPR), or every lane draws all of them; the 1 + negative target slots fit one block of TB
    or take several."""
    return ("shuffled" if neg <= lpr else "serial", "one block" if 1 + neg <= tb else "several blocks")


@pytest.fixture
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def test_sweep_reaches_every_rung_and_noise_path():
    assert {RUNGS[d][:2] for d, _ in SWEEP} == {(1, 1), (2, 1), (4, 1), (8, 1), (16, 1), (32, 1), (32, 2), (32, 3),
                                               (32, 4)}
    assert {_path(n, RUNGS[d][0], RUNGS[d][2]) for d, n in SWEEP} == {
        (a, b) for a in ("shuffled", "serial") for b in ("one block", "several blocks")}
    assert {d for d in RUNGS if d % 4} == {3, 13, 387}


# ---- every rung x every noise path, on corpora whose centers share no row --------------------------------------

@functools.lru_cache(maxsize=None)
def _corpus(neg, kind, n_sent=16):
    """Sentences ``x y -1`` whose centers read pairwise disjoint W_out rows, so no result depends on the order the
    lane-groups run in.  Built greedily at step 0: a candidate sentence that would read a row another center reads
    is replaced by a boundary.  Returns (tokens, [(center, its targets)])."""
    _, cdf, last = noise_dist(kind)
    words = iter(np.random.default_rng(neg).permutation(VOCAB).tolist())
    tok, rep, used = [], [], set()
    while len(rep) < 2 * n_sent:
        x, y = next(words), next(words)
        i = len(tok)
        tx = R.center_targets(i, [y], neg, VOCAB, 0, SEED, PH, cdf=cdf, last_nonzero=last)
        ty = R.center_targets(i + 1, [x], neg, VOCAB, 0, SEED, PH, cdf=cdf, last_nonzero=last)
        rx, ry = {t for t, _ in tx[0]}, {t for t, _ in ty[0]}
        if rx & ry or (rx | ry) & used or -1 in rx | ry:
            tok.append(-1)
            continue
        used |= rx | ry
        tok += [x, y, -1]
        rep += [(x, tx), (y, ty)]
    return np.array(tok, dtype=np.int64), rep


@pytest.mark.parametrize("noise", ["uniform", "unigram"])
@pytest.mark.parametrize("dim,neg", SWEEP)
def test_window_kernel_matches_fp64_replay_at_every_rung(dev, dim, neg, noise):
    from fps_b200.models.w2v import DeviceSkipGram

    lr = 0.1
    counts, cdf, last = noise_dist(noise)
    tok, rep = _corpus(neg, noise)
    m = DeviceSkipGram(VOCAB, dim, learning_rate=lr, negative=neg, seed=SEED, noise_counts=counts, sample=0.0)
    try:
        if counts is not None:
            assert np.array_equal(m._noise_cdf.cpu().numpy(), cdf) and m._noise_last == last < VOCAB - 1
        W_in, W_out = tables(VOCAB, dim, dim ** -0.25, dim + neg, dev)
        m.w_in.local.copy_(W_in)
        m.w_out.local.copy_(W_out)
        centers = [c for c, _ in rep]
        rows = sorted({t for _, tg in rep for ctx in tg for t, _ in ctx})
        at = {w: k for k, w in enumerate(rows)}
        w_in = W_in[centers, :dim].double().cpu().numpy()
        w_out = W_out[rows, :dim].double().cpu().numpy()
        loss = 0.0
        for k, (c, tg) in enumerate(rep):
            D, lsum = R.center_update(w_in[k].copy(), w_out, [[(at[t], lab) for t, lab in ctx] for ctx in tg], lr,
                                      R.target_block(dim))
            w_in[k] += D
            loss += lsum
        m.train_tokens(torch.from_numpy(tok).to(dev), window=5)
        torch.cuda.synchronize()
        got_in, got_out = m.w_in.local, m.w_out.local
        close(got_in[centers, :dim].cpu().numpy(), w_in, "W_in")
        close(got_out[rows, :dim].cpu().numpy(), w_out, "W_out")
        keep_in = torch.ones(VOCAB, dtype=torch.bool, device=dev)
        keep_in[centers] = False
        keep_out = torch.ones(VOCAB, dtype=torch.bool, device=dev)
        keep_out[rows] = False
        assert torch.equal(got_in[:VOCAB][keep_in], W_in[keep_in])
        assert torch.equal(got_out[:VOCAB][keep_out], W_out[keep_out])
        assert not got_in[:, dim:].any() and not got_out[:, dim:].any()
        st, ts = m.stats.cpu(), m.token_stats.cpu()
        assert st[1].item() == len(rep) * (1 + neg)
        assert abs(st[0].item() - loss) <= 1e-5 * loss
        assert ts.tolist() == [len(tok), len(rep), len(rep), 0]
        assert int(m.nan_flag.item()) == 0
    finally:
        m.close()


# ---- voided and repeated targets: one sentence `x y` per call on a tiny vocabulary ------------------------------

def _blocks(slots, tb):
    return [slots[b:b + tb] for b in range(0, len(slots), tb)]


@pytest.mark.parametrize("noise", ["uniform", "on the context"])
@pytest.mark.parametrize("max_tries", [1, 2])
@pytest.mark.parametrize("dim,neg", [(16, 12), (100, 12), (512, 12), (4, 255), (512, 255)])
def test_void_and_repeated_targets_match_fp64_replay(dev, dim, neg, max_tries, noise):
    """With W_in[y] = 0 the center y has one context and w = 0, so it pushes g * 0 to every W_out row: W_out,
    W_in[x], the loss and the counters do not depend on when the two lane-groups run.  W_in[y] = sum g v reads rows
    x pushes to, before or after; it is held to the bound that leaves."""
    lr, tb = 0.1, RUNGS[dim][2]
    if noise == "uniform":
        vocab, x, y, cdf, last = 4, 0, 1, None, 0
    else:   # words 0 and 4 have weight 0; 12 / 14 of the draws for the context y = 3 are y
        vocab, x, y, last = 5, 1, 3, 3
        cdf = np.cumsum([0.0, 1.0, 1.0, 12.0, 0.0])
    cdf_d = torch.from_numpy(cdf).to(dev) if cdf is not None else None
    tokens = torch.tensor([x, y], device=dev)
    seen = set()
    for step in range(2 if neg == 255 else 6):
        W_in, W_out = tables(vocab, dim, 0.5, step, dev)
        W_in[y] = 0.0
        in0 = W_in.cpu().numpy()
        w_in, w_out = W_in[:, :dim].double().cpu().numpy(), W_out[:, :dim].double().cpu().numpy()
        u_x = w_in[x].copy()
        noise_kw = dict(cdf=cdf, last_nonzero=last, max_tries=max_tries)
        want = R.train_call(w_in, w_out, [x, y], lr=lr, window=5, negative_count=neg, step=step, seed=SEED,
                            philox=PH, **noise_kw)
        st, ts, nan = fused(W_in, W_out, dim, tokens, vocab, lr=lr, window=5, neg=neg, step=step,
                            max_tries=max_tries, cdf=cdf_d, last=last)
        got_in, got_out = W_in.cpu().numpy(), W_out.cpu().numpy()
        close(got_out[:, :dim], w_out, f"W_out, step {step}")
        close(got_in[x, :dim], w_in[x], f"W_in[x], step {step}")
        sx = [t for t, _ in R.center_targets(0, [y], neg, vocab, step, SEED, PH, **noise_kw)[0]]
        sy = [t for t, _ in R.center_targets(1, [x], neg, vocab, step, SEED, PH, **noise_kw)[0]]
        bound = 0.5 * lr * lr * np.abs(u_x) * sum(sx.count(t) for t in sy if t >= 0)
        tol = bound + RTOL * np.abs(w_in[y]) + ATOL_OF_MAX * np.abs(w_in[y]).max()
        assert (np.abs(got_in[y, :dim] - w_in[y]) <= tol).all(), f"W_in[y], step {step}"
        others = [w for w in range(vocab) if w not in (x, y)]
        assert np.array_equal(got_in[others], in0[others])
        assert not got_in[:, dim:].any() and not got_out[:, dim:].any()
        assert st[1].item() == want["targets"] == sum(t >= 0 for t in sx + sy)
        assert abs(st[0].item() - want["loss"]) <= 1e-5 * want["loss"]
        assert ts.tolist() == [2, 2, 2, 0] and want["contexts"] == 2 and nan == 0
        blocks = _blocks(sx, tb)
        live = [[t for t in b if t >= 0] for b in blocks]
        if any(len(b) != len(set(b)) for b in live):
            seen.add("repeat inside a block")
        if any(set(a) & set(b) for k, a in enumerate(live) for b in live[k + 1:]):
            seen.add("repeat in a later block")
        if any(-1 in b for b in blocks[:-1]):
            seen.add("void before a block boundary")
    assert seen == {"repeat inside a block", "repeat in a later block", "void before a block boundary"}


# ---- grid-stride rounds ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [4, 100])   # LPR 1 and LPR 32
def test_grid_stride_rounds_match_replay_and_default_grid(dev, dim):
    """Sentences ``x y -1`` of distinct words with no negatives: each row is read and pushed by one center, so the
    tables are deterministic at any size.  There are 1.5 entries per lane-group of a grid of one CTA per SM: the
    default grid takes them in one round, and the grid a large reserve_total shrinks to one CTA per SM in two."""
    lr = 0.1
    groups = native.sm_count(0) * 256 // RUNGS[dim][0]
    n_sent = groups // 2 + 1
    vocab = 2 * n_sent
    tok = np.full((n_sent, 3), -1, dtype=np.int64)
    tok[:, :2] = np.random.default_rng(dim).permutation(vocab).reshape(n_sent, 2)
    tok = tok.reshape(-1)
    assert len(tok) > groups
    W_in, W_out = tables(vocab, dim, dim ** -0.25, 7, dev)
    w_in, w_out = W_in[:, :dim].double().cpu().numpy(), W_out[:, :dim].double().cpu().numpy()
    want = R.train_call(w_in, w_out, tok, lr=lr, window=5, negative_count=0, step=0, seed=SEED, philox=PH)
    tokens = torch.from_numpy(tok).to(dev)
    runs = []
    for reserve in (0, 1 << 20):
        a, b = W_in.clone(), W_out.clone()
        st, ts, nan = fused(a, b, dim, tokens, vocab, lr=lr, window=5, neg=0, reserve=reserve)
        close(a[:, :dim].cpu().numpy(), w_in, f"W_in, reserve {reserve}")
        close(b[:, :dim].cpu().numpy(), w_out, f"W_out, reserve {reserve}")
        assert st[1].item() == want["targets"] == 2 * n_sent
        assert abs(st[0].item() - want["loss"]) <= 1e-5 * want["loss"]
        assert ts.tolist() == [len(tok), 2 * n_sent, 2 * n_sent, 0] and nan == 0
        runs.append((a, b))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


# ---- the ends of a call ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_sentence_cut_by_both_ends_of_the_call(dev, dtype):
    """One 9-word sentence with no boundary token, radii up to 5: most windows stop at the start or the end of the
    call.  The centers share rows, applied Hogwild-style: reading a row before or after another center's push
    (lr/2 |w| ~ 5e-6 at rows of +-0.05 and lr = 2e-4) changes a center's delta by about (lr/2)^2 |w| ~ 5e-10, far
    inside the tolerance of 5e-7, so the reference applies the centers one after the other.  One context more or
    less would move rows by ~5e-6."""
    from fps_b200.models.w2v import DeviceSkipGram

    vocab, dim, neg, lr, window = 20000, 64, 3, 2e-4, 5
    tok = np.random.default_rng(3).permutation(vocab)[:9]
    m = DeviceSkipGram(vocab, dim, learning_rate=lr, negative=neg, seed=SEED, sample=0.0)
    try:
        W_in, W_out = tables(vocab, dim, 0.05, 5, dev)
        m.w_in.local.copy_(W_in)
        m.w_out.local.copy_(W_out)
        w_in, w_out = W_in[:, :dim].double().cpu().numpy(), W_out[:, :dim].double().cpu().numpy()
        want = R.train_call(w_in, w_out, tok, lr=lr, window=window, negative_count=neg, step=0, seed=SEED,
                            philox=PH)
        seq, pos, _, _ = R.compact(tok, vocab, None, 0, SEED, PH)
        wins = R.windows(seq, pos, window, 0, SEED, PH)
        r = R.radii(pos, window, 0, SEED, PH)
        assert sum(e - r[e] < 0 for e, _ in wins) >= 2 and sum(e + r[e] > 8 for e, _ in wins) >= 2
        m.train_tokens(torch.from_numpy(tok).to(dev, dtype), window=window)
        torch.cuda.synchronize()
        close(m.w_in.local[:vocab, :dim].cpu().numpy(), w_in, "W_in")
        close(m.w_out.local[:vocab, :dim].cpu().numpy(), w_out, "W_out")
        st = m.stats.cpu()
        assert st[1].item() == want["targets"] == want["contexts"] * (1 + neg)
        assert abs(st[0].item() - want["loss"]) <= 1e-5 * want["loss"]
        assert m.token_stats.tolist() == [9, 9, want["contexts"], 0] == [9, 9, sum(len(c) for _, c in wins), 0]
        assert int(m.nan_flag.item()) == 0
    finally:
        m.close()


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("case", ["boundaries and dropped ids", "all subsampled away", "one token"])
def test_call_without_contexts_leaves_tables_and_stats_alone(dev, case, dtype):
    vocab, dim = 50, 36
    keep_p = None
    if case == "boundaries and dropped ids":
        tok = np.array([-1, 50, -1, -7, 1 << 20, -1, 51])
    elif case == "all subsampled away":   # no entry at all: n_comp = 0
        tok = np.arange(40) % vocab
        keep_p = np.zeros(vocab)
    else:
        tok = np.array([17])
    W_in, W_out = tables(vocab, dim, 0.5, 1, dev)
    in0, out0 = W_in.clone(), W_out.clone()
    st, ts, nan = fused(W_in, W_out, dim, torch.from_numpy(tok).to(dev, dtype), vocab, lr=0.1, window=5, neg=5,
                        keep_p=torch.from_numpy(keep_p).to(dev) if keep_p is not None else None)
    _, _, kept, dropped = R.compact(tok, vocab, keep_p, 0, SEED, PH)
    assert torch.equal(W_in, in0) and torch.equal(W_out, out0)
    assert st.tolist() == [0.0, 0.0] and nan == 0
    assert ts.tolist() == [len(tok), kept, 0, dropped]
    assert (kept, dropped) == {"boundaries and dropped ids": (0, 4), "all subsampled away": (0, 0),
                               "one token": (1, 0)}[case]
