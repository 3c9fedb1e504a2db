"""NumPy reference of :meth:`DeviceSkipGram.train_tokens` (DESIGN §2.13): the keep probabilities, the Philox draws
of subsampling, dynamic windows and negatives, the compaction, the center-window SGNS update, and the CBOW update of
``train_tokens(cbow=True)`` (DESIGN §2.14).

Every draw is a Philox4x32-10 value with counter ``(c0, c1, c2, c3)`` and key ``(seed lo, seed hi)``, where ``i`` is
the token's position in the call.  The functions take the generator as ``philox(c0, c1, c2, c3, k0, k1) -> (x, y,
z, w)`` (uint32 arrays, broadcasting over the counters), so the reference is replayed with an independent
implementation of it:

* keep:      ``(i, 0, 0, step)``, ``u = ((x << 32 | y) >> 11) * 2**-53``, kept iff ``u < p[w]`` (fp64);
* radius:    ``(i, 1, 0, step)``, ``r = 1 + ((x << 32 | y) mod window)``;
* negative:  ``(i, 2 | slot << 8, j | t << 8, step)`` for tries ``t`` (from ``x, y``) and ``t + 1`` (``z, w``),
  ``t`` even, of negative ``j`` of context number ``slot`` of the center.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import numpy as np

U64 = np.uint64


def keep_probabilities(counts, sample: float) -> np.ndarray:
    """word2vec.c's subsampling rule in fp64: with ``f_w = c_w / sum(c)``, word ``w`` is kept with probability
    ``min(1, (sqrt(f_w / sample) + 1) * sample / f_w)``; a word of count 0 has probability 1.  ``sample = 0``:
    every word is kept (all ones)."""
    c = np.asarray(counts, dtype=np.float64).reshape(-1)
    p = np.ones_like(c)
    if sample <= 0:
        return p
    f = c / c.sum()
    nz = f > 0
    p[nz] = np.minimum(1.0, (np.sqrt(f[nz] / sample) + 1.0) * sample / f[nz])
    return p


def _h64(r) -> np.ndarray:
    return (r[0].astype(U64) << U64(32)) | r[1].astype(U64)


def _draw(philox, i, c1, c2, step: int, seed: int):
    i = np.asarray(i, dtype=np.int64)
    return philox((i & 0xFFFFFFFF).astype(np.uint32), np.uint32(c1) if np.isscalar(c1) else c1,
                  np.uint32(c2) if np.isscalar(c2) else c2, np.uint32(step & 0xFFFFFFFF),
                  seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)


def keep_mask(tokens, p: Optional[np.ndarray], step: int, seed: int, philox: Callable) -> np.ndarray:
    """Whether each token is kept: valid ids ``[0, len(p))`` drawn under their keep probability (``p=None`` keeps
    every valid id).  Boundaries are not kept words."""
    t = np.asarray(tokens, dtype=np.int64)
    vocab = len(p) if p is not None else np.iinfo(np.int64).max
    valid = (t >= 0) & (t < vocab)
    if p is None:
        return valid
    u = (_h64(_draw(philox, np.arange(t.size), 0, 0, step, seed)) >> U64(11)).astype(np.float64) * 2.0 ** -53
    return valid & (u < p[np.where(valid, t, 0)])


def compact(tokens, vocab: int, p: Optional[np.ndarray], step: int, seed: int, philox: Callable):
    """The compacted sequence of one call: ``(seq, pos, kept, dropped)`` = int32 entries (``-1`` = boundary), their
    call positions, the number of kept words and the number of ids outside ``[0, vocab)`` other than ``-1``."""
    t = np.asarray(tokens, dtype=np.int64)
    boundary = (t < 0) | (t >= vocab)
    kept = keep_mask(t, p, step, seed, philox) if p is not None else ~boundary
    entry = kept | boundary
    pos = np.flatnonzero(entry)
    seq = np.where(boundary[pos], -1, t[pos]).astype(np.int32)
    return seq, pos.astype(np.int32), int(kept.sum()), int((boundary & (t != -1)).sum())


def radii(pos, window: int, step: int, seed: int, philox: Callable) -> np.ndarray:
    """The dynamic window radius ``1 .. window`` of the token at each call position."""
    return (1 + _h64(_draw(philox, pos, 1, 0, step, seed)) % U64(window)).astype(np.int64)


def windows(seq, pos, window: int, step: int, seed: int, philox: Callable) -> List[Tuple[int, List[int]]]:
    """``[(entry, [context entries])]`` for every kept center of the compacted sequence, contexts in increasing
    position, stopping at a boundary or the end of the call."""
    seq = np.asarray(seq)
    r = radii(pos, window, step, seed, philox)
    out = []
    n = len(seq)
    for e in range(n):
        if seq[e] < 0:
            continue
        lo = e
        while lo - 1 >= max(e - r[e], 0) and seq[lo - 1] >= 0:
            lo -= 1
        hi = e
        while hi + 1 <= min(e + r[e], n - 1) and seq[hi + 1] >= 0:
            hi += 1
        out.append((e, list(range(lo, e)) + list(range(e + 1, hi + 1))))
    return out


def negative(i: int, slot: int, j: int, ctx: int, vocab: int, step: int, seed: int, philox: Callable,
             cdf: Optional[np.ndarray] = None, last_nonzero: int = 0, max_tries: int = 32) -> int:
    """Noise word ``j`` of context ``slot`` of the center at call position ``i``: uniform ``h mod vocab``, or the
    53-bit uniform times ``cdf[-1]`` through an upper-bound search of ``cdf``; a draw equal to ``ctx`` is redrawn,
    and ``-1`` (void) when all ``max_tries`` are."""
    for t in range(0, max_tries, 2):
        r = _draw(philox, i, np.uint32(2 | (slot << 8)), np.uint32(j | (t << 8)), step, seed)
        hs = (int(_h64((r[0], r[1]))), int(_h64((r[2], r[3]))))
        for q in range(2):
            if t + q >= max_tries:
                break
            if cdf is not None:
                x = float(hs[q] >> 11) * 2.0 ** -53 * float(cdf[-1])
                c = int(np.searchsorted(cdf, x, side="right"))
                c = c if c < len(cdf) else int(last_nonzero)
            else:
                c = hs[q] % int(vocab)
            if c != ctx:
                return c
    return -1


def center_targets(i: int, contexts_words, negative_count: int, vocab: int, step: int, seed: int,
                   philox: Callable, **noise) -> List[List[Tuple[int, float]]]:
    """``[[(word, label), ...] per context]``: the context's target slots ``0 .. negative_count``, the context word
    with label 1, then its noise words with label 0.  A void draw keeps its slot as ``(-1, 0.0)``."""
    out = []
    for slot, ctx in enumerate(contexts_words):
        tg = [(int(ctx), 1.0)]
        for j in range(negative_count):
            tg.append((negative(i, slot, j, int(ctx), vocab, step, seed, philox, **noise), 0.0))
        out.append(tg)
    return out


def target_block(width: int) -> int:
    """Target slots the kernel pulls per block for rows of ``width`` floats: 8, or 6 over 384 floats."""
    return 6 if int(width) > 384 else 8


def center_update(u: np.ndarray, w_out: np.ndarray, targets, lr: float, block: int = 8):
    """The update of one center (DESIGN §2.13) applied in place to ``w_out`` (rows indexed by word).  ``u`` is the
    center's row as pulled; returns ``(D, loss)``, the delta to add to it and ``sum -log sigmoid(+-d)``.  Each
    context's targets (:func:`center_targets`) are read in blocks of ``block`` slots, a void slot (word ``-1``)
    included and then skipped: a row repeated inside a block is read as it was before the block."""
    dt = u.dtype
    D = np.zeros_like(u)
    loss = 0.0
    for tg in targets:
        w = u + D
        e = np.zeros_like(u)
        for b0 in range(0, len(tg), block):
            blk = [(t, label) for t, label in tg[b0:b0 + block] if t >= 0]
            vs = [w_out[t].copy() for t, _ in blk]
            for (t, label), v in zip(blk, vs):
                d = dt.type(np.dot(w, v))
                g = dt.type(lr) * (dt.type(label) - dt.type(1.0) / (dt.type(1.0) + np.exp(-d)))
                loss += float(np.logaddexp(0.0, -d if label else d))
                e += g * v
                w_out[t] += g * w
        D += e
    return D, loss


def cbow_update(w_in: np.ndarray, w_out: np.ndarray, context_words, targets, lr: float, block: int = 8):
    """The CBOW update of one center (DESIGN §2.14) applied in place to both tables.  ``h`` is the mean of the
    ``context_words`` rows of ``w_in`` as pulled, summed in the order given (a repeated word counts each time);
    ``targets`` is the center's one slot list (``[(center, 1.0), noise ...]``), trained on ``h`` by
    :func:`center_update`, which returns the error ``e``.  ``e`` is then added, unscaled, to the row of every
    context word, once per occurrence.  Returns ``(e, loss)``; with no context words nothing changes."""
    if len(context_words) == 0:
        return np.zeros(w_in.shape[1], dtype=w_in.dtype), 0.0
    rows = [w_in[c].copy() for c in context_words]
    h = np.zeros_like(rows[0])
    for r in rows:
        h += r
    h /= w_in.dtype.type(len(rows))
    e, loss = center_update(h, w_out, [targets], lr, block)
    for c in context_words:
        w_in[c] += e
    return e, loss


def cbow_centers(seq, pos, window: int, negative_count: int, vocab: int, step: int, seed: int, philox: Callable,
                 **noise) -> List[Tuple[List[int], List[Tuple[int, float]]]]:
    """``[(context words, targets)]`` of every CBOW center with at least one context, in compacted order: the
    context words in increasing position, and the targets of :func:`center_targets` for the center word alone, so
    the noise words are those of context slot 0, rejected against the center word."""
    seq = np.asarray(seq)
    out = []
    for e, ctx in windows(seq, pos, window, step, seed, philox):
        if ctx:
            tg = center_targets(int(pos[e]), [seq[e]], negative_count, vocab, step, seed, philox, **noise)[0]
            out.append(([int(c) for c in seq[ctx]], tg))
    return out


def train_call(w_in: np.ndarray, w_out: np.ndarray, tokens, *, lr: float, window: int, negative_count: int,
               step: int, seed: int, philox: Callable, p: Optional[np.ndarray] = None, cdf=None,
               last_nonzero: int = 0, max_tries: int = 32, cbow: bool = False, order=None) -> dict:
    """One :meth:`DeviceSkipGram.train_tokens` call applied sequentially, center by center in compacted order, to
    the tables in place, in target blocks of :func:`target_block` of the row width.  ``cbow=True`` replays CBOW
    (:func:`cbow_update`; the negatives are those of context slot 0, rejected against the center word).  ``order``
    ``"reverse"`` applies the centers last to first.  Returns the counters ``tokens, kept, contexts, dropped`` and
    ``loss, targets`` (void draws are not targets; a CBOW center with no context trains and counts nothing)."""
    vocab = w_in.shape[0]
    block = target_block(w_in.shape[1])
    seq, pos, kept, dropped = compact(tokens, vocab, p, step, seed, philox)
    loss, n_tgt, n_ctx = 0.0, 0, 0
    noise = dict(cdf=cdf, last_nonzero=last_nonzero, max_tries=max_tries)
    if cbow:
        plan = cbow_centers(seq, pos, window, negative_count, vocab, step, seed, philox, **noise)
        for ctx, tg in (plan[::-1] if order == "reverse" else plan):
            _, l = cbow_update(w_in, w_out, ctx, tg, lr, block)
            loss += l
            n_tgt += sum(t >= 0 for t, _ in tg)
            n_ctx += len(ctx)
        return dict(tokens=len(np.asarray(tokens)), kept=kept, contexts=n_ctx, dropped=dropped, loss=loss,
                    targets=n_tgt)
    wins = windows(seq, pos, window, step, seed, philox)
    for e, ctx in (wins[::-1] if order == "reverse" else wins):
        tg = center_targets(int(pos[e]), seq[ctx], negative_count, vocab, step, seed, philox, **noise)
        D, l = center_update(w_in[seq[e]].copy(), w_out, tg, lr, block)
        w_in[seq[e]] += D
        loss += l
        n_tgt += sum(t >= 0 for c in tg for t, _ in c)
        n_ctx += len(ctx)
    return dict(tokens=len(np.asarray(tokens)), kept=kept, contexts=n_ctx, dropped=dropped, loss=loss,
                targets=n_tgt)
