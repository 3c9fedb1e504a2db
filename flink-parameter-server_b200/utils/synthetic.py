"""Synthetic rating streams with learnable structure (there is no network for datasets).

``lowrank_ratings(users, items)`` evaluates a fixed rank-``rank`` ground-truth model whose factors are
pseudo-random *functions of the id* (no tables, so 10M x 1M problems cost nothing to describe):

    r(u, i) = scale / sqrt(rank) * sum_f a_f(u) * b_f(i),      a_f, b_f ~ U(-1, 1) hashed from (id, f, seed)

Used by the convergence gates (tests/mp_replica_check.py, bench.py ``config.quality``): every parallel
mode must reach the same held-out RMSE as the single-worker run on the same update budget.
"""
from __future__ import annotations

import torch

_M1, _M2 = 0x9E3779B97F4A7C15 - (1 << 64), 0xBF58476D1CE4E5B9 - (1 << 64)   # as signed int64


def _mix(x: torch.Tensor) -> torch.Tensor:
    """splitmix64-style finaliser on int64 tensors (wrap-around arithmetic)."""
    x = (x ^ ((x >> 30) & 0x3FFFFFFFF)) * _M2
    x = (x ^ ((x >> 27) & 0x1FFFFFFFFF)) * _M1
    return x ^ ((x >> 31) & 0x1FFFFFFFF)


def hashed_uniform(ids: torch.Tensor, f: int, seed: int) -> torch.Tensor:
    """U(-1, 1) as a pure function of (id, f, seed); fp32."""
    x = _mix(ids.to(torch.int64) * _M1 + (f + 1) * 0x632BE5AB + seed * 0x1B873593)
    return ((x >> 40) & 0xFFFFFF).to(torch.float32) * (2.0 / 16777216.0) - 1.0


def lowrank_ratings(users: torch.Tensor, items: torch.Tensor, rank: int = 8, seed: int = 0,
                    scale: float = 1.5) -> torch.Tensor:
    r = torch.zeros(users.shape, dtype=torch.float32, device=users.device)
    for f in range(rank):
        r += hashed_uniform(users, f, 2 * seed + 1) * hashed_uniform(items, f, 2 * seed + 2)
    return r * (scale / rank ** 0.5)


def lowrank_implicit(num_users: int, num_items: int, per_user: int, held_out: int, seed: int,
                     beta: float = 4.0, rank: int = 8):
    """Implicit feedback with a learnable ranking: every user "consumes" ``per_user`` distinct items, the
    Gumbel top-``per_user`` of ``beta * lowrank_ratings(u, i)`` (a draw without replacement with
    probabilities ~ ``exp(beta * r)``), and ``held_out`` of them, chosen at random, are kept apart.

    Returns int64 CPU tensors ``(train_users, train_items, test_users, test_items)``; the train pairs are
    in a random stream order, the test pairs ordered by user.  A pure function of its arguments; it
    scores every (user, item) pair, so it is meant for small sizes (about 10^4 x 10^4)."""
    if not 0 <= held_out < per_user <= num_items:
        raise ValueError("need 0 <= held_out < per_user <= num_items")
    g = torch.Generator().manual_seed(int(seed))
    scale = 1.5 / rank ** 0.5                  # lowrank_ratings as a product of its per-id factors
    iid = torch.arange(num_items)
    B = torch.stack([hashed_uniform(iid, f, 2 * seed + 2) for f in range(rank)], 1)
    tr_u, tr_i, te_u, te_i = [], [], [], []
    for lo in range(0, num_users, 1024):
        uid = torch.arange(lo, min(lo + 1024, num_users))
        A = torch.stack([hashed_uniform(uid, f, 2 * seed + 1) for f in range(rank)], 1)
        u01 = torch.rand((uid.numel(), num_items), generator=g).clamp_(1e-12, 1.0 - 1e-7)
        keys = beta * scale * (A @ B.T) - torch.log(-torch.log(u01))
        top = keys.topk(per_user, dim=1).indices
        order = torch.rand((uid.numel(), per_user), generator=g).argsort(1)
        top = top.gather(1, order)
        users = uid[:, None].expand(-1, per_user)
        te_u.append(users[:, :held_out].reshape(-1)); te_i.append(top[:, :held_out].reshape(-1))
        tr_u.append(users[:, held_out:].reshape(-1)); tr_i.append(top[:, held_out:].reshape(-1))
    tr_u, tr_i = torch.cat(tr_u), torch.cat(tr_i)
    perm = torch.randperm(tr_u.numel(), generator=g)
    return tr_u[perm], tr_i[perm], torch.cat(te_u), torch.cat(te_i)


def topic_corpus(vocab: int, topics: int, sentence_len: int, sentences: int, seed: int = 0,
                 zipf: float = 1.0) -> torch.Tensor:
    """A seeded token stream with known neighbours for word2vec: word ``w`` belongs to topic ``w % topics``, each
    sentence draws one topic uniformly and ``sentence_len`` words of it, the word of rank ``w // topics`` in its
    topic with weight ``1 / (rank + 1) ** zipf``.  So low ids are frequent (a Zipf-like corpus that subsampling
    acts on) and two words are true neighbours iff they share a topic.

    Returns a 1-D int64 CPU tensor: the sentences, each followed by ``-1`` (a sentence boundary)."""
    if not 1 <= topics <= vocab or sentence_len < 1 or sentences < 1:
        raise ValueError("need 1 <= topics <= vocab, sentence_len >= 1 and sentences >= 1")
    g = torch.Generator().manual_seed(int(seed))
    per = -(-vocab // topics)                             # ranks in the largest topic
    rank = torch.arange(per, dtype=torch.float64)
    topic = torch.randint(0, topics, (sentences,), generator=g)
    size = (vocab - 1 - torch.arange(topics)) // topics + 1   # words of each topic
    out = torch.full((sentences, sentence_len + 1), -1, dtype=torch.int64)
    for k in range(topics):
        rows = torch.nonzero(topic == k).flatten()
        if rows.numel() == 0:
            continue
        w = (rank[: int(size[k])] + 1.0) ** -float(zipf)
        r = torch.multinomial(w, rows.numel() * sentence_len, replacement=True, generator=g)
        out[rows, :sentence_len] = (r * topics + k).view(rows.numel(), sentence_len)
    return out.reshape(-1)


def planted_fm(num_features: int, fields: int, k: int, n: int, seed: int = 0, loss: str = "logistic"):
    """One-hot examples with labels from a planted factorization machine, for the FM quality gates.

    Field ``f`` owns the ids ``[f * per, (f + 1) * per)``, ``per = num_features // fields``; every example takes one
    id per field, uniformly.  The planted model has ``w*_i = U(-1, 1)`` and ``v*_i,f = U(-1, 1)`` hashed from
    ``(id, f, seed)``; its score is the linear term scaled to unit standard deviation plus the pairwise term
    ``sum_{a<b} <v*_a, v*_b>`` scaled to standard deviation 2, so a model with factors can beat a linear one.
    ``"logistic"``: ``y ~ Bernoulli(sigmoid(score))``; ``"squared"``: ``y = score + N(0, 0.25)``.

    Returns ``(row_ptr, cols, labels)`` on the CPU: int64 ``[n + 1]``, int64 ``[n * fields]``, float32 ``[n]``."""
    if fields < 1 or num_features < fields or k < 1 or n < 0:
        raise ValueError("planted_fm needs fields >= 1, num_features >= fields, k >= 1 and n >= 0")
    if loss not in ("logistic", "squared"):
        raise ValueError(f"loss must be 'logistic' or 'squared', got {loss!r}")
    per = num_features // fields
    g = torch.Generator().manual_seed(seed)
    cols = torch.randint(0, per, (n, fields), generator=g) + torch.arange(fields) * per
    lin = hashed_uniform(cols, 0, 2 * seed + 1).sum(1) / (fields / 3.0) ** 0.5
    v = torch.stack([hashed_uniform(cols, f + 1, 2 * seed + 1) for f in range(k)], -1)   # [n, fields, k]
    s = v.sum(1)
    pairs = 0.5 * ((s * s).sum(1) - (v * v).sum((1, 2)))
    npairs = fields * (fields - 1) / 2
    score = lin + (2.0 / max(npairs * k / 9.0, 1e-12) ** 0.5) * pairs if fields > 1 else lin
    if loss == "logistic":
        labels = (torch.rand(n, generator=g) < torch.sigmoid(score)).to(torch.float32)
    else:
        labels = (score + 0.25 * torch.randn(n, generator=g)).to(torch.float32)
    row_ptr = torch.arange(n + 1, dtype=torch.int64) * fields
    return row_ptr, cols.reshape(-1).to(torch.int64), labels


def planted_ffm(num_features: int, fields: int, k: int, n: int, seed: int = 0, loss: str = "logistic"):
    """One-hot examples with labels from a planted field-aware factorization machine, for the FFM quality gates.

    Field ``f`` owns the ids ``[f * per, (f + 1) * per)``, ``per = num_features // fields``; every example takes one
    id per field, uniformly, in field order.  The planted model has ``w*_i = U(-1, 1)`` and one slab per (id, field)
    ``V*[i, f]_c = U(-1, 1)`` hashed from ``(id, f, c, seed)``; its score is the linear term scaled to unit standard
    deviation plus the pair term ``sum_{a<b} <V*[i_a, f_b], V*[i_b, f_a]>`` scaled to standard deviation 2, as in
    :func:`planted_fm`.  ``"logistic"``: ``y ~ Bernoulli(sigmoid(score))``; ``"squared"``: ``y = score + N(0, 0.25)``.

    Returns ``(row_ptr, cols, fields, labels)`` on the CPU: int64 ``[n + 1]``, int64 ``[n * fields]``, int32
    ``[n * fields]``, float32 ``[n]``."""
    if fields < 1 or num_features < fields or k < 1 or n < 0:
        raise ValueError("planted_ffm needs fields >= 1, num_features >= fields, k >= 1 and n >= 0")
    if loss not in ("logistic", "squared"):
        raise ValueError(f"loss must be 'logistic' or 'squared', got {loss!r}")
    per = num_features // fields
    g = torch.Generator().manual_seed(seed)
    cols = torch.randint(0, per, (n, fields), generator=g) + torch.arange(fields) * per
    lin = hashed_uniform(cols, 0, 2 * seed + 1).sum(1) / (fields / 3.0) ** 0.5
    pairs = torch.zeros(n)
    for a in range(fields):
        for b in range(a + 1, fields):
            for c in range(k):
                pairs += (hashed_uniform(cols[:, a], 1 + b * k + c, 2 * seed + 1)
                          * hashed_uniform(cols[:, b], 1 + a * k + c, 2 * seed + 1))
    npairs = fields * (fields - 1) / 2
    score = lin + (2.0 / max(npairs * k / 9.0, 1e-12) ** 0.5) * pairs if fields > 1 else lin
    if loss == "logistic":
        labels = (torch.rand(n, generator=g) < torch.sigmoid(score)).to(torch.float32)
    else:
        labels = (score + 0.25 * torch.randn(n, generator=g)).to(torch.float32)
    row_ptr = torch.arange(n + 1, dtype=torch.int64) * fields
    field_ids = torch.arange(fields, dtype=torch.int32).repeat(n)
    return row_ptr, cols.reshape(-1).to(torch.int64), field_ids, labels
