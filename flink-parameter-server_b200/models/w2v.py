"""word2vec skip-gram with negative sampling on the parameter server (BASELINE.json config 4:
"word2vec skip-gram negative-sampling dim=300, push fused with paramUpdate").

Both embedding matrices live on the PS (``W_in`` and ``W_out``, sharded ``word % G``); a worker
step over a micro-batch of (center, context) pairs is ONE launch of the fused pull+SGD+push kernel
(ops/csrc/fps_core.cu with ``err_mode = 2``: ``g = lr * (label - sigmoid(u.v))``): it pulls both rows
from their owners, and pushes ``g*v`` to ``W_in[center]`` and ``g*u`` to ``W_out[context]`` with
``red.global.add.v4.f32`` -- the additive paramUpdate happens in the owner's memory system.
``negative`` extra pairs per positive are sampled on the device (uniform over the vocabulary) with
label 0.  Not part of the reference's algorithm suite; it exercises the same API on a 1.2 KB row.
``optimizer="adagrad"`` replaces the global rate by row-wise AdaGrad (DESIGN §2.10), with one fp32
accumulator per row of each table on that row's shard.  ``noise_counts`` draws the negatives from the unigram
noise ``counts ** noise_power`` (Mikolov et al. 2013) instead (DESIGN §2.11).
``train_tokens`` / ``fit_tokens`` train from a token stream (DESIGN §2.13): frequent-word subsampling, dynamic
windows and sentence boundaries on the device, and one fused kernel that trains each kept center over its whole
window, holding ``W_in[center]`` in registers and pushing it once.  ``cbow=True`` trains CBOW on the same windows
(DESIGN §2.14): one fused kernel averages the context rows, trains the center word against the noise words and
pushes the error to every context row.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.distributed as dist

from ..errors import FactorIsNotANumberException
from ..ops import native
from ..store.replica_cache import ReplicaCache
from ..store.sharded_table import ShardedTable
from .w2v_ref import keep_probabilities

ERR_LOGISTIC = 2


def check_noise(noise_counts, vocab: int, noise_power: float) -> np.ndarray:
    """Validate the unigram counts of :class:`DeviceSkipGram` and return them as float64: one finite,
    non-negative count per word, not all zero, and a finite ``noise_power >= 0``.  Raises ``ValueError``."""
    if not (math.isfinite(float(noise_power)) and float(noise_power) >= 0):
        raise ValueError(f"noise_power must be a finite number >= 0, got {noise_power!r}")
    return _counts(noise_counts, vocab, "noise_counts")


def _counts(counts, vocab: int, name: str) -> np.ndarray:
    c = (counts.detach().cpu().numpy() if torch.is_tensor(counts)
         else np.asarray(counts)).astype(np.float64).reshape(-1)
    if c.size != int(vocab):
        raise ValueError(f"{name} must hold one count per word of the vocabulary ({vocab}), got {c.size}")
    if not np.isfinite(c).all():
        raise ValueError(f"{name} must be finite")
    if (c < 0).any():
        raise ValueError(f"{name} must be >= 0")
    if not (c > 0).any():
        raise ValueError(f"{name} must have a positive count for at least one word")
    return c


def check_sample(sample) -> float:
    """Validate the subsampling threshold of :class:`DeviceSkipGram`: a finite number >= 0."""
    if not (math.isfinite(float(sample)) and float(sample) >= 0):
        raise ValueError(f"sample must be a finite number >= 0 (0 keeps every word), got {sample!r}")
    return float(sample)


def check_token_call(tokens, window, optimizer: str, sample: float, has_counts: bool, cbow=False) -> None:
    """The refusals of :meth:`DeviceSkipGram.train_tokens`, each a ``ValueError`` that names the fix."""
    if not isinstance(cbow, bool):
        raise ValueError(f"cbow must be True (CBOW) or False (skip-gram), got {cbow!r}: pass a bool, "
                         "e.g. cbow=bool(flag)")
    if optimizer != "sgd":
        raise ValueError(f"train_tokens trains with plain SGD only, not optimizer={optimizer!r}: build the model "
                         "with optimizer='sgd', or train (center, context) pairs with step()")
    if not isinstance(window, (int, np.integer)) or int(window) < 1:
        raise ValueError(f"window must be an integer >= 1, got {window!r}")
    if sample > 0 and not has_counts:
        raise ValueError("sample > 0 needs the corpus counts: pass word_counts (or noise_counts) to DeviceSkipGram, "
                         "or sample=0 to keep every word")
    if not torch.is_tensor(tokens) or tokens.dtype not in (torch.int32, torch.int64) or tokens.dim() != 1:
        raise ValueError("tokens must be a 1-D int32 or int64 tensor of word ids (-1 = sentence boundary); "
                         "convert with tokens.to(torch.int64)")


def expected_records(n_tokens: int, window: int, negative: int, cbow: bool = False) -> int:
    """Row pushes a call of ``n_tokens`` is expected to make with no subsampling and no boundaries: every
    center has ``window + 1`` contexts on average (a radius uniform on ``1..window``, both sides), each with
    ``1 + negative`` targets in skip-gram.  A CBOW center pushes its ``1 + negative`` targets once and then every
    context row.  Feeds the replica flush policy without reading device counters."""
    if cbow:
        return max(1, int(n_tokens) * ((1 + int(negative)) + (int(window) + 1)))
    return max(1, int(n_tokens) * (int(window) + 1) * (1 + int(negative)))


class DeviceSkipGram:
    def __init__(self, vocab: int, dim: int = 300, learning_rate: float = 0.025, negative: int = 5,
                 group=None, seed: int = 0, device: Optional[int] = None,
                 replica_cache: Optional[bool] = None, sync_every: int = 4, optimizer: str = "sgd",
                 noise_counts=None, noise_power: float = 0.75, word_counts=None, sample: float = 1e-3):
        """``noise_counts``: ``[vocab]`` word counts.  The negatives are then drawn from ``counts ** noise_power``
        (0.75 is word2vec's choice; words of count 0 are never drawn) by a sampler kernel over an fp64 inverse
        CDF, instead of uniformly over the vocabulary inside the training kernel.  ``None`` = uniform.

        ``word_counts`` (default: ``noise_counts``) are the corpus counts and ``sample`` the threshold of
        word2vec's frequent-word subsampling in :meth:`train_tokens` (``0`` keeps every word); :meth:`step` does
        not subsample."""
        noise = check_noise(noise_counts, vocab, noise_power) if noise_counts is not None else None
        self.sample = check_sample(sample)
        words = _counts(word_counts, vocab, "word_counts") if word_counts is not None else noise
        if optimizer not in ("sgd", "adagrad"):
            raise ValueError(f"optimizer must be 'sgd' or 'adagrad', got {optimizer!r}")
        self.optimizer = optimizer
        ready = dist.is_available() and dist.is_initialized()
        if optimizer == "adagrad" and (replica_cache or (replica_cache is None and ready
                                                         and dist.get_world_size(group) > 1)):
            raise ValueError("optimizer='adagrad' is not supported with the replica cache, the multi-GPU "
                             "default: pass replica_cache=False to read and update the rows on their owners")
        self.vocab, self.dim, self.lr, self.negative, self.seed = vocab, dim, learning_rate, negative, seed
        b = 0.5 / dim
        self.w_in = ShardedTable(vocab, dim, group=group, device=device, init_range=(-b, b), seed=2 * seed + 1)
        self.w_out = ShardedTable(vocab, dim, group=group, device=device, init="zeros")
        self.dev = self.w_in.cuda_device
        self.stats = torch.zeros(2, dtype=torch.float32, device=self.dev)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.step_no = 0
        # multi-GPU: train local replicas of both tables and exchange deltas in the background
        # (store/replica_cache.py) instead of moving 2 x 1200 B per update over NVLink
        if replica_cache is None:
            replica_cache = self.w_in.world > 1
        # row-wise AdaGrad state: one fp32 per row of W_in and of W_out, partitioned like the tables
        self.acc_in = self.w_in.row_accumulators() if optimizer == "adagrad" else None
        self.acc_out = self.w_out.row_accumulators() if optimizer == "adagrad" else None
        self.rep_in = ReplicaCache(self.w_in, sync_every) if replica_cache else None
        self.rep_out = ReplicaCache(self.w_out, sync_every) if replica_cache else None
        self._ones = None
        self._neighbours = None   # most_similar's scorer over the normalised W_in shard
        self._snapshot_step = -1  # step_no the normalised snapshot was taken at
        # unigram noise: the fp64 inverse CDF of counts ** noise_power and the last word it can return
        self.noise_power = float(noise_power)
        self._noise_cdf, self._noise_last = None, 0
        if noise is not None:
            with torch.cuda.device(self.dev):
                self._noise_cdf = native.noise_cdf(torch.from_numpy(noise).to(self.dev), self.noise_power)
            self._noise_last = int(np.flatnonzero(noise > 0)[-1])
        # subsampling: the fp64 keep probability of every word, built once on the host
        self._keep_p = None
        if words is not None and self.sample > 0:
            self._keep_p = torch.from_numpy(keep_probabilities(words, self.sample)).to(self.dev)
        self._has_counts = words is not None
        self.token_stats = torch.zeros(4, dtype=torch.int64, device=self.dev)   # tokens, kept, contexts, dropped
        self._w2v_scratch = None

    def step(self, centers: torch.Tensor, contexts: torch.Tensor) -> None:
        if self._ones is None or self._ones.numel() != centers.numel():
            self._ones = torch.ones(centers.numel(), dtype=torch.float32, device=self.dev)
        tin = self.rep_in.table_c if self.rep_in else self.w_in.table_c
        tout = self.rep_out.table_c if self.rep_out else self.w_out.table_c
        if self.rep_in:   # policy + exchange kernels first (side streams), then the training kernel
            n = centers.numel() * (1 + self.negative)
            self.rep_in.after_step(n); self.rep_out.after_step(n)
        labels, neg = self._ones, self.negative
        if self._noise_cdf is not None and neg > 0:
            # expanded (center, word, label) records: each pair, then its negatives drawn from the noise
            centers, contexts, labels = native.neg_sample_noise(centers, contexts, self._ones, neg, self._noise_cdf,
                                                                self._noise_last, seed=self.seed, step=self.step_no)
            neg = 0
        native.mf_sgd_fused(centers, contexts, labels, tin, 1, tout, self.lr,
                            err_mode=ERR_LOGISTIC, neg_rate=neg, num_items=self.vocab,
                            seed=self.seed, step=self.step_no, stats=self.stats, nan_flag=self.nan_flag,
                            kernel="reg",
                            item_acc=self.acc_out.table_c if self.acc_out else None,
                            user_acc=self.acc_in.table_c if self.acc_in else None,
                            reserve_total=(self.rep_in.reserve_total() + self.rep_out.reserve_total())
                            if self.rep_in else 0)
        self.step_no += 1

    def train_tokens(self, tokens: torch.Tensor, window: int = 5, learning_rate: Optional[float] = None,
                     cbow: bool = False) -> None:
        """Train skip-gram on one micro-batch of text (DESIGN §2.13): ``tokens`` is a 1-D int32 or int64 device
        tensor of word ids, ``-1`` marking a sentence boundary (any other id outside ``[0, vocab)`` is one too, and
        is counted as dropped in :attr:`token_stats`).  Frequent words are subsampled with the rule of word2vec.c,
        each kept center draws a radius on ``1..window`` and trains its contexts within it, never across a
        boundary or the end of the call, against ``negative`` noise words each.

        ``cbow=True`` trains CBOW on the same windows instead (DESIGN §2.14): the mean of a center's context rows
        predicts the center word against ``negative`` noise words, and the error is added, unscaled, to every
        context row, as word2vec.c does.  word2vec.c's default rate for CBOW is 0.05 (0.025 for skip-gram); the
        model's rate is used as given.

        Two launches and no host synchronisation; the call uses and advances :attr:`step_no` like :meth:`step`.
        :attr:`stats` accumulates ``[sum -log sigmoid(+-d), targets trained]`` and :attr:`token_stats` ``[tokens,
        kept, contexts, dropped]``.  ``learning_rate`` overrides the model's rate for this call."""
        check_token_call(tokens, window, self.optimizer, self.sample, self._has_counts, cbow)
        if not tokens.is_cuda:
            tokens = tokens.to(self.dev, non_blocking=True)
        n = tokens.numel()
        if self._w2v_scratch is None or self._w2v_scratch[0].numel() < n:
            self._w2v_scratch = native.w2v_scratch(n, self.dev)
        tin = self.rep_in.table_c if self.rep_in else self.w_in.table_c
        tout = self.rep_out.table_c if self.rep_out else self.w_out.table_c
        if self.rep_in:   # policy + exchange kernels first (side streams), then the training kernels
            rec = expected_records(n, window, self.negative, cbow)
            self.rep_in.after_step(rec); self.rep_out.after_step(rec)
        seq, pos, n_comp = native.w2v_subsample(tokens.contiguous(), self.vocab, self._keep_p, seed=self.seed,
                                                step=self.step_no, token_stats=self.token_stats,
                                                scratch=self._w2v_scratch)
        native.w2v_window_fused(seq, pos, n_comp, tin, tout, self.lr if learning_rate is None else learning_rate,
                                window=int(window), negative=self.negative, vocab=self.vocab, seed=self.seed,
                                step=self.step_no, cdf=self._noise_cdf, last_nonzero=self._noise_last,
                                stats=self.stats, token_stats=self.token_stats, nan_flag=self.nan_flag,
                                reserve_total=(self.rep_in.reserve_total() + self.rep_out.reserve_total())
                                if self.rep_in else 0, cbow=cbow)
        self.step_no += 1

    def fit_tokens(self, tokens: torch.Tensor, epochs: int = 1, batch_tokens: int = 1 << 20, window: int = 5,
                   min_learning_rate: Optional[float] = None, cbow: bool = False) -> None:
        """Train on a whole corpus: ``tokens`` (a device tensor, or a host tensor, pinned for asynchronous copies)
        is cut into calls of ``batch_tokens`` tokens, ``epochs`` times over, through :meth:`train_tokens`.  The
        rate decays linearly over all tokens of all epochs, as in word2vec.c, from the model's rate to
        ``min_learning_rate`` (default ``lr * 1e-4``), each call taking the rate at its first token.  ``cbow``
        selects CBOW as in :meth:`train_tokens`."""
        if int(epochs) < 1 or int(batch_tokens) < 1:
            raise ValueError("epochs and batch_tokens must be >= 1")
        check_token_call(tokens, window, self.optimizer, self.sample, self._has_counts, cbow)
        floor = self.lr * 1e-4 if min_learning_rate is None else float(min_learning_rate)
        n = tokens.numel()
        total = max(1, n * int(epochs))
        done = 0
        for _ in range(int(epochs)):
            for lo in range(0, n, int(batch_tokens)):
                batch = tokens[lo:lo + int(batch_tokens)]
                lr = max(floor, self.lr * (1.0 - done / total))
                self.train_tokens(batch, window=window, learning_rate=lr, cbow=cbow)
                done += batch.numel()

    def flush(self) -> None:
        if self.rep_in:
            self.rep_in.flush(); self.rep_out.flush()

    def similarity(self, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        self.flush()
        va, vb = self.w_in.pull(a), self.w_in.pull(b)
        return torch.nn.functional.cosine_similarity(va, vb)

    def most_similar(self, words: torch.Tensor, K: int = 10):
        """Cosine nearest neighbours of each query word among the input embeddings ``W_in``.

        Returns ``(scores [n, K], word_ids [n, K])``, best first.  The query word itself is never in its
        own list.  Rows with fewer than ``K`` other words end in ``(-3e38, -1)`` entries; a word whose
        vector is zero gets cosine 0 for every neighbour.  Scores come from the TF32 tensor-core top-K
        (``DistributedTopK``): they are within ~1e-3 of the fp32 cosine, and neighbours whose cosines
        differ by less than that may be ordered differently from an fp32 ranking.

        Every rank scores the queries against its own ``W_in`` shard, normalised row by row (a snapshot
        kept until the next :meth:`step`); the queries are the raw rows, pulled by the scoring kernel.
        Ranking by ``q . w / |w|`` is ranking by cosine, so only the K winners are divided by ``|q|``.
        In a multi-rank job the call is collective: every rank passes the same ``words``."""
        from .mf.device_topk import DistributedTopK

        self.flush()
        w = self.w_in
        if w.world > 1:
            w.barrier()                        # every rank's deltas are in the master shards
        if self._snapshot_step != self.step_no:
            ids = w.local_ids()
            n_valid = max(int((ids < self.vocab).sum()), 1)     # slots past the vocabulary are padding
            snap = torch.nn.functional.normalize(w.local[:n_valid], dim=1)  # zero rows stay zero
            if self._neighbours is None:
                self._neighbours = DistributedTopK(w, snap.contiguous(), ids[:n_valid], group=w.group)
            else:                              # the scorer reads the snapshot in place
                self._neighbours.local.items.copy_(snap)
            self._snapshot_step = self.step_no
        q = words.to(self.dev, torch.int64).reshape(-1).contiguous()
        n = q.numel()
        exclude = (torch.arange(n + 1, device=self.dev, dtype=torch.int64), q)   # each query's own id
        sc, ids = self._neighbours.topk(q, K, exclude=exclude)
        if sc.shape[1] < K:                    # a one-rank vocabulary smaller than K
            sc = torch.nn.functional.pad(sc, (0, K - sc.shape[1]), value=-3.0e38)
            ids = torch.nn.functional.pad(ids, (0, K - ids.shape[1]), value=-1)
        qnorm = w.pull(q).norm(dim=1, keepdim=True)
        cos = torch.where(qnorm > 0, sc / qnorm.clamp_min(1e-30), torch.zeros_like(sc))
        return torch.where(ids >= 0, cos, sc), ids

    def score(self, centers: torch.Tensor, contexts: torch.Tensor) -> torch.Tensor:
        """sigmoid(W_in[center] . W_out[context]) -- the model's co-occurrence probability."""
        self.flush()
        u = self.w_in.pull(centers)
        return torch.sigmoid(self.w_out.pull_dot(contexts, torch.nn.functional.pad(
            u, (0, self.w_out.stride - u.shape[1])).contiguous()))

    def check_finite(self):
        if int(self.nan_flag.item()):
            raise FactorIsNotANumberException("non-finite skip-gram update")

    def barrier(self):
        self.flush()
        self.w_in.barrier()

    def close(self):
        gather = getattr(self._neighbours, "_p2p_gather", None)
        if gather is not None:
            gather.close()
        if self.acc_in is not None:
            self.acc_in.close(); self.acc_out.close()
        self.w_in.close(); self.w_out.close()
