"""Device tier of the factorization machine (Rendle 2010) on sparse features: one fused CSR kernel per micro-batch.

``DeviceFactorizationMachine`` keeps every parameter in one :class:`ShardedTable` of ``num_features + 1`` rows of
``1 + num_factors`` floats: row ``i`` is ``[w_i | v_i,1 .. v_i,k]`` and row ``num_features`` is the bias row, with
the global bias ``w0`` in column 0.  ``fps_fm_step`` (ops/csrc/fps_fm.cu, DESIGN §2.15) pulls each example's rows,
predicts, and pushes the SGD deltas with ``red.add`` in one launch.  ``num_factors=0`` is sparse linear (squared
loss) or logistic regression.
"""
from __future__ import annotations

import math
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..errors import FactorIsNotANumberException
from ..ops import native
from ..store.sharded_table import ShardedTable
from .pa.sparse import SparseVector

MAX_FACTORS = native.FM_MAX_DIM - 1


def check_fm_config(num_features: int, num_factors: int, loss: str, reg_linear: float, reg_factors: float,
                    partition: str, replica: bool) -> None:
    """The refusals of :class:`DeviceFactorizationMachine`, before any device state exists."""
    if int(num_features) < 1:
        raise ValueError(f"num_features must be >= 1, got {num_features}")
    if not 0 <= int(num_factors) <= MAX_FACTORS:
        raise ValueError(f"num_factors must lie in [0, {MAX_FACTORS}] (rows of 1 + k floats, at most "
                         f"{native.FM_MAX_DIM}); got {num_factors}")
    if loss not in native.FM_LOSSES:
        raise ValueError(f"loss must be one of {sorted(native.FM_LOSSES)}, got {loss!r}")
    if not (float(reg_linear) >= 0 and float(reg_factors) >= 0):
        raise ValueError(f"reg_linear and reg_factors must be >= 0 (0 turns regularisation off); got "
                         f"{reg_linear}, {reg_factors}")
    if partition not in ("hash", "range"):
        raise ValueError(f"partition must be 'hash' or 'range', got {partition!r}")
    if replica:
        raise ValueError("the factorization machine runs in the direct mode only: use replica=False")


def check_fm_batch(vectors: Sequence[SparseVector], labels: Sequence[Optional[float]], num_features: int,
                   loss: str) -> np.ndarray:
    """The float32 label column of a host batch (``None`` -> NaN, predict only).  Refuses a length mismatch, a
    logistic label outside {0, 1} and a feature id outside ``[0, num_features)`` with ``ValueError``."""
    if len(vectors) != len(labels):
        raise ValueError(f"{len(vectors)} vectors but {len(labels)} labels")
    lab = np.array([np.nan if l is None else float(l) for l in labels], dtype=np.float32)
    live = ~np.isnan(lab)
    if loss == "logistic" and ((lab[live] != 0) & (lab[live] != 1)).any():
        raise ValueError(f"logistic labels must be 0 or 1 (NaN predicts); got {lab[live & (lab != 0) & (lab != 1)][:8]}")
    if loss == "squared" and not np.isfinite(lab[live]).all():
        raise ValueError("squared-loss labels must be finite (NaN predicts)")
    for v in vectors:
        if v.activeSize and (int(v.indices.min()) < 0 or int(v.indices.max()) >= num_features):
            raise ValueError(f"feature ids must lie in [0, {num_features}); got "
                             f"[{int(v.indices.min())}, {int(v.indices.max())}]")
    return lab


class DeviceFactorizationMachine:
    """Factorization machine trained by fused device SGD (DESIGN §2.15).

    ``yhat = w0 + sum_j x_j w_j + 1/2 sum_f ((sum_j x_j v_j,f)^2 - sum_j x_j^2 v_j,f^2)`` over the entries of an
    example; ``loss`` ``"logistic"`` (labels 0 / 1) or ``"squared"``.  Feature rows take plain SGD with lazy L2
    (``reg_linear`` on ``w``, ``reg_factors`` on ``v``) on the rows an entry touches; ``w0`` takes one step per
    micro-batch, the mean gradient of its labelled examples, unregularised (``bias=False`` keeps it at 0).  The
    factors start uniform in ``init_range`` as a pure function of ``(id, seed)``; ``w`` and ``w0`` start at 0."""

    def __init__(self, num_features: int, num_factors: int, *, loss: str = "logistic", learning_rate: float = 0.05,
                 reg_linear: float = 0.0, reg_factors: float = 0.0, init_range=(-0.01, 0.01), bias: bool = True,
                 partition: str = "hash", group=None, device: Optional[int] = None, seed: int = 0,
                 replica: bool = False):
        check_fm_config(num_features, num_factors, loss, reg_linear, reg_factors, partition, replica)
        self.num_features, self.k = int(num_features), int(num_factors)
        self.loss, self.lr = loss, float(learning_rate)
        self.reg_linear, self.reg_factors, self.bias = float(reg_linear), float(reg_factors), bool(bias)
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.dev = torch.device("cuda", self.device)
        self.table = ShardedTable(self.num_features + 1, 1 + self.k, partition=partition, group=group,
                                  device=self.device, init="uniform", init_range=init_range, seed=seed)
        if self.table.owns_shard:
            # w and the whole bias row start at 0: a pure function of the id, so every rank count starts equal
            self.table.local[:, 0] = 0.0
            self.table.local[self.table.local_ids() == self.num_features] = 0.0
        self.table.barrier()
        self._stats = torch.zeros(2, dtype=torch.float32, device=self.dev)
        self._flags = torch.zeros(2, dtype=torch.int32, device=self.dev)   # non-finite delta, bad feature id
        self._bias_state = native.fm_state(self.dev)

    # ---- device front door ---------------------------------------------------------------------------------
    def _launch(self, row_ptr, cols, vals, labels, predict_only: bool) -> torch.Tensor:
        pred = torch.empty(row_ptr.numel() - 1 if row_ptr.numel() else 0, dtype=torch.float32, device=self.dev)
        native.fm_step(self.table.table_c, row_ptr, cols, vals, labels, pred, num_features=self.num_features,
                       loss=self.loss, lr=self.lr, reg_linear=self.reg_linear, reg_factors=self.reg_factors,
                       bias=self.bias, bias_state=self._bias_state, predict_only=predict_only, stats=self._stats,
                       nan_flag=self._flags[0:1], bad_id=self._flags[1:2])
        return pred

    def step_csr(self, row_ptr: torch.Tensor, cols: torch.Tensor, vals: Optional[torch.Tensor],
                 labels: torch.Tensor) -> torch.Tensor:
        """One micro-batch, one launch, no host sync.  ``row_ptr`` int64 ``[n + 1]``, ``cols`` int32 / int64,
        ``vals`` float32 or ``None`` (one-hot), ``labels`` float32 ``[n]`` (NaN: predict only).  Returns the raw
        scores ``yhat`` from before each example's own update (progressive validation)."""
        return self._launch(row_ptr, cols, vals, labels, False)

    def predict_csr(self, row_ptr: torch.Tensor, cols: torch.Tensor,
                    vals: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Raw scores ``yhat`` of a CSR batch; nothing is pushed and ``stats`` do not move."""
        return self._launch(row_ptr, cols, vals, None, True)

    def step(self, vectors: Sequence[SparseVector], labels: Sequence[Optional[float]]) -> List[float]:
        """One micro-batch from the host; ``None`` labels only predict.  Bad labels and feature ids are refused
        before anything is copied."""
        lab = check_fm_batch(vectors, labels, self.num_features, self.loss)
        n = len(vectors)
        row_ptr = np.zeros(n + 1, dtype=np.int64)
        for i, v in enumerate(vectors):
            row_ptr[i + 1] = row_ptr[i] + v.activeSize
        cols = np.concatenate([v.indices for v in vectors]).astype(np.int64) if n else np.zeros(0, np.int64)
        vals = np.concatenate([v.values for v in vectors]).astype(np.float32) if n else np.zeros(0, np.float32)
        to = lambda x: torch.from_numpy(x).to(self.dev, non_blocking=True)
        return self.step_csr(to(row_ptr), to(cols), to(vals), to(lab)).cpu().tolist()

    # ---- observation -----------------------------------------------------------------------------------------
    @property
    def stats(self) -> torch.Tensor:
        """Device float32 ``[loss sum, labelled examples]`` since construction (or the caller's last ``zero_``):
        logistic: ``sum softplus(yhat) - y yhat``; squared: ``sum (yhat - y)^2`` (RMSE = sqrt(s[0] / s[1]))."""
        return self._stats

    @property
    def bias_pushed(self) -> float:
        """Sum of the ``w0`` deltas this process has pushed (one host sync)."""
        return float(self._bias_state[0][3].item())

    def check(self) -> None:
        """Raise ``FactorIsNotANumberException`` after a non-finite delta and ``IndexError`` after an entry whose
        feature id was outside ``[0, num_features)`` (such entries are skipped).  One host sync."""
        nan, bad = self._flags.cpu().tolist()
        if bad:
            raise IndexError(f"a feature id outside [0, {self.num_features}) was skipped")
        if nan:
            raise FactorIsNotANumberException("non-finite factorization-machine update")

    def model(self, only_nonzero: bool = True) -> List[Tuple[int, np.ndarray]]:
        """``(id, [w | v_1 .. v_k])`` of this rank's rows; id ``num_features`` is the bias row ``[w0 | 0 ..]``."""
        ids, vals = self.table.dump_local(only_touched=False)
        if only_nonzero:
            nz = (vals != 0).any(1)
            ids, vals = ids[nz], vals[nz]
        ids, vals = ids.cpu().tolist(), vals.cpu().numpy().astype(np.float64)
        return [(i, v.copy()) for i, v in zip(ids, vals)]

    def load_model(self, model: Iterable[Tuple[int, object]]) -> None:
        """Overwrite the given rows (any rank may load any id)."""
        model = list(model)
        if not model:
            return
        ids = torch.tensor([m[0] for m in model], dtype=torch.int64, device=self.dev)
        vals = torch.tensor(np.array([np.asarray(m[1], dtype=np.float32).reshape(1 + self.k) for m in model]),
                            device=self.dev)
        self.table.load(ids, vals.contiguous())

    def barrier(self) -> None:
        self.table.barrier()

    def close(self) -> None:
        self.table.close()


def roc_auc(scores, labels) -> float:
    """Area under the ROC curve of ``scores`` for 0 / 1 ``labels`` (ties share their rank)."""
    s = np.asarray(scores, dtype=np.float64)
    y = np.asarray(labels) > 0.5
    n_pos, n_neg = int(y.sum()), int((~y).sum())
    if n_pos == 0 or n_neg == 0:
        return math.nan
    order = np.argsort(s, kind="mergesort")
    _, first, counts = np.unique(s[order], return_index=True, return_counts=True)
    ranks = np.empty(len(s))
    ranks[order] = np.repeat(first + 0.5 * (counts - 1) + 1.0, counts)
    return float((ranks[y].sum() - n_pos * (n_pos + 1) / 2.0) / (n_pos * n_neg))
