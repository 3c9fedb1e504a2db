"""Device tier of the factorization machine (Rendle 2010) on sparse features: one fused CSR kernel per micro-batch.

``DeviceFactorizationMachine`` keeps every parameter in one :class:`ShardedTable` of ``num_features + 1`` rows of
``1 + num_factors`` floats: row ``i`` is ``[w_i | v_i,1 .. v_i,k]`` and row ``num_features`` is the bias row, with
the global bias ``w0`` in column 0.  ``fps_fm_step`` (ops/csrc/fps_fm.cu, DESIGN §2.15) pulls each example's rows,
predicts, and pushes the SGD deltas with ``red.add`` in one launch.  ``num_factors=0`` is sparse linear (squared
loss) or logistic regression.

Both train with plain SGD (``optimizer="sgd"``, the default) or libffm's element-wise AdaGrad (``"adagrad"``, DESIGN
§2.17), whose accumulators live in a second table of the same geometry.

``DeviceFieldAwareFM`` is the field-aware FM (Juan et al. 2016, libffm): every feature keeps one latent vector per
field, and a pair of entries interacts through the vectors each keeps for the other's field.  ``fps_ffm_step``
(ops/csrc/fps_ffm.cu, DESIGN §2.16) runs it one warp per example, pairs spread across lanes.  ``read_libffm``
parses libffm's text format.
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
OPTIMIZERS = ("sgd", "adagrad")


def _check_optimizer(optimizer: str) -> None:
    if optimizer not in OPTIMIZERS:
        raise ValueError(f"optimizer must be one of {list(OPTIMIZERS)}, got {optimizer!r}")


def check_fm_config(num_features: int, num_factors: int, loss: str, reg_linear: float, reg_factors: float,
                    partition: str, replica: bool, optimizer: str = "sgd") -> None:
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
    _check_optimizer(optimizer)


def check_fm_labels(labels: Sequence[Optional[float]], loss: str) -> np.ndarray:
    """The float32 label column of a host batch (``None`` -> NaN, predict only).  Refuses a logistic label outside
    {0, 1} and a non-finite squared-loss label with ``ValueError``."""
    lab = np.array([np.nan if l is None else float(l) for l in labels], dtype=np.float32)
    live = ~np.isnan(lab)
    if loss == "logistic" and ((lab[live] != 0) & (lab[live] != 1)).any():
        raise ValueError(f"logistic labels must be 0 or 1 (NaN predicts); got {lab[live & (lab != 0) & (lab != 1)][:8]}")
    if loss == "squared" and not np.isfinite(lab[live]).all():
        raise ValueError("squared-loss labels must be finite (NaN predicts)")
    return lab


def check_fm_batch(vectors: Sequence[SparseVector], labels: Sequence[Optional[float]], num_features: int,
                   loss: str) -> np.ndarray:
    """The float32 label column of a host batch (``None`` -> NaN, predict only).  Refuses a length mismatch, a
    logistic label outside {0, 1} and a feature id outside ``[0, num_features)`` with ``ValueError``."""
    if len(vectors) != len(labels):
        raise ValueError(f"{len(vectors)} vectors but {len(labels)} labels")
    lab = check_fm_labels(labels, loss)
    for v in vectors:
        if v.activeSize and (int(v.indices.min()) < 0 or int(v.indices.max()) >= num_features):
            raise ValueError(f"feature ids must lie in [0, {num_features}); got "
                             f"[{int(v.indices.min())}, {int(v.indices.max())}]")
    return lab


class _FmState:
    """Observation and IO shared by the factorization machines: the device counters, the ``w0`` state, the
    flags, the table and the AdaGrad accumulators.  Subclasses set ``table``, ``dev`` and ``optimizer`` and call
    ``_alloc_state``."""

    _bad_entry = "a feature id outside [0, {nf}) was skipped"

    def _alloc_state(self) -> None:
        self._stats = torch.zeros(2, dtype=torch.float32, device=self.dev)
        self._flags = torch.zeros(2, dtype=torch.int32, device=self.dev)   # non-finite delta, bad entry
        self._bias_state = native.fm_state(self.dev)
        # AdaGrad's H = G - 1 per element, in the table's geometry: the zero heap is libffm's G = 1
        self._acc = self.table.row_accumulators(self.table.stride) if self.optimizer == "adagrad" else None

    @property
    def _acc_c(self) -> Optional[native.ShardTableC]:
        return self._acc.table_c if self._acc is not None else None

    def accumulators(self) -> Tuple[List[int], np.ndarray]:
        """AdaGrad: ``(ids, H)`` of this rank's rows, ``H`` ``[n, dim]`` in the table's row layout (the element
        ``(id, col)`` is the accumulator of that row's column ``col``).  ``H = G - 1`` in libffm's terms."""
        if self._acc is None:
            raise ValueError("accumulators exist with optimizer='adagrad' only")
        ids, H = self._acc.dump_local()
        return ids.cpu().tolist(), H[:, :self.table.dim].cpu().numpy().astype(np.float64)

    def load_accumulators(self, ids, rows) -> None:
        """Overwrite the accumulators of ``ids`` (rows this rank owns) from ``[n, dim]`` rows, as
        :meth:`accumulators` returns them."""
        if self._acc is None:
            raise ValueError("accumulators exist with optimizer='adagrad' only")
        ids = torch.tensor(list(ids), dtype=torch.int64, device=self.dev)
        if ids.numel() == 0:
            return
        rows = torch.from_numpy(np.ascontiguousarray(rows, dtype=np.float32)).reshape(ids.numel(), self.table.dim)
        full = torch.zeros(ids.numel(), self.table.stride, dtype=torch.float32)
        full[:, :self.table.dim] = rows
        self._acc.load(ids, full.to(self.dev))

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
        """Raise ``FactorIsNotANumberException`` after a non-finite delta and ``IndexError`` after an entry the
        kernel skipped (its feature id, or field, out of range).  One host sync."""
        nan, bad = self._flags.cpu().tolist()
        if bad:
            raise IndexError(self._bad_entry.format(nf=self.num_features, nfields=getattr(self, "num_fields", 0)))
        if nan:
            raise FactorIsNotANumberException("non-finite factorization-machine update")

    def _dump(self, only_nonzero: bool):
        ids, vals = self.table.dump_local(only_touched=False)
        if only_nonzero:
            nz = (vals != 0).any(1)
            ids, vals = ids[nz], vals[nz]
        return ids.cpu().tolist(), vals.cpu().numpy().astype(np.float64)

    def _load(self, ids, rows: np.ndarray) -> None:
        ids = torch.tensor(ids, dtype=torch.int64, device=self.dev)
        self.table.load(ids, torch.from_numpy(np.ascontiguousarray(rows, dtype=np.float32)).to(self.dev))

    def barrier(self) -> None:
        self.table.barrier()

    def close(self) -> None:
        if self._acc is not None:
            self._acc.close()
        self.table.close()


class DeviceFactorizationMachine(_FmState):
    """Factorization machine trained by fused device SGD (DESIGN §2.15).

    ``yhat = w0 + sum_j x_j w_j + 1/2 sum_f ((sum_j x_j v_j,f)^2 - sum_j x_j^2 v_j,f^2)`` over the entries of an
    example; ``loss`` ``"logistic"`` (labels 0 / 1) or ``"squared"``.  Feature rows take plain SGD with lazy L2
    (``reg_linear`` on ``w``, ``reg_factors`` on ``v``) on the rows an entry touches; ``w0`` takes one step per
    micro-batch, the mean gradient of its labelled examples, unregularised (``bias=False`` keeps it at 0).  The
    factors start uniform in ``init_range`` as a pure function of ``(id, seed)``; ``w`` and ``w0`` start at 0.
    ``optimizer="adagrad"`` steps every element of a feature row by ``-lr * gam / sqrt(G)`` with ``G = 1 + sum gam^2``
    over its own gradients (libffm's rule, DESIGN §2.17); ``w0`` keeps the SGD step."""

    def __init__(self, num_features: int, num_factors: int, *, loss: str = "logistic", learning_rate: float = 0.05,
                 reg_linear: float = 0.0, reg_factors: float = 0.0, init_range=(-0.01, 0.01), bias: bool = True,
                 partition: str = "hash", group=None, device: Optional[int] = None, seed: int = 0,
                 replica: bool = False, optimizer: str = "sgd"):
        check_fm_config(num_features, num_factors, loss, reg_linear, reg_factors, partition, replica,
                        optimizer=optimizer)
        self.optimizer = optimizer
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
        self._alloc_state()

    # ---- device front door ---------------------------------------------------------------------------------
    def _launch(self, row_ptr, cols, vals, labels, predict_only: bool) -> torch.Tensor:
        pred = torch.empty(row_ptr.numel() - 1 if row_ptr.numel() else 0, dtype=torch.float32, device=self.dev)
        native.fm_step(self.table.table_c, row_ptr, cols, vals, labels, pred, num_features=self.num_features,
                       loss=self.loss, lr=self.lr, reg_linear=self.reg_linear, reg_factors=self.reg_factors,
                       bias=self.bias, bias_state=self._bias_state, predict_only=predict_only, stats=self._stats,
                       nan_flag=self._flags[0:1], bad_id=self._flags[1:2], acc=self._acc_c)
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

    # ---- model IO ------------------------------------------------------------------------------------------
    def model(self, only_nonzero: bool = True) -> List[Tuple[int, np.ndarray]]:
        """``(id, [w | v_1 .. v_k])`` of this rank's rows; id ``num_features`` is the bias row ``[w0 | 0 ..]``."""
        ids, vals = self._dump(only_nonzero)
        return [(i, v.copy()) for i, v in zip(ids, vals)]

    def load_model(self, model: Iterable[Tuple[int, object]]) -> None:
        """Overwrite the given rows (any rank may load any id)."""
        model = list(model)
        if not model:
            return
        self._load([m[0] for m in model],
                   np.array([np.asarray(m[1], dtype=np.float32).reshape(1 + self.k) for m in model]))


MAX_FFM_FACTORS = native.FFM_MAX_FACTORS
MAX_FFM_FIELDS = native.FFM_MAX_FIELDS


def check_ffm_config(num_features: int, num_fields: int, num_factors: int, loss: str, reg_linear: float,
                     reg_factors: float, partition: str, replica: bool, optimizer: str = "sgd") -> None:
    """The refusals of :class:`DeviceFieldAwareFM`, before any device state exists."""
    if int(num_features) < 1:
        raise ValueError(f"num_features must be >= 1, got {num_features}")
    if not 1 <= int(num_factors) <= MAX_FFM_FACTORS:
        raise ValueError(f"num_factors must lie in [1, {MAX_FFM_FACTORS}], got {num_factors}; for a linear model "
                         f"use DeviceFactorizationMachine(num_factors=0)")
    if not 1 <= int(num_fields) <= MAX_FFM_FIELDS:
        raise ValueError(f"num_fields must lie in [1, {MAX_FFM_FIELDS}], got {num_fields}; hash rarer fields "
                         f"together to fit")
    if loss not in native.FM_LOSSES:
        raise ValueError(f"loss must be one of {sorted(native.FM_LOSSES)}, got {loss!r}")
    if not (float(reg_linear) >= 0 and float(reg_factors) >= 0):
        raise ValueError(f"reg_linear and reg_factors must be >= 0 (0 turns regularisation off); got "
                         f"{reg_linear}, {reg_factors}")
    if partition not in ("hash", "range"):
        raise ValueError(f"partition must be 'hash' or 'range', got {partition!r}")
    if replica:
        raise ValueError("the field-aware FM runs in the direct mode only: use replica=False")
    _check_optimizer(optimizer)


class DeviceFieldAwareFM(_FmState):
    """Field-aware factorization machine trained by fused device SGD (DESIGN §2.16).

    An example is a run of entries ``(field f, feature i, value x)``;
    ``yhat = w0 + sum_a x_a w_a + sum_{a<b} <V[i_a, f_b], V[i_b, f_a]> x_a x_b`` over every pair of its entries in
    order.  ``loss`` ``"logistic"`` (labels 0 / 1) or ``"squared"``.  Plain SGD with lazy L2: ``reg_linear`` on the
    ``w`` of every entry, ``reg_factors`` on both slabs of every pair (libffm's rule); ``w0`` takes one step per
    micro-batch, the mean gradient of its labelled examples (``bias=False`` keeps it at 0).  Row ``i`` of the table
    is ``[w_i | 0 0 0 | V_i,0 | .. | V_i,F-1]``, each slab ``round_up(k, 4)`` floats with zero padding.  The
    factors start uniform in ``init_range`` as a pure function of ``(id, seed)``; ``w`` and ``w0`` start at 0.
    ``optimizer="adagrad"`` is libffm's training rule: every ``w`` and slab element steps by ``-lr * gam / sqrt(G)``,
    ``G = 1 + sum gam^2`` over its own gradients (DESIGN §2.17); ``w0`` keeps the SGD step."""

    _bad_entry = "a feature id outside [0, {nf}) or a field outside [0, {nfields}) was skipped"

    def __init__(self, num_features: int, num_fields: int, num_factors: int, *, loss: str = "logistic",
                 learning_rate: float = 0.05, reg_linear: float = 0.0, reg_factors: float = 0.0,
                 init_range=(-0.01, 0.01), bias: bool = True, partition: str = "hash", group=None,
                 device: Optional[int] = None, seed: int = 0, replica: bool = False, optimizer: str = "sgd"):
        check_ffm_config(num_features, num_fields, num_factors, loss, reg_linear, reg_factors, partition, replica,
                         optimizer=optimizer)
        self.optimizer = optimizer
        self.num_features, self.num_fields, self.k = int(num_features), int(num_fields), int(num_factors)
        self.kp = 4 * -(-self.k // 4)
        self.loss, self.lr = loss, float(learning_rate)
        self.reg_linear, self.reg_factors, self.bias = float(reg_linear), float(reg_factors), bool(bias)
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.dev = torch.device("cuda", self.device)
        stride = native.ffm_stride(self.num_fields, self.k)
        self.table = ShardedTable(self.num_features + 1, stride, partition=partition, group=group,
                                  device=self.device, init="uniform", init_range=init_range, seed=seed)
        if self.table.owns_shard:
            # w, columns 1..3, every slab's padding and the whole bias row start at 0: a pure function of the id,
            # so every rank count starts equal, and the padding stays 0
            loc = self.table.local
            loc[:, 0:4] = 0.0
            loc[:, 4:].view(loc.shape[0], self.num_fields, self.kp)[:, :, self.k:] = 0.0
            loc[self.table.local_ids() == self.num_features] = 0.0
        self.table.barrier()
        self._alloc_state()

    # ---- device front door ---------------------------------------------------------------------------------
    def _launch(self, row_ptr, cols, fields, vals, labels, predict_only: bool) -> torch.Tensor:
        pred = torch.empty(row_ptr.numel() - 1 if row_ptr.numel() else 0, dtype=torch.float32, device=self.dev)
        native.ffm_step(self.table.table_c, row_ptr, cols, fields, vals, labels, pred,
                        num_features=self.num_features, num_fields=self.num_fields, num_factors=self.k,
                        loss=self.loss, lr=self.lr, reg_linear=self.reg_linear, reg_factors=self.reg_factors,
                        bias=self.bias, bias_state=self._bias_state, predict_only=predict_only, stats=self._stats,
                        nan_flag=self._flags[0:1], bad_id=self._flags[1:2], acc=self._acc_c)
        return pred

    def step_csr(self, row_ptr: torch.Tensor, cols: torch.Tensor, fields: torch.Tensor,
                 vals: Optional[torch.Tensor], labels: torch.Tensor) -> torch.Tensor:
        """One micro-batch, one launch, no host sync.  ``row_ptr`` int64 ``[n + 1]``, ``cols`` int32 / int64,
        ``fields`` int32, ``vals`` float32 or ``None`` (one-hot), ``labels`` float32 ``[n]`` (NaN: predict only).
        Returns the raw scores ``yhat`` from before each example's own update (progressive validation)."""
        return self._launch(row_ptr, cols, fields, vals, labels, False)

    def predict_csr(self, row_ptr: torch.Tensor, cols: torch.Tensor, fields: torch.Tensor,
                    vals: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Raw scores ``yhat`` of a CSR batch; nothing is pushed and ``stats`` do not move."""
        return self._launch(row_ptr, cols, fields, vals, None, True)

    def step(self, examples: Sequence[Sequence[Tuple[int, int, float]]],
             labels: Sequence[Optional[float]]) -> List[float]:
        """One micro-batch from the host, each example a sequence of ``(field, feature, value)`` triples (libffm's
        order); ``None`` labels only predict.  Bad labels, features and fields are refused before anything is
        copied."""
        if len(examples) != len(labels):
            raise ValueError(f"{len(examples)} examples but {len(labels)} labels")
        lab = check_fm_labels(labels, self.loss)
        n = len(examples)
        row_ptr = np.zeros(n + 1, dtype=np.int64)
        for i, ex in enumerate(examples):
            row_ptr[i + 1] = row_ptr[i] + len(ex)
        trip = np.array([t for ex in examples for t in ex], dtype=np.float64).reshape(-1, 3)
        fields, cols, vals = trip[:, 0].astype(np.int64), trip[:, 1].astype(np.int64), trip[:, 2]
        if len(cols) and (cols.min() < 0 or cols.max() >= self.num_features):
            raise ValueError(f"feature ids must lie in [0, {self.num_features}); got [{cols.min()}, {cols.max()}]")
        if len(fields) and (fields.min() < 0 or fields.max() >= self.num_fields):
            raise ValueError(f"fields must lie in [0, {self.num_fields}); got [{fields.min()}, {fields.max()}]")
        to = lambda x: torch.from_numpy(x).to(self.dev, non_blocking=True)
        return self.step_csr(to(row_ptr), to(cols), to(fields.astype(np.int32)), to(vals.astype(np.float32)),
                             to(lab)).cpu().tolist()

    # ---- model IO ------------------------------------------------------------------------------------------
    def model(self, only_nonzero: bool = True) -> List[Tuple[int, float, np.ndarray]]:
        """``(id, w, V[num_fields, k])`` of this rank's rows, padding stripped; id ``num_features`` is the bias
        row, ``w0`` in ``w``."""
        ids, vals = self._dump(only_nonzero)
        V = vals[:, 4:].reshape(len(ids), self.num_fields, self.kp)[:, :, :self.k]
        return [(i, float(vals[j, 0]), V[j].copy()) for j, i in enumerate(ids)]

    def load_model(self, model: Iterable[Tuple[int, float, object]]) -> None:
        """Overwrite the given rows from ``(id, w, V[num_fields, k])`` (any rank may load any id)."""
        model = list(model)
        if not model:
            return
        rows = np.zeros((len(model), native.ffm_stride(self.num_fields, self.k)), dtype=np.float32)
        for j, (_, w, V) in enumerate(model):
            rows[j, 0] = w
            rows[j, 4:].reshape(self.num_fields, self.kp)[:, :self.k] = np.asarray(V, dtype=np.float32).reshape(
                self.num_fields, self.k)
        self._load([m[0] for m in model], rows)


def read_libffm(lines_or_path) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Parse libffm's text format, one example per line: ``label field:feature:value ...``.  ``lines_or_path``: a
    path or an iterable of lines; blank lines are skipped.  Returns numpy CSR ``(row_ptr int64 [n + 1], fields
    int32, cols int64, vals float32, labels float32 [n])``.  A malformed token raises ``ValueError`` naming its
    line; bounds are the model's to check."""
    if isinstance(lines_or_path, (str, bytes)) or hasattr(lines_or_path, "__fspath__"):
        with open(lines_or_path) as f:
            lines = f.read().splitlines()
    else:
        lines = list(lines_or_path)
    row_ptr, fields, cols, vals, labels = [0], [], [], [], []
    for no, line in enumerate(lines, 1):
        tok = line.split()
        if not tok:
            continue
        try:
            labels.append(float(tok[0]))
            for t in tok[1:]:
                f, i, v = t.split(":")
                fields.append(int(f))
                cols.append(int(i))
                vals.append(float(v))
        except ValueError:
            raise ValueError(f"line {no}: malformed libffm example {line.strip()!r} (want 'label field:feature:value "
                             f"...')") from None
        row_ptr.append(len(cols))
    return (np.array(row_ptr, np.int64), np.array(fields, np.int32), np.array(cols, np.int64),
            np.array(vals, np.float32), np.array(labels, np.float32))


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
