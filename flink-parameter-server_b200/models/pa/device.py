"""Device tier of the passive-aggressive classifiers: one fused CSR kernel per micro-batch.

``DevicePassiveAggressive`` keeps the per-feature parameters in a :class:`ShardedTable` (hash or
range partitioned over the PS ranks, PassiveAggressiveParameterServer.scala:262-281) and runs
``fps_pa_step`` (ops/csrc/fps_pa.cu): per example nnz pulls + sparse dot + update rule + nnz pushes,
all inside the kernel through peer-mapped shard pointers.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ...api import Left, Right
from ...errors import FactorIsNotANumberException
from ...ops import native
from ...runtime.stream import ResultStream, as_stream
from ...store.sharded_table import ShardedTable
from .algorithms import (PassiveAggressiveBinaryAlgorithmImpl, PassiveAggressiveBinaryAlgorithmImplI,
                         PassiveAggressiveBinaryAlgorithmImplII, PassiveAggressiveCostBasedImplML,
                         PassiveAggressiveCostBasedImplPB, PassiveAggressiveOneVersusAllImpl,
                         PassiveAggressiveOneVersusAllImplI, PassiveAggressiveOneVersusAllImplII)
from .sparse import SparseVector


def algo_to_device(algo) -> Tuple[str, float, Optional[np.ndarray]]:
    """Map a host algorithm object to (kernel algo name, aggressiveness, cost matrix)."""
    if isinstance(algo, (PassiveAggressiveBinaryAlgorithmImpl, PassiveAggressiveOneVersusAllImpl)):
        return "PA", 0.0, None
    if isinstance(algo, (PassiveAggressiveBinaryAlgorithmImplI, PassiveAggressiveOneVersusAllImplI)):
        return "PAI", algo.aggressiveness, None
    if isinstance(algo, (PassiveAggressiveBinaryAlgorithmImplII, PassiveAggressiveOneVersusAllImplII)):
        return "PAII", algo.aggressiveness, None
    if isinstance(algo, (PassiveAggressiveCostBasedImplPB, PassiveAggressiveCostBasedImplML)):
        L = algo.labelCount
        cost = np.array([[algo.cost(i, j) for j in range(L)] for i in range(L)], dtype=np.float32)
        return ("PB" if isinstance(algo, PassiveAggressiveCostBasedImplPB) else "ML"), 0.0, cost
    raise TypeError(f"no device kernel for {type(algo).__name__}")


MAX_LABELS = 1024  # PA_MAX_LABELS of ops/csrc/fps_pa.cu


def labels_array(labels: Sequence[Optional[int]], binary: bool, num_labels: int) -> np.ndarray:
    """The int32 label column of one micro-batch: ``None`` -> ``native.PA_UNLABELLED`` (predict only).
    A binary label must be +1 or -1 and a class index must lie in ``[0, num_labels)``; anything else raises
    ``ValueError``.  The kernels index their decision vector and the cost matrix with the label, and a
    binary ``0`` (``int(False)``) would train towards no target at all."""
    lab = np.array([native.PA_UNLABELLED if l is None else int(l) for l in labels], dtype=np.int64)
    live = lab != native.PA_UNLABELLED
    if binary:
        wrong = live & (lab != 1) & (lab != -1)
        what = "binary labels must be +1 or -1"
    else:
        wrong = live & ((lab < 0) | (lab >= num_labels))
        what = f"class labels must lie in [0, {num_labels})"
    if wrong.any():
        raise ValueError(f"{what}; got {lab[wrong][:8].tolist()}")
    return lab.astype(np.int32)


class DevicePassiveAggressive:
    def __init__(self, feature_count: int, num_labels: int = 1, binary: bool = True, algo: str = "PA",
                 aggressiveness: float = 0.0, cost: Optional[np.ndarray] = None,
                 range_partitioning: bool = False, group=None, device: Optional[int] = None):
        if not binary and not 1 <= int(num_labels) <= MAX_LABELS:
            raise ValueError(f"num_labels must lie in [1, {MAX_LABELS}]; got {num_labels}")
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.dev = torch.device("cuda", self.device)
        self.binary, self.L, self.algo, self.C = binary, (1 if binary else num_labels), algo, aggressiveness
        self.table = ShardedTable(feature_count, self.L, partition="range" if range_partitioning else "hash",
                                  group=group, device=self.device, init="zeros", track_touched=True)
        self.cost = torch.as_tensor(cost, dtype=torch.float32, device=self.dev).contiguous() \
            if cost is not None else None
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=self.dev)

    def step_csr(self, row_ptr: torch.Tensor, cols: torch.Tensor, vals: torch.Tensor,
                 labels: torch.Tensor) -> torch.Tensor:
        """One micro-batch; ``labels``: binary +-1 / class index / ``native.PA_UNLABELLED``.
        Returns predictions (made with the parameters *before* each example's own update).
        The labels are not checked here (that would wait for the device): the caller guarantees +-1 for a
        binary model and ``[0, num_labels)`` for a multiclass one.  :meth:`step` checks them."""
        pred = torch.empty(labels.numel(), dtype=torch.int32, device=self.dev)
        # mark every referenced feature as touched (what close() dumps)
        if self.table.track_touched:
            pass
        native.pa_step(self.table.table_c, row_ptr, cols, vals, labels, pred, binary=self.binary,
                       num_labels=self.L, algo=self.algo, aggressiveness=self.C, cost=self.cost,
                       nan_flag=self.nan_flag)
        return pred

    def step(self, vectors: Sequence[SparseVector], labels: Sequence[Optional[int]]) -> List[int]:
        """One micro-batch from the host; ``None`` labels only predict.  Refuses bad labels before any copy."""
        lab = labels_array(labels, self.binary, self.L)
        n = len(vectors)
        row_ptr = np.zeros(n + 1, dtype=np.int64)
        for i, v in enumerate(vectors):
            row_ptr[i + 1] = row_ptr[i] + v.activeSize
        cols = np.concatenate([v.indices for v in vectors]).astype(np.int32) if n else np.zeros(0, np.int32)
        vals = np.concatenate([v.values for v in vectors]).astype(np.float32) if n else np.zeros(0, np.float32)
        to = lambda x: torch.from_numpy(x).to(self.dev, non_blocking=True)
        pred = self.step_csr(to(row_ptr), to(cols), to(vals), to(lab))
        return pred.cpu().tolist()

    def model(self, only_nonzero: bool = True) -> List[Tuple[int, object]]:
        ids, vals = self.table.dump_local(only_touched=False)
        if only_nonzero:
            nz = (vals != 0).any(1)
            ids, vals = ids[nz], vals[nz]
        ids, vals = ids.cpu().tolist(), vals.cpu().numpy().astype(np.float64)
        if self.binary:
            return [(i, float(v[0])) for i, v in zip(ids, vals)]
        return [(i, v.copy()) for i, v in zip(ids, vals)]

    def load_model(self, model: Iterable[Tuple[int, object]]) -> None:
        model = list(model)
        if not model:
            return
        ids = torch.tensor([m[0] for m in model], dtype=torch.int64, device=self.dev)
        vals = torch.tensor(np.array([np.atleast_1d(np.asarray(m[1], dtype=np.float32)) for m in model]),
                            device=self.dev)
        self.table.load(ids, vals.contiguous())

    def check_finite(self):
        if int(self.nan_flag.item()):
            raise FactorIsNotANumberException("non-finite passive-aggressive update")

    def close(self):
        self.table.close()


def _run_device(model, inputSource, pa: DevicePassiveAggressive, batch_size: int, label_of, id_of):
    if model is not None:
        pa.load_model(as_stream(model).collect())
        pa.table.barrier()
    results = []
    buf = []

    def flush():
        if not buf:
            return
        vecs = [(d.value[0] if d.is_left else d.value[1]) for d in buf]
        labels = [label_of(d) if d.is_left else None for d in buf]
        preds = pa.step(vecs, labels)
        for d, p in zip(buf, preds):
            if not d.is_left:
                results.append(Left((id_of(d), p)))
        buf.clear()

    for rec in as_stream(inputSource).collect():
        buf.append(rec)
        if len(buf) >= batch_size:
            flush()
    flush()
    pa.check_finite()
    pa.table.barrier()
    for kv in pa.model():
        results.append(Right(kv))
    out = ResultStream(results)
    out.device_model = pa
    return out


def transform_binary_device(model, inputSource, algo, featureCount, rangePartitioning=False,
                            pullLimit: int = 0, batch_size: int = 256, group=None):
    name, C, _ = algo_to_device(algo)
    pa = DevicePassiveAggressive(featureCount, 1, True, name, C, None, rangePartitioning, group)
    return _run_device(model, inputSource, pa, batch_size,
                       lambda d: 1 if d.value[1] else -1,
                       lambda d: d.value[1])


def transform_multiclass_device(model, inputSource, algo, labelCount, featureCount,
                                rangePartitioning=False, pullLimit: int = 0, batch_size: int = 256,
                                group=None, long_id: bool = False):
    name, C, cost = algo_to_device(algo)
    pa = DevicePassiveAggressive(featureCount, labelCount, False, name, C, cost, rangePartitioning, group)
    return _run_device(model, inputSource, pa, batch_size, lambda d: int(d.value[1]),
                       (lambda d: d.value[0]) if long_id else (lambda d: d.value[1]))
