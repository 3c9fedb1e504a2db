"""``FlinkParameterServer.transform*`` -- the library entry points (layer L1, FPS:64-1173).

Every reference overload is available through :func:`transform`, dispatched on its arguments:

====================================================================  ========================
call                                                                  reference
====================================================================  ========================
``transform(data, wl, paramInit, paramUpdate, wP, psP, wait)``         C1  FPS:64-80
``transformLoose(data, wl, paramInit, paramUpdate, wP, psP, wait)``    C2  FPS:122-139
``transform(data, wl, psLogic, wP, psP, wait)``                        C3/C4 FPS:172-292
``transform(data, wl, psLogic, paramPartitioner, wInPartition, wP,     C5/C6 FPS:340-672
 psP, workerReceiver, workerSender, psReceiver, psSender, wait)``
``transformWithModelLoad(model)(data, wl, psLogic, ...)``              C9  FPS:715-908
``transformWithDoubleModelLoad(model)(data, wl, psLogic, ...)``        C10 FPS:950-1173
====================================================================  ========================

The returned :class:`ResultStream` is the ``DataStream[Either[WOut, PSOut]]`` of the reference:
``Left`` = worker outputs, ``Right`` = PS outputs.

Backends: ``backend="local"`` runs the callbacks on the in-process asynchronous engine (host
tier); declarative device logics (``runtime.device_engine``) run on the fused GPU tier.
"""
from __future__ import annotations

from typing import Any, Callable, List, Optional, Tuple

from ..api import (LooseParameterServerLogic, LooseWorkerLogic, ParameterServer,
                   ParameterServerClient, ParameterServerLogic, RuntimeContext, WorkerLogic)
from ..parallel.partitioner import HashPartitioner, as_partitioner, stable_hash
from ..protocol.messages import PSToWorker, PullAnswer, WorkerToPS
from ..protocol.senders import (SimplePSReceiver, SimplePSSender, SimpleWorkerReceiver,
                                SimpleWorkerSender)
from ..server.logics import LooseSimplePSLogic, SimplePSLogic
from .local_engine import LocalEngine
from .stream import DataStream, ResultStream, as_stream

DEFAULT_ITERATION_WAIT_TIME = 10000  # ms, like the reference's algorithm defaults


# ------------------------------------------------------------------------------------------
# default partitioners (FPS:191-203)
# ------------------------------------------------------------------------------------------
def _first(msg):
    """Batched messages are routed by their (homogeneous) first element."""
    return msg[0] if isinstance(msg, (list, tuple)) else msg


def default_param_partitioner(psParallelism: int) -> Callable[[Any], int]:
    def part(msg) -> int:
        m = _first(msg)
        return stable_hash(m.paramId) % psParallelism

    part.fps_default = "hash"        # lets the engine route by id without building a message (local_engine.py)
    return part


def default_worker_partitioner(workerParallelism: int) -> Callable[[Any], int]:
    def part(msg) -> int:
        return _first(msg).workerPartitionIndex

    part.fps_default = "worker_index"
    return part


# ------------------------------------------------------------------------------------------
# the fully general engine call (C5 / C6)
# ------------------------------------------------------------------------------------------
def device_ps_logic(psLogic, backend: str):
    """``backend="device"``: swap a built-in host store for its device-resident twin
    (server/device_logics.py).  User-defined server logics are arbitrary Python and stay on the host."""
    if backend in (None, "local", "host"):
        return psLogic
    if backend != "device":
        raise ValueError(f"unknown backend {backend!r} (local | device)")
    from ..server.device_logics import to_device_logic

    inner = psLogic
    dev = to_device_logic(inner)
    if dev is None:
        import warnings

        warnings.warn(f"{type(psLogic).__name__} is user-defined server code: it runs on the host tier; "
                      "only the built-in stores (Simple / Loose / Range / Lock) are device-resident",
                      RuntimeWarning, stacklevel=3)
        return psLogic
    return dev


def transform_general(trainingData, workerLogic: LooseWorkerLogic,
                      psLogic: LooseParameterServerLogic,
                      paramPartitioner: Callable[[Any], int], wInPartition: Callable[[Any], int],
                      workerParallelism: int, psParallelism: int, workerReceiver, workerSender,
                      psReceiver, psSender, iterationWaitTime: float = DEFAULT_ITERATION_WAIT_TIME,
                      call_worker_open: bool = True) -> ResultStream:
    # device-resident stores keep the general engine path (the one validated on the GPU); host stores with the
    # stock protocol take the engine's fast path
    on_device = type(psLogic).__name__ == "DeviceStoreLogic" and not getattr(psLogic, "emulate", False)
    engine = LocalEngine(workerParallelism, psParallelism, iterationWaitTime,
                         call_worker_open=call_worker_open, fast_path=False if on_device else None)
    out = engine.run(trainingData, workerLogic, psLogic, paramPartitioner, wInPartition,
                     workerReceiver, workerSender, psReceiver, psSender)
    out.engine = engine
    return out


def transform(trainingData, workerLogic, *args, **kw) -> ResultStream:
    """Dispatching front door; see the module docstring for the accepted forms."""
    names_general = ["psLogic", "paramPartitioner", "wInPartition", "workerParallelism",
                     "psParallelism", "workerReceiver", "workerSender", "psReceiver", "psSender",
                     "iterationWaitTime"]
    names_logic = ["psLogic", "workerParallelism", "psParallelism", "iterationWaitTime"]
    names_fn = ["paramInit", "paramUpdate", "workerParallelism", "psParallelism",
                "iterationWaitTime"]
    backend = kw.pop("backend", "local")
    from ..api import BatchedWorkerLogic

    if isinstance(workerLogic, BatchedWorkerLogic):
        if backend != "device":
            raise ValueError('a BatchedWorkerLogic runs on the device tensor tier: pass backend="device"')
        from .device_engine import transform_batched

        return transform_batched(trainingData, workerLogic, *args, **kw)
    first = args[0] if args else None
    if isinstance(first, LooseParameterServerLogic) or "psLogic" in kw:
        second = args[1] if len(args) > 1 else None
        general = (len(args) > 1 and callable(second) and not isinstance(second, int)) or \
            "paramPartitioner" in kw or "workerSender" in kw or "psSender" in kw
        names = names_general if general else names_logic
    else:
        names = names_fn
    if len(args) > len(names):
        raise TypeError("too many positional arguments for transform")
    params = dict(zip(names, args))
    for k, v in kw.items():
        if k in params:
            raise TypeError(f"transform got multiple values for {k}")
        params[k] = v
    wait = params.get("iterationWaitTime", DEFAULT_ITERATION_WAIT_TIME)
    wP, psP = int(params["workerParallelism"]), int(params["psParallelism"])
    if "paramInit" in params:
        loose = bool(params.pop("loose", False))
        cls = LooseSimplePSLogic if loose else SimplePSLogic
        psLogic = cls(params["paramInit"], params["paramUpdate"])
    else:
        psLogic = params["psLogic"]
    psLogic = device_ps_logic(psLogic, backend)
    return transform_general(
        trainingData, workerLogic, psLogic,
        params.get("paramPartitioner") or default_param_partitioner(psP),
        params.get("wInPartition") or default_worker_partitioner(wP),
        wP, psP,
        params.get("workerReceiver") or SimpleWorkerReceiver(),
        params.get("workerSender") or SimpleWorkerSender(),
        params.get("psReceiver") or SimplePSReceiver(),
        params.get("psSender") or SimplePSSender(),
        wait)


def transformLoose(trainingData, workerLogic, paramInit, paramUpdate, workerParallelism,
                   psParallelism, iterationWaitTime=DEFAULT_ITERATION_WAIT_TIME,
                   backend: str = "local") -> ResultStream:
    """C2: ``PullP != PushP`` with ``LooseSimplePSLogic`` (FPS:122-139)."""
    return transform(trainingData, workerLogic, LooseSimplePSLogic(paramInit, paramUpdate),
                     workerParallelism, psParallelism, iterationWaitTime, backend=backend)


# ------------------------------------------------------------------------------------------
# model loading (C9 / C10)
# ------------------------------------------------------------------------------------------
class _EOF:
    """End-of-model marker (one per worker, fanned out to every PS shard, FPS:790-792)."""

    __slots__ = ()

    def __repr__(self):
        return "EOF"


class _ShardIndex:
    """An id that addresses PS shard ``index`` directly (the ``Left(psIdx)`` ids of FPS:831)."""

    __slots__ = ("index",)

    def __init__(self, index: int):
        self.index = index


class _ModelParam:
    __slots__ = ("id", "value")

    def __init__(self, id, value):
        self.id, self.value = id, value


class _WorkerModel:
    """A worker-local model entry of the double model load (``ModelWorkerData``, FPS:967-986)."""

    __slots__ = ("id", "value")

    def __init__(self, id, value):
        self.id, self.value = id, value


class _LoadingWorkerLogic(LooseWorkerLogic):
    """Worker wrapper: push model records, buffer training data until the model EOF, then replay
    (FPS:782-808, 1035-1069)."""

    def __init__(self, inner: LooseWorkerLogic, psParallelism: int):
        self.inner = inner
        self.psP = psParallelism
        self.receivedEOF = False
        self.dataBuffer: List[Any] = []

    def open(self):
        self.inner.open()

    def close(self):
        self.inner.close()

    def fork(self):
        from .local_engine import clone_logic

        return _LoadingWorkerLogic(clone_logic(self.inner), self.psP)

    def onRecv(self, rec, ps):
        if isinstance(rec, _ModelParam):
            ps.push(rec.id, rec)                       # model records are PUSHED to the PS
        elif isinstance(rec, _WorkerModel):
            self.inner.updateModel(rec.id, rec.value)  # BaseMFWorkerLogic.updateModel (FPS:1050)
        elif isinstance(rec, _EOF):
            self.receivedEOF = True
            for psIdx in range(self.psP):
                ps.push(_ShardIndex(psIdx), rec)
            buf, self.dataBuffer = self.dataBuffer, []
            for d in buf:
                self.inner.onRecv(d, ps)
        elif self.receivedEOF:
            self.inner.onRecv(rec, ps)
        else:
            self.dataBuffer.append(rec)

    def onPullRecv(self, paramId, paramValue, ps):
        if isinstance(paramValue, _EOF):
            return  # keep-alive answers of the double model load are ignored (FPS:1067-1069)
        self.inner.onPullRecv(paramId, paramValue, ps)


class _LoadingPSLogic(LooseParameterServerLogic):
    """PS wrapper: count down one EOF per worker, buffer pulls until then (FPS:848-887)."""

    def __init__(self, inner: LooseParameterServerLogic, workerParallelism: int):
        self.inner = inner
        self.wP = workerParallelism
        self.eofCountDown = workerParallelism
        self.pullBuffer: List[Tuple[Any, int]] = []

    def fork(self):
        from .local_engine import clone_logic

        return _LoadingPSLogic(clone_logic(self.inner), self.wP)

    def open(self, parameters, runtimeContext):
        self.inner.open(parameters, runtimeContext)
        if hasattr(self.inner, "flush"):          # device-resident inner store: batched execution
            self.flush = self.inner.flush

    def close(self, ps):
        self.inner.close(ps)

    def onPullRecv(self, id, workerPartitionIndex, ps):
        if self.eofCountDown == 0:
            self.inner.onPullRecv(id, workerPartitionIndex, ps)
        else:
            self.pullBuffer.append((id, workerPartitionIndex))

    def onPushRecv(self, id, deltaUpdate, ps):
        if isinstance(deltaUpdate, _EOF):
            self.eofCountDown -= 1
            if self.eofCountDown == 0:
                buf, self.pullBuffer = self.pullBuffer, []
                for pid, widx in buf:
                    self.inner.onPullRecv(pid, widx, ps)
        elif isinstance(deltaUpdate, _ModelParam):
            self.inner.onPushRecv(id, deltaUpdate.value, ps)
        else:
            self.inner.onPushRecv(id, deltaUpdate, ps)


def _loading_partitioner(user_part: Callable[[Any], int]) -> Callable[[Any], int]:
    def part(msg) -> int:
        m = _first(msg)
        pid = m.paramId
        if isinstance(pid, _ShardIndex):
            return pid.index
        return user_part(msg)

    return part


def _prepare_load(model_stream: DataStream, trainingData, wrap) -> DataStream:
    model = as_stream(model_stream).map(wrap).rebalance().with_eof(_EOF)
    data = as_stream(trainingData)
    return model.union(data)


def transformWithModelLoad(model):
    """``transformWithModelLoad(model)(trainingData, workerLogic, psLogic, paramPartitioner,
    wInPartition, workerParallelism, psParallelism, iterationWaitTime)`` (FPS:715-908).

    ``model`` is a stream of ``(id, value)``; every entry reaches its PS shard (as a push, so the
    ``psLogic`` must accept push-before-pull, FPS:678-680) before any training record is handled.
    """

    def run(trainingData, workerLogic, psLogic, paramPartitioner=None, wInPartition=None,
            workerParallelism=1, psParallelism=1,
            iterationWaitTime=DEFAULT_ITERATION_WAIT_TIME, backend: str = "local") -> ResultStream:
        wP, psP = int(workerParallelism), int(psParallelism)
        from ..api import BatchedWorkerLogic

        if isinstance(workerLogic, BatchedWorkerLogic):
            # tensor tier: psLogic = (paramInit, paramUpdate, {num_ids, dim, ...}); the model is loaded
            # into the shards with one-sided stores before the first micro-batch
            from .device_engine import transform_batched

            init, update, opts = psLogic
            return transform_batched(trainingData, workerLogic, init, update, wP, psP, iterationWaitTime,
                                     model=model, paramPartitioner=paramPartitioner, **opts)
        psLogic = device_ps_logic(psLogic, backend)
        user_part = paramPartitioner or default_param_partitioner(psP)
        stream = _prepare_load(model, trainingData, lambda kv: _ModelParam(kv[0], kv[1]))
        return transform_general(
            stream, _LoadingWorkerLogic(workerLogic, psP), _LoadingPSLogic(psLogic, wP),
            _loading_partitioner(user_part), wInPartition or default_worker_partitioner(wP),
            wP, psP, SimpleWorkerReceiver(), SimpleWorkerSender(), SimplePSReceiver(),
            SimplePSSender(), iterationWaitTime)

    return run


def transformWithDoubleModelLoad(model):
    """Model stream of ``Left((id, p))`` (server parameter) / ``Right((id, p))`` (worker-local
    entry handed to ``workerLogic.updateModel``) (FPS:950-1173)."""

    def run(trainingData, workerLogic, psLogic, paramPartitioner=None, wInPartition=None,
            workerParallelism=1, psParallelism=1,
            iterationWaitTime=DEFAULT_ITERATION_WAIT_TIME,
            workerModelPartitioner: Optional[Callable[[Any, int], int]] = None,
            backend: str = "local") -> ResultStream:
        wP, psP = int(workerParallelism), int(psParallelism)
        psLogic = device_ps_logic(psLogic, backend)
        user_part = paramPartitioner or default_param_partitioner(psP)

        def wrap(e):
            (k, v) = e.value
            return _ModelParam(k, v) if e.is_left else _WorkerModel(k, v)

        m = as_stream(model).map(wrap)
        if workerModelPartitioner is not None:
            # worker-local entries must land on the worker that owns them
            def route(rec, n):
                if isinstance(rec, _WorkerModel):
                    return workerModelPartitioner(rec.id, n)
                return stable_hash(rec.id) % n

            m = m.partition_custom(route)
        else:
            m = m.rebalance()
        stream = m.with_eof(_EOF).union(as_stream(trainingData))
        return transform_general(
            stream, _LoadingWorkerLogic(workerLogic, psP), _LoadingPSLogic(psLogic, wP),
            _loading_partitioner(user_part), wInPartition or default_worker_partitioner(wP),
            wP, psP, SimpleWorkerReceiver(), SimpleWorkerSender(), SimplePSReceiver(),
            SimplePSSender(), iterationWaitTime)

    return run


# snake_case aliases
transform_loose = transformLoose
transform_with_model_load = transformWithModelLoad
transform_with_double_model_load = transformWithDoubleModelLoad
