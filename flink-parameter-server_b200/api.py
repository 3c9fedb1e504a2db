"""User-facing parameter-server API (layer L3 of the reference).

Names and contracts follow the reference so user code ports 1:1:

=================================  ==========================================================
reference                          here
=================================  ==========================================================
``WorkerLogic`` (WL:22)            :class:`WorkerLogic`  (= ``LooseWorkerLogic`` with P == P)
``LooseWorkerLogic`` (WL:39-74)    :class:`LooseWorkerLogic`
``ParameterServerClient``          :class:`ParameterServerClient` (``pull / push / output``)
``ParameterServerLogic``           :class:`ParameterServerLogic` (FPS:1250, 1269-1304)
``ParameterServer`` (FPS:1307)     :class:`ParameterServer` (``answerPull / output``)
``Either`` outputs                 :class:`Left` (worker output) / :class:`Right` (PS output)
=================================  ==========================================================

On top of the per-record callbacks the device design adds *batched* callbacks
(:class:`BatchedWorkerLogic`): a worker receives a micro-batch of records and pulls / pushes whole
id tensors, which the device backend executes as fused gather / red.add kernels over NVLink peer
memory.  Per-record logics run unchanged on every backend through the scalar adapter.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Generic, TypeVar

T = TypeVar("T")
Id = TypeVar("Id")
P = TypeVar("P")
PullP = TypeVar("PullP")
PushP = TypeVar("PushP")
WOut = TypeVar("WOut")
PSOut = TypeVar("PSOut")


# ------------------------------------------------------------------------------------------
# Either
# ------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Left:
    """``Left(x)`` -- worker output in the result stream (FPS:471)."""

    value: Any

    @property
    def is_left(self) -> bool:
        return True

    @property
    def is_right(self) -> bool:
        return False

    isLeft = is_left
    isRight = is_right


@dataclass(frozen=True)
class Right:
    """``Right(x)`` -- parameter-server output in the result stream (FPS:472)."""

    value: Any

    @property
    def is_left(self) -> bool:
        return False

    @property
    def is_right(self) -> bool:
        return True

    isLeft = is_left
    isRight = is_right


Either = (Left, Right)


class CtorFork:
    """Mixin: remember constructor arguments so the engine can build one fresh instance per
    parallel subtask with ``fork()`` (the analogue of Flink shipping a serialised copy of the logic
    to every subtask).  Use it for logics that own locks, threads or RNGs (not deep-copyable)."""

    def __new__(cls, *args, **kwargs):
        obj = super().__new__(cls)
        obj._ctor_args = (args, kwargs)
        return obj

    def fork(self):
        args, kwargs = self._ctor_args
        return type(self)(*args, **kwargs)


# ------------------------------------------------------------------------------------------
# worker side
# ------------------------------------------------------------------------------------------
class ParameterServerClient(Generic[Id, P, WOut]):
    """Handle a worker uses to talk to the PS (M/ParameterServerClient.scala:14-22).

    All three calls are fire-and-forget; the answer to a pull arrives later through
    ``WorkerLogic.onPullRecv``.
    """

    def pull(self, id: Id) -> None:
        raise NotImplementedError

    def push(self, id: Id, deltaUpdate: P) -> None:
        raise NotImplementedError

    def output(self, out: WOut) -> None:
        raise NotImplementedError


class LooseWorkerLogic(Generic[T, Id, PullP, PushP, WOut]):
    """Worker callbacks where the pulled type may differ from the pushed type (WL:39-74)."""

    def open(self) -> None:
        """Called once before any record (FPS:376-379)."""

    def onRecv(self, data: T, ps: ParameterServerClient) -> None:
        """A training record arrived."""
        raise NotImplementedError

    def onPullRecv(self, paramId: Id, paramValue: PullP, ps: ParameterServerClient) -> None:
        """The answer to an earlier ``ps.pull(paramId)`` arrived."""
        raise NotImplementedError

    def close(self) -> None:
        """Called when the iteration terminates."""

    # snake_case aliases -------------------------------------------------------------
    def on_recv(self, data, ps):
        return self.onRecv(data, ps)

    def on_pull_recv(self, paramId, paramValue, ps):
        return self.onPullRecv(paramId, paramValue, ps)


class WorkerLogic(LooseWorkerLogic[T, Id, P, P, WOut]):
    """``WorkerLogic[T, Id, P, WOut] = LooseWorkerLogic[T, Id, P, P, WOut]`` (WL:22)."""


class BatchedWorkerLogic(WorkerLogic):
    """Micro-batch worker callbacks (device-tier extension; see module docstring).

    ``onRecvBatch`` gets a batch object (any structure of tensors) and a
    :class:`BatchedParameterServerClient`; ``onPullRecvBatch`` gets the id tensor of a pull and
    the ``[n, dim]`` value tensor gathered from the owning shards.
    """

    def onRecvBatch(self, batch: Any, ps: "BatchedParameterServerClient") -> None:
        raise NotImplementedError

    def onPullRecvBatch(self, ids: Any, values: Any, ps: "BatchedParameterServerClient") -> None:
        raise NotImplementedError

    # scalar adapter so a batched logic also runs on per-record backends
    def onRecv(self, data, ps):
        self.onRecvBatch(data, ps)

    def onPullRecv(self, paramId, paramValue, ps):
        self.onPullRecvBatch(paramId, paramValue, ps)


class BatchedParameterServerClient(ParameterServerClient):
    """``pull(ids)`` / ``push(ids, deltas)`` on whole tensors."""

    def pull_now(self, ids: Any) -> Any:
        """Synchronous fused gather (device backends); returns the ``[n, dim]`` values."""
        raise NotImplementedError


# ------------------------------------------------------------------------------------------
# server side
# ------------------------------------------------------------------------------------------
class ParameterServer(Generic[Id, P, PSOut]):
    """Handle a server logic uses to answer pulls and emit outputs (FPS:1307-1311)."""

    def answerPull(self, id: Id, value: P, workerPartitionIndex: int) -> None:
        raise NotImplementedError

    def output(self, out: PSOut) -> None:
        raise NotImplementedError

    def answer_pull(self, id, value, workerPartitionIndex):
        return self.answerPull(id, value, workerPartitionIndex)


@dataclass
class RuntimeContext:
    """What ``ParameterServerLogic.open`` learns about its placement (FPS:1303)."""

    index_of_this_subtask: int
    number_of_parallel_subtasks: int

    def getIndexOfThisSubtask(self) -> int:
        return self.index_of_this_subtask

    def getNumberOfParallelSubtasks(self) -> int:
        return self.number_of_parallel_subtasks


class LooseParameterServerLogic(Generic[Id, PullP, PushP, PSOut]):
    """Server callbacks (FPS:1269-1304)."""

    def onPullRecv(self, id: Id, workerPartitionIndex: int, ps: ParameterServer) -> None:
        raise NotImplementedError

    def onPushRecv(self, id: Id, deltaUpdate: PushP, ps: ParameterServer) -> None:
        raise NotImplementedError

    def open(self, parameters: dict, runtimeContext: RuntimeContext) -> None:
        """Called once with the shard index / count before any message."""

    def close(self, ps: ParameterServer) -> None:
        """Called when the iteration terminates; *WithClose logics dump the model here."""

    def on_pull_recv(self, id, workerPartitionIndex, ps):
        return self.onPullRecv(id, workerPartitionIndex, ps)

    def on_push_recv(self, id, deltaUpdate, ps):
        return self.onPushRecv(id, deltaUpdate, ps)


class ParameterServerLogic(LooseParameterServerLogic[Id, P, P, PSOut]):
    """``ParameterServerLogic[Id, P, PSOut] = LooseParameterServerLogic[Id, P, P, PSOut]`` (FPS:1250)."""
