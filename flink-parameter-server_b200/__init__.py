"""fps_b200 -- a Hopper (H100, sm_90a) native asynchronous parameter-server framework with
the capabilities of FlinkML/flink-parameter-server.

Public surface (reference names kept):

* ``transform``, ``transformLoose``, ``transformWithModelLoad``, ``transformWithDoubleModelLoad``
* ``WorkerLogic``, ``LooseWorkerLogic``, ``ParameterServerClient``, ``ParameterServerLogic``,
  ``LooseParameterServerLogic``, ``ParameterServer``, ``Left`` / ``Right``
* ``addPullLimiter``, ``addBlockingPullLimiter``, ``WorkerLogicWithFuture``
* server stores in :mod:`fps_b200.server`, wire protocol / batching in :mod:`fps_b200.protocol`
* algorithms in :mod:`fps_b200.models` (matrix factorisation, passive-aggressive, sketches, ...)
* device tier: :mod:`fps_b200.store` (sharded HBM tables), :mod:`fps_b200.ops` (sm_90a kernels),
  :mod:`fps_b200.parallel` (NVLink symmetric-heap fabric, partitioners, NCCL baseline)
"""
from .api import (BatchedParameterServerClient, BatchedWorkerLogic, Either, Left,
                  LooseParameterServerLogic, LooseWorkerLogic, ParameterServer,
                  ParameterServerClient, ParameterServerLogic, Right, RuntimeContext, WorkerLogic)
from .limiter import (PSClientWithFuture, PullAnswerFuture, WorkerLogicWithFuture,
                      addBlockingPullLimiter, addPullLimiter)
from .runtime.stream import DataStream, ResultStream
from .runtime.transform import (transform, transform_general, transformLoose,
                                transformWithDoubleModelLoad, transformWithModelLoad)

__version__ = "0.1.0"


class FlinkParameterServer:
    """Namespace alias so ``FlinkParameterServer.transform(...)`` reads like the reference."""

    transform = staticmethod(transform)
    transformLoose = staticmethod(transformLoose)
    transformWithModelLoad = staticmethod(transformWithModelLoad)
    transformWithDoubleModelLoad = staticmethod(transformWithDoubleModelLoad)
