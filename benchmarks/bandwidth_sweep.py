#!/usr/bin/env python
"""BASELINE.json config 5: pull / push bandwidth sweep, vector dim 64 .. 1M floats, at N GPUs, vs the
NCCL send/recv baseline.

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 benchmarks/bandwidth_sweep.py

Every rank pulls (then pushes) `rows` vectors of `dim` floats that live on OTHER ranks' shards
(ids owned by rank+1, rank+2, ... round robin), i.e. all traffic crosses NVLink.  Times are CUDA
events on the launching stream, max over ranks; GB/s is per GPU per direction.  The NCCL arm moves the
same bytes with batched isend/irecv between the same pairs.  Roofline: 450 GB/s per direction per GPU,
the NVLink 4 data-sheet rate of an H100 SXM (a ceiling, not a measured peer-copy rate).
"""
import json
import os

import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    lr = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    from fps_b200.store.sharded_table import ShardedTable

    total_bytes = int(os.environ.get("SWEEP_BYTES", 256 << 20))
    out = []
    for dim in [64, 256, 1024, 4096, 16384, 65536, 262144, 1048576]:
        rows = max(2 * (world - 1), total_bytes // (dim * 4))
        rows -= rows % max(1, world - 1)
        per_shard = rows // max(1, world - 1) + 1
        table = ShardedTable(per_shard * world, dim, init="zeros")
        # ids owned by the other ranks, spread round robin: id = slot * world + owner
        k = torch.arange(rows, device=dev)
        owner = (rank + 1 + k % (world - 1)) % world if world > 1 else torch.zeros_like(k)
        ids = ((k // max(1, world - 1)) * world + owner).to(torch.int64)
        buf = torch.empty((rows, table.stride), dtype=torch.float32, device=dev)
        delta = torch.ones((rows, table.stride), dtype=torch.float32, device=dev)
        nbytes = rows * dim * 4
        t_pull = timed(lambda: table.pull(ids, buf))
        t_push = timed(lambda: table.push(ids, delta))
        # NCCL arm: same bytes, same peers
        send = [delta[j::max(1, world - 1)].contiguous() for j in range(max(1, world - 1))]
        recv = [torch.empty_like(s) for s in send]

        def nccl():
            ops = []
            for j in range(world - 1):
                peer_to = (rank + 1 + j) % world
                peer_from = (rank - 1 - j) % world
                ops.append(dist.P2POp(dist.isend, send[j], peer_to))
                ops.append(dist.P2POp(dist.irecv, recv[j], peer_from))
            for w in dist.batch_isend_irecv(ops):
                w.wait()

        t_nccl = timed(nccl) if world > 1 else float("nan")
        rec = {"dim": dim, "rows": rows, "bytes": nbytes, "n_gpus": world,
               "pull_ms": t_pull, "pull_GBs": nbytes / t_pull / 1e6,
               "push_ms": t_push, "push_GBs": nbytes / t_push / 1e6,
               "nccl_sendrecv_ms": t_nccl, "nccl_GBs": nbytes / t_nccl / 1e6 if world > 1 else None,
               "pull_frac_of_450": nbytes / t_pull / 1e6 / 450.0}
        if rank == 0:
            print(json.dumps(rec), flush=True)
        out.append(rec)
        table.close()
        del buf, delta, send, recv
        torch.cuda.empty_cache()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
