"""Replica <-> master exchange kernel over a REAL NVLink peer, in ONE process (so it can run under ncu).

GPU 0 holds a replica (owner-major, 2 segments) and the master shard 0; master shard 1 lives in GPU 1's
HBM and is reached through peer access.  The exchange of destination 1 therefore moves every row over
NVLink in both directions (bulk reads of v, REDG of d), exactly like one remote segment of an N-GPU job.

    python benchmarks/exchange_peer_bench.py [--rows 500000] [--dim 64] [--ctas 32,64,132,264] [--stages 4]

Prints one JSON line: per CTA count the exchange time, GB/s per direction over the link and the local HBM
bytes moved.  Under ncu add ``--once`` (one exchange per configuration, no timing loop).
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rows", type=int, default=500_000, help="rows per segment")
    p.add_argument("--dim", type=int, default=64)
    p.add_argument("--ctas", default="16,32,64,132,264")
    p.add_argument("--stages", type=int, default=4)
    p.add_argument("--iters", type=int, default=10)
    p.add_argument("--once", action="store_true")
    a = p.parse_args()
    from fps_b200.ops import native

    two = torch.cuda.device_count() >= 2
    d0 = torch.device("cuda", 0)
    d1 = torch.device("cuda", 1 if two else 0)
    if two:
        native.enable_peer(0, 1)
    torch.cuda.set_device(0)
    stride = (a.dim + 3) // 4 * 4
    rps = a.rows
    master0 = torch.randn(rps, stride, device=d0)
    master1 = torch.randn(rps, stride, device=d1)           # the peer shard (NVLink)
    tc = native.ShardTableC()
    tc.base[0] = master0.data_ptr(); tc.base[1] = master1.data_ptr()
    tc.rows_per_shard = rps; tc.div = rps; tc.num_shards = 2; tc.dim = a.dim; tc.stride = stride
    tc.mode = native.PART_HASH; tc.shard_shift = 1
    cache = torch.cat([master0, master1.to(d0)]).contiguous()
    base = cache.clone()
    seg_bytes = rps * stride * 4
    out = {"rows_per_segment": rps, "dim": a.dim, "segment_MB": seg_bytes / 1e6, "peer": two, "runs": []}
    for n_ctas in [int(x) for x in a.ctas.split(",")]:
        times = []
        for it in range(1 if a.once else a.iters + 2):
            cache[rps:] += 0.001 * (it + 1)                  # every row of segment 1 has a pending delta
            master1 += 0.002                                  # ... and a foreign contribution to fold in
            torch.cuda.synchronize(d1); torch.cuda.synchronize(d0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            native.replica_exchange(tc, cache, base, mask=0b10, n_ctas=n_ctas, n_stages=a.stages)
            e1.record()
            torch.cuda.synchronize(d0)
            times.append(e0.elapsed_time(e1))
        t = min(times[2:]) if len(times) > 2 else times[-1]
        out["runs"].append({"ctas": n_ctas, "stages": a.stages, "ms": t,
                            "link_GBps_per_direction": seg_bytes / t / 1e6,
                            "local_hbm_GB": 5 * seg_bytes / 1e9})
    # correctness of the last state: replica == master == base on segment 1 (up to fp32 rounding)
    torch.cuda.synchronize(d1); torch.cuda.synchronize(d0)
    err = (cache[rps:] - master1.to(d0)).abs().max().item()
    out["max_abs_replica_minus_master"] = err
    print(json.dumps(out))


if __name__ == "__main__":
    main()
