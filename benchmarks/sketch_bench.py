#!/usr/bin/env python
"""Streaming-sketch update throughput (K8-K10): (word, tweet) occurrences/s and one-sided reductions/s
for Bloom (red.or.b32), tug-of-war (red.add.s32) and MinHash (red.min.u64) on one GPU."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    from fps_b200.models.sketch.device import DeviceSketch

    n_keys, n_occ = 1_000_000, 4_000_000
    g = torch.Generator(device="cpu").manual_seed(0)
    # Zipf-like key popularity (word frequencies)
    u = torch.rand(n_occ, generator=g)
    keys = (n_keys * u ** 3).to(torch.int32).clamp_(max=n_keys - 1).to(dev)
    tweets = torch.randint(0, 1 << 40, (n_occ,), generator=g, dtype=torch.int64).to(dev)
    res = {}
    for kind, hashes, arr in [("bloom", 8, 4096), ("tow", 64, 0), ("minhash", 32, 0)]:
        sk = DeviceSketch(kind, n_keys, hashes, arr)
        for _ in range(3):
            sk.update_ids(keys, tweets)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            sk.update_ids(keys, tweets)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        res[kind] = {"occurrences_per_s": n_occ / ms * 1e3, "reductions_per_s": n_occ * hashes / ms * 1e3,
                     "ms_per_batch": ms, "num_hashes": hashes, "keys": n_keys,
                     "table_MB": sk.table.local.numel() * 4 / 1e6}
        sk.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
