#!/usr/bin/env python
"""WARP against BPR matrix factorisation on one GPU: step time and achieved bandwidth.

    python benchmarks/mf_warp_bench.py [--out profiles/h100_mf_warp_bench.json]

Records, in one process:

* the card (name, power limit, max SM clock), before and after;
* at the shape of ``bench.py --gpus 1`` (10M users x 1M items, k = 64, 4.19M positives per step as 5 micro-batches
  with distinct users and distinct items each, packed64), device-timed steps, every configuration alternated
  round by round, median and range over the rounds:
  - BPR with 1 and with ``T`` negatives sampled in the kernel (the references);
  - WARP with ``T`` candidates sampled in the kernel, best case (margin 1e3: the first candidate violates) and
    worst case (margin -1e3: none violates), at the dispatcher's trial block and at every trial block.
  The rows hold values of about 0.01, so x stays far inside either margin.

Bytes model (256-byte rows): a BPR triple pulls and pushes u, v_i and v_j, ``2 * (2 + n)`` rows for ``n`` negatives.
A WARP positive pulls u, v_i and each candidate it examines (``2 + n``), and pushes u, v_i and v_j when it updates
(3 more); ``n`` and the update rate are read from the kernel's own counters.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "benchmarks"))

from mf_bpr_bench import BATCH, ITEMS, K, ROW_BYTES, USERS, bench_batches, card  # noqa: E402

LR = 1e-4           # small enough that nothing grows over the run: the timing does not depend on it
BEST, WORST = 1e3, -1e3


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(REPO, "profiles", "h100_mf_warp_bench.json"))
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--T", type=int, default=10)
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mf_warp_bench.py measures on a GPU; none is visible")
    import fps_b200  # noqa: F401
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.ops import native

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"card": card(), "shape": {"users": USERS, "items": ITEMS, "k": K, "positives_per_step": BATCH,
                                      "micro_batches": -(-BATCH // min(ITEMS, USERS)), "format": "packed64",
                                      "T": a.T}}
    steps = bench_batches(native, dev)
    bpr1 = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=LR, negative_sample_rate=1, seed=1, loss="bpr")
    bprT = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=LR, negative_sample_rate=a.T, seed=1, loss="bpr")
    warp = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=LR, negative_sample_rate=a.T, seed=1, loss="warp")
    counters = {}

    def warp_step(margin, tb, name):
        st = counters.setdefault(name, torch.zeros(4, device=dev))

        def run(mb):
            native.mf_warp_fused(mb, None, None, warp._users, warp._items.table_c, LR, margin=margin,
                                 n_neg=a.T, num_items=ITEMS, seed=warp.seed, step=warp.step_no, stats=st,
                                 nan_flag=warp._nan_flag, trial_block=tb)
            warp.step_no += 1
        return run

    configs = {"bpr_n1": bpr1.step, f"bpr_n{a.T}": bprT.step}
    for case, margin in (("best", BEST), ("worst", WORST)):
        configs[f"warp_{case}"] = warp_step(margin, 0, f"warp_{case}")
        for tb in native.WARP_TRIAL_BLOCKS:
            configs[f"warp_{case}_tb{tb}"] = warp_step(margin, tb, f"warp_{case}_tb{tb}")

    def timed(fn, n_steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in range(n_steps):
            for mb in steps[s % len(steps)]:
                fn(mb)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n_steps

    for fn in configs.values():
        timed(fn, a.warmup)
    ms = {c: [] for c in configs}
    for _ in range(a.rounds):
        for c, fn in configs.items():
            ms[c].append(timed(fn, a.steps))
    # the kernel's counters, from one micro-batch (float atomics are exact below 2^24)
    for c, fn in configs.items():
        if c in counters:
            counters[c].zero_()
            fn(steps[0][0])
    torch.cuda.synchronize()
    out = {}
    for c in configs:
        med = statistics.median(ms[c])
        if c.startswith("bpr"):
            n = int(c.split("_n")[1])
            rows = 2 * (2 + n)
            extra = {"negatives": n}
        else:
            st = counters[c].cpu()
            trials, upd = float(st[2] / st[3]), float(st[1] / st[3])
            rows = 2 + trials + 3 * upd
            extra = {"mean_trials": round(trials, 4), "update_rate": round(upd, 4)}
        out[c] = {"ms_per_step_rounds": [round(x, 4) for x in ms[c]], "ms_per_step_median": round(med, 4),
                  "ms_per_step_range": [round(min(ms[c]), 4), round(max(ms[c]), 4)],
                  "positives_per_s": BATCH / (med * 1e-3), "model_rows_per_positive": round(rows, 4),
                  "achieved_bytes_per_s_model": BATCH * rows * ROW_BYTES / (med * 1e-3), **extra}
    for m in (bpr1, bprT, warp):
        m.check_finite()
        m.close()
    res["throughput"] = out
    res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
