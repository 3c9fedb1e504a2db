#!/usr/bin/env python
"""Row-wise AdaGrad against SGD for device matrix factorisation on one GPU: step time.

    python benchmarks/mf_adagrad_bench.py [--out profiles/h100_mf_adagrad_bench.json]

Records, in one process:

* the card (name, power limit, max SM clock), before and after;
* step device time at the shape of ``bench.py --gpus 1`` (10M users x 1M items, k = 64, 4.19M ratings per
  step as 5 micro-batches with distinct users and distinct items each, packed64), per launch:
  pointwise SGD against pointwise AdaGrad, and BPR with one negative sampled in the kernel, SGD against
  AdaGrad; the pointwise SGD step window (the default of ``DeviceOnlineMF`` at this shape) for context.
  The configurations are alternated round by round; the median and the spread over the rounds are kept.
* a bytes model (``BYTES``): a row access is 256 B at k = 64; an accumulator access is one 4-byte load or
  reduction, which costs a whole 32-byte sector.  Pointwise moves 4 rows per rating (pull u and v, push
  both); AdaGrad adds 2 accumulator loads and 2 reductions.  BPR with one negative moves 6 rows; AdaGrad
  adds 3 loads and 3 reductions.
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

from mf_bpr_bench import BATCH, ITEMS, K, USERS, bench_batches, card, timed  # noqa: E402

ROW, SECTOR = 4 * K, 32
BYTES = {
    "pointwise_sgd": 4 * ROW, "pointwise_adagrad": 4 * ROW + 4 * SECTOR, "pointwise_sgd_window": 4 * ROW,
    "bpr_sgd": 6 * ROW, "bpr_adagrad": 6 * ROW + 6 * SECTOR,
}


def throughput(a, native, dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    steps = bench_batches(native, dev)
    kw = dict(learning_rate=0.01, seed=1)
    bpr = dict(loss="bpr", negative_sample_rate=1)
    models = {
        "pointwise_sgd": DeviceOnlineMF(USERS, ITEMS, K, step_window=0, **kw),
        "pointwise_adagrad": DeviceOnlineMF(USERS, ITEMS, K, optimizer="adagrad", **kw),
        "bpr_sgd": DeviceOnlineMF(USERS, ITEMS, K, **bpr, **kw),
        "bpr_adagrad": DeviceOnlineMF(USERS, ITEMS, K, optimizer="adagrad", **bpr, **kw),
    }
    if not a.no_window:
        models["pointwise_sgd_window"] = DeviceOnlineMF(USERS, ITEMS, K, **kw)
    for m in models.values():
        timed(m, steps, a.warmup)
    ms = {c: [] for c in models}
    for _ in range(a.rounds):
        for c, m in models.items():
            ms[c].append(timed(m, steps, a.steps))
    out = {}
    for c, m in models.items():
        med = statistics.median(ms[c])
        out[c] = {"ms_per_step_rounds": [round(x, 4) for x in ms[c]], "ms_per_step_median": round(med, 4),
                  "ms_per_step_spread": round(max(ms[c]) - min(ms[c]), 4),
                  "ratings_per_s": BATCH / (med * 1e-3), "model_bytes_per_rating": BYTES[c],
                  "achieved_bytes_per_s_model": BATCH * BYTES[c] / (med * 1e-3)}
        m.check_finite()
        m.close()
    out["pointwise_adagrad_over_sgd_time"] = (out["pointwise_adagrad"]["ms_per_step_median"]
                                              / out["pointwise_sgd"]["ms_per_step_median"])
    out["bpr_adagrad_over_sgd_time"] = out["bpr_adagrad"]["ms_per_step_median"] / out["bpr_sgd"]["ms_per_step_median"]
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(REPO, "profiles", "h100_mf_adagrad_bench.json"))
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--no-window", action="store_true", help="skip the step-window SGD context row")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mf_adagrad_bench.py measures on a GPU; none is visible")
    import fps_b200  # noqa: F401
    from fps_b200.ops import native

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"card": card(), "shape": {"users": USERS, "items": ITEMS, "k": K, "ratings_per_step": BATCH,
                                      "micro_batches": -(-BATCH // min(ITEMS, USERS)), "format": "packed64",
                                      "bpr_negatives_per_positive": 1},
           "timing": {"steps_per_round": a.steps, "rounds": a.rounds, "warmup_steps": a.warmup,
                      "clock": "CUDA events around the steps of a round, divided by the steps"}}
    res["throughput"] = throughput(a, native, dev)
    res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
