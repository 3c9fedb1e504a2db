#!/usr/bin/env python
"""Negatives from the items each worker has seen, and skip-gram unigram noise, against uniform draws: step
time and sampler time on one GPU.

    python benchmarks/negative_sampling_bench.py [--out profiles/h100_negative_sampling_bench.json]

Records, in one process:

* the card (name, power limit, max SM clock), before and after;
* step device time at the shape of ``bench.py --gpus 1`` (10M users x 1M items, k = 64, 4.19M ratings per step
  as 5 micro-batches, packed64) with one negative per rating and ``user_memory=128``: pointwise and BPR,
  ``negative_sampling="uniform"`` against ``"seen"``.  The registry is warm: the warm-up steps have seen every
  item the timed steps rate.
* the sampler kernel alone on one such micro-batch (838,861 ratings, ring of 128): ``fps_neg_sample`` against
  ``fps_neg_sample_seen``;
* ``DeviceSkipGram`` with a 1M-word vocabulary, dim 300, ``negative=5``, 131,072 pairs per step: uniform
  against unigram noise (Zipf counts, power 0.75).

Every configuration is alternated with its counterpart round by round; the median and the spread over the
rounds are kept.
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

VOCAB, DIM, SG_NEG, SG_PAIRS = 1_000_000, 300, 5, 1 << 17


def _events(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _summary(rounds):
    med = statistics.median(rounds)
    return {"ms_rounds": [round(x, 4) for x in rounds], "ms_median": round(med, 4),
            "ms_spread": round(max(rounds) - min(rounds), 4)}


def _alternate(fns, rounds, n):
    ms = {c: [] for c in fns}
    for _ in range(rounds):
        for c, fn in fns.items():
            ms[c].append(fn(n))
    return {c: _summary(v) for c, v in ms.items()}


def mf_steps(a, native, dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    steps = bench_batches(native, dev)
    models = {}
    for loss in ("pointwise", "bpr"):
        for mode in ("uniform", "seen"):
            models[f"{loss}_{mode}"] = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=0.01, seed=1, loss=loss,
                                                      negative_sample_rate=1, user_memory=128,
                                                      negative_sampling=mode)
    for m in models.values():
        timed(m, steps, max(a.warmup, len(steps)))
    out = _alternate({c: (lambda n, m=m: timed(m, steps, n)) for c, m in models.items()}, a.rounds, a.steps)
    for c, m in models.items():
        out[c]["ms_per_step_median"] = out[c].pop("ms_median")
        m.check_finite()
        if m.negative_sampling == "seen":
            out[c]["registry_items"] = int(m.seen_items().numel())
        m.close()
    for loss in ("pointwise", "bpr"):
        out[f"{loss}_seen_over_uniform_time"] = (out[f"{loss}_seen"]["ms_per_step_median"]
                                                 / out[f"{loss}_uniform"]["ms_per_step_median"])
    return out


def sampler_alone(a, native, dev):
    mb = bench_batches(native, dev)[0][0]
    n, memory = mb.numel(), 128
    n_local = USERS
    state = {}
    for c in ("fps_neg_sample", "fps_neg_sample_seen"):
        state[c] = (torch.full((n_local, memory), -1, dtype=torch.int32, device=dev),
                    torch.zeros(n_local, dtype=torch.int32, device=dev))
    reg = native.seen_registry(ITEMS, dev)
    native.neg_sample_seen(torch.zeros(ITEMS, dtype=torch.int32, device=dev),
                           torch.arange(ITEMS, dtype=torch.int32, device=dev), torch.ones(ITEMS, device=dev), 0, reg)
    seen_u, seen_p = state["fps_neg_sample"]
    reg_u, reg_p = state["fps_neg_sample_seen"]
    fns = {
        "fps_neg_sample": lambda k: _events(lambda: native.neg_sample(mb, None, None, 1, ITEMS, seen_u, seen_p, 1,
                                                                      seed=1, step=0), k),
        "fps_neg_sample_seen": lambda k: _events(lambda: native.neg_sample_seen(mb, None, None, 1, reg, reg_u, reg_p,
                                                                                1, seed=1, step=0), k),
    }
    for fn in fns.values():
        fn(a.warmup)
    out = _alternate(fns, a.rounds, 50)
    out["ratings"] = n
    out["seen_over_uniform_time"] = out["fps_neg_sample_seen"]["ms_median"] / out["fps_neg_sample"]["ms_median"]
    return out


def skipgram(a, dev):
    import numpy as np

    from fps_b200.models.w2v import DeviceSkipGram

    counts = (1e7 / np.arange(1, VOCAB + 1)).astype(np.float64)     # Zipf
    models = {"uniform": DeviceSkipGram(VOCAB, DIM, negative=SG_NEG, seed=1),
              "unigram": DeviceSkipGram(VOCAB, DIM, negative=SG_NEG, seed=1, noise_counts=counts)}
    g = torch.Generator().manual_seed(3)
    batches = [(torch.randint(0, VOCAB, (SG_PAIRS,), generator=g).int().to(dev),
                torch.randint(0, VOCAB, (SG_PAIRS,), generator=g).int().to(dev)) for _ in range(3)]

    def run(m, k):
        def one():
            run.i = getattr(run, "i", 0) + 1
            m.step(*batches[run.i % len(batches)])
        return _events(one, k)

    for m in models.values():
        run(m, a.warmup)
    out = _alternate({c: (lambda k, m=m: run(m, k)) for c, m in models.items()}, a.rounds, a.steps)
    for m in models.values():
        m.check_finite()
        m.close()
    out["pairs_per_step"] = SG_PAIRS
    out["unigram_over_uniform_time"] = out["unigram"]["ms_median"] / out["uniform"]["ms_median"]
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(REPO, "profiles", "h100_negative_sampling_bench.json"))
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=5)
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("negative_sampling_bench.py measures on a GPU; none is visible")
    import fps_b200  # noqa: F401
    from fps_b200.ops import native

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"card": card(), "shape": {"users": USERS, "items": ITEMS, "k": K, "ratings_per_step": BATCH,
                                      "micro_batches": -(-BATCH // min(ITEMS, USERS)), "format": "packed64",
                                      "negatives_per_rating": 1, "user_memory": 128,
                                      "skipgram": {"vocab": VOCAB, "dim": DIM, "negative": SG_NEG,
                                                   "pairs_per_step": SG_PAIRS, "noise": "Zipf counts ** 0.75"}},
           "timing": {"steps_per_round": a.steps, "rounds": a.rounds, "warmup_steps": a.warmup,
                      "clock": "CUDA events around the steps (or 50 sampler launches) of a round, divided by them"}}
    res["mf_step"] = mf_steps(a, native, dev)
    res["sampler_kernel"] = sampler_alone(a, native, dev)
    res["skipgram_step"] = skipgram(a, dev)
    res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
