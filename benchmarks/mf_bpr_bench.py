#!/usr/bin/env python
"""Pairwise (BPR) against pointwise matrix factorisation on one GPU: speed and ranking quality.

    python benchmarks/mf_bpr_bench.py [--out profiles/h100_mf_bpr_bench.json]

Records, in one process:

* the card (name, power limit, max SM clock);
* throughput at the shape of ``bench.py --gpus 1`` (10M users x 1M items, k = 64, 4M positives per step as
  5 micro-batches with distinct users and distinct items each, packed64): the BPR step with one negative
  sampled in the kernel against the pointwise step with one sampled negative (logistic loss, err_mode 2),
  device-timed steps, the two alternated round by round.  Bytes model: a BPR triple moves 6 rows of
  256 B (pull u, v_i, v_j; push the three deltas), a pointwise positive with one negative 8 (pull u and v,
  push both, twice);
* quality on ``lowrank_implicit``: BPR (with and without its L2 term) and pointwise-logistic (which has no
  regulariser) trained with the same update budget (same positives, one negative each, same epochs),
  held-out sampled AUC and recall@10 of the ``DeviceTopK`` list without each user's train items.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

USERS, ITEMS, K, BATCH, HOST_BUFFERS = 10_000_000, 1_000_000, 64, 4 * 1024 * 1024, 3
ROW_BYTES = 4 * K
BYTES_PER_POSITIVE = {"bpr": 6 * ROW_BYTES, "pointwise": 8 * ROW_BYTES}


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # the card name still comes from torch
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi_error": f"{type(exc).__name__}: {exc}"}


def bench_batches(native, dev):
    """Micro-batches of the ``bench.py --gpus 1`` shape; every record is a positive (rating 1)."""
    n_sub = -(-BATCH // min(ITEMS, USERS))
    g = torch.Generator().manual_seed(1000)
    sizes = [len(c) for c in torch.arange(BATCH).tensor_split(n_sub)]
    steps = []
    for _ in range(HOST_BUFFERS):
        users = torch.randperm(USERS, generator=g)[:BATCH].split(sizes)
        step = []
        for j, n in enumerate(sizes):
            i = torch.randperm(ITEMS, generator=g)[:n].to(torch.int32)
            step.append(native.pack_ratings(users[j].to(torch.int32), i, torch.ones(n)).to(dev))
        steps.append(step)
    return steps


def timed(model, steps, n_steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(n_steps):
        for mb in steps[s % len(steps)]:
            model.step(mb)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n_steps


def throughput(a, native, dev):
    from fps_b200.models.mf.device import DeviceOnlineMF

    steps = bench_batches(native, dev)
    models = {
        "pointwise": DeviceOnlineMF(USERS, ITEMS, K, learning_rate=0.01, negative_sample_rate=1, err_mode=2,
                                    seed=1),
        "bpr": DeviceOnlineMF(USERS, ITEMS, K, learning_rate=0.01, negative_sample_rate=1, seed=1, loss="bpr"),
    }
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
                  "positives_per_s": BATCH / (med * 1e-3),
                  "model_bytes_per_positive": BYTES_PER_POSITIVE[c],
                  "achieved_bytes_per_s_model": BATCH * BYTES_PER_POSITIVE[c] / (med * 1e-3)}
        m.check_finite()
        m.close()
    out["bpr_over_pointwise_positives_per_s"] = out["bpr"]["positives_per_s"] / out["pointwise"]["positives_per_s"]
    return out


def quality(a, dev):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.utils.synthetic import lowrank_implicit

    nu, ni, per, held = a.q_users, a.q_items, 40, 10
    tu, ti, eu, ei = lowrank_implicit(nu, ni, per, held, seed=7)
    du, di = tu.int().to(dev), ti.int().to(dev)
    ones = torch.ones(du.numel(), device=dev)
    # train items per user, sorted (the exclusion CSR of DeviceTopK)
    order = torch.argsort(tu * ni + ti)
    offsets = torch.zeros(nu + 1, dtype=torch.int64)
    offsets[1:] = torch.bincount(tu, minlength=nu).cumsum(0)
    excl = (offsets.to(dev), ti[order].to(dev))
    g = torch.Generator().manual_seed(3)
    jn = torch.randint(0, ni, (eu.numel(), 100), generator=g).to(dev)
    consumed = torch.zeros(nu, ni, dtype=torch.bool, device=dev)
    consumed[tu.to(dev), ti.to(dev)] = True
    consumed[eu.to(dev), ei.to(dev)] = True
    test = torch.zeros(nu, ni, dtype=torch.bool, device=dev)
    test[eu.to(dev), ei.to(dev)] = True
    res = {"users": nu, "items": ni, "per_user": per, "held_out": held, "k": a.q_k, "epochs": a.q_epochs,
           "batch": a.q_batch, "init": 0.1, "bpr_reg": a.q_reg, "pointwise_reg": 0.0}
    # BPR with and without its L2 term (the pointwise kernel has no regulariser), so the gap between the
    # losses can be told apart from the effect of the regulariser
    configs = [(f"bpr_reg{r}", dict(loss="bpr", regularization=r)) for r in a.q_reg]
    configs.append(("pointwise_logistic_reg0", dict(err_mode=2)))
    for name, kw in configs:
        for lr in a.q_lr:
            m = DeviceOnlineMF(nu, ni, a.q_k, range_min=-0.1, range_max=0.1, learning_rate=lr,
                               negative_sample_rate=1, seed=5, **kw)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.q_epochs):
                for s in range(0, du.numel(), a.q_batch):
                    m.step(du[s:s + a.q_batch], di[s:s + a.q_batch], ones[s:s + a.q_batch])
            e1.record()
            torch.cuda.synchronize()
            m.check_finite()
            U, V = m.users[:nu], m.items.local[:ni]
            pos = (U[eu.to(dev)] * V[ei.to(dev)]).sum(1, keepdim=True)
            neg = torch.einsum("qk,qjk->qj", U[eu.to(dev)], V[jn])
            valid = ~consumed[eu.to(dev)[:, None], jn]
            auc = float(((pos > neg) & valid).sum() / valid.sum())
            _, rows = DeviceTopK(V.contiguous()).topk(10, q_local=U.contiguous(), exclude=excl)
            hits = test.gather(1, rows.long().clamp(min=0)) & (rows >= 0)
            res[f"{name}_lr{lr}"] = {"heldout_auc": round(auc, 4),
                                     "recall_at_10": round(float(hits.sum()) / eu.numel(), 4),
                                     "train_ms": round(e0.elapsed_time(e1), 1)}
            m.close()
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(REPO, "profiles", "h100_mf_bpr_bench.json"))
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=4)
    p.add_argument("--q-users", type=int, default=10_000)
    p.add_argument("--q-items", type=int, default=10_000)
    p.add_argument("--q-k", type=int, default=32)
    p.add_argument("--q-epochs", type=int, default=20)
    p.add_argument("--q-batch", type=int, default=4096)
    p.add_argument("--q-reg", type=float, nargs="+", default=[0.0, 0.01], help="BPR L2 weights to train")
    p.add_argument("--q-lr", type=float, nargs="+", default=[0.05, 0.2])
    p.add_argument("--skip-throughput", action="store_true")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mf_bpr_bench.py measures on a GPU; none is visible")
    import fps_b200  # noqa: F401
    from fps_b200.ops import native

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"card": card(), "shape": {"users": USERS, "items": ITEMS, "k": K, "positives_per_step": BATCH,
                                      "micro_batches": -(-BATCH // min(ITEMS, USERS)), "format": "packed64",
                                      "negatives_per_positive": 1}}
    if not a.skip_throughput:
        res["throughput"] = throughput(a, native, dev)
    res["quality"] = quality(a, dev)
    res["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
