#!/usr/bin/env python
"""Where the time of one single-GPU MF step goes, at the shape and with the inputs of ``bench.py --gpus 1``.

    python benchmarks/mf_step_breakdown.py [--out profiles/h100_mf_step_breakdown.json]

Records, in one process:

* the card (name, power limit, max SM clock);
* per-kernel device times and the gaps between kernels, from ``torch.profiler`` (one run of its own);
* a bytes model of one micro-batch next to each kernel's time;
* a streaming HBM ceiling on the same card (``copy_`` of 2 GiB);
* A/B rows: the step's device time with 16 MB and 4 MB item buckets and without the deal, the configurations
  alternated round by round, with the spread over the rounds.  (``DeviceOnlineMF.step`` deals a micro-batch only
  when it has more records than the table has rows, so at this shape the bucket rows run without the deal too.)
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

USERS, ITEMS, K, BATCH, HOST_BUFFERS = 10_000_000, 1_000_000, 64, 4 * 1024 * 1024, 6


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
    """The micro-batches of ``bench.py --gpus 1`` (same generator, seed and order; packed64)."""
    n_sub = -(-BATCH // min(ITEMS, USERS))
    g = torch.Generator().manual_seed(1000)
    sizes = [len(c) for c in torch.arange(BATCH).tensor_split(n_sub)]
    steps = []
    for _ in range(HOST_BUFFERS):
        users = torch.randperm(USERS, generator=g)[:BATCH].split(sizes)
        step = []
        for j, n in enumerate(sizes):
            u = users[j].to(torch.int32)
            i = torch.randperm(ITEMS, generator=g)[:n].to(torch.int32)
            r = torch.rand(n, generator=g, dtype=torch.float32).half().float()
            step.append(native.pack_ratings(u, i, r).to(dev))
        steps.append(step)
    return steps, sizes


# name -> bytes of item rows per bucket of the L2-blocking deal (fps_bucket.cu); 0 = no deal
CONFIGS = {"bucket_16MB": 16 << 20, "bucket_4MB": 4 << 20, "no_blocking": 0}


def apply(model, block_bytes):
    if block_bytes == 0:
        model.block_buckets = 1           # one bucket: step() skips the deal
        return
    row_bytes = model.items.stride * 4
    shift = max(0, max(1, block_bytes // row_bytes).bit_length() - 1)
    while -(-ITEMS >> shift) > 64:
        shift += 1
    model.block_shift, model.block_buckets = shift, max(1, -(-ITEMS >> shift))


def timed(model, steps, n_steps, first):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(n_steps):
        model.stats.zero_()
        for b in steps[(first + s) % len(steps)]:
            model.step(b)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n_steps


def kernel_class(name: str) -> str:
    n = name.lower()
    if "memset" in n:
        return "memset"
    if "bucket" in n:                     # fps_bucket_deal_kernel (hist + scatter in older builds)
        return "bucket"
    if "mf_sgd_fused" in n:
        return "fused"
    return "other"


def profile(model, steps, n_steps):
    from torch.profiler import ProfilerActivity, profile as tprofile

    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        timed(model, steps, n_steps, 0)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    ev = [e for e in trace.get("traceEvents", [])
          if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    ev.sort(key=lambda e: e["ts"])
    per = {}
    for e in ev:
        c = "memset" if e["cat"] == "gpu_memset" else kernel_class(e["name"])
        if c == "other" and ("zero" in e["name"].lower() or "fill" in e["name"].lower()):
            c = "stats_reset"
        d = per.setdefault(c, {"count": 0, "us": 0.0, "names": set()})
        d["count"] += 1; d["us"] += e["dur"]; d["names"].add(e["name"][:120])
    busy = sum(e["dur"] for e in ev)
    span = (ev[-1]["ts"] + ev[-1]["dur"] - ev[0]["ts"]) if ev else 0.0
    gaps = [max(0.0, b["ts"] - (a["ts"] + a["dur"])) for a, b in zip(ev, ev[1:])]
    return {
        "steps": n_steps,
        "kernels": {c: {"launches_per_step": d["count"] / n_steps, "us_per_step": d["us"] / n_steps,
                        "us_per_launch": d["us"] / d["count"], "names": sorted(d["names"])}
                    for c, d in per.items()},
        "busy_us_per_step": busy / n_steps, "span_us_per_step": span / n_steps,
        "gap_us_per_step": sum(gaps) / n_steps,
        "gap_us_median": statistics.median(gaps) if gaps else None,
    }


def hbm_ceiling():
    x = torch.empty(1 << 29, dtype=torch.float32, device="cuda")   # 2 GiB
    x.uniform_()
    y = torch.empty_like(x)
    for _ in range(3):
        y.copy_(x)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        y.copy_(x)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    moved = 2 * x.numel() * 4
    del x, y
    torch.cuda.empty_cache()
    return {"bytes_per_copy": moved, "ms_per_copy": ms, "tb_per_s": moved / (ms * 1e-3) / 1e12}


def bytes_model(n_per_mb, row_bytes, record_bytes, sort_pass_bytes):
    user = n_per_mb * row_bytes * 2
    item = n_per_mb * row_bytes * 2
    return {
        "records_per_micro_batch": n_per_mb, "row_bytes": row_bytes,
        "user_rows_bytes": user, "item_rows_bytes": item,
        "records_read_by_fused_bytes": n_per_mb * record_bytes,
        "reorder_bytes": sort_pass_bytes,
        "note": "computed from shapes: each update reads and writes back one user row and one item row",
    }


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(REPO, "profiles", "h100_mf_step_breakdown.json"))
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--steps", type=int, default=40)
    p.add_argument("--warmup", type=int, default=4)
    p.add_argument("--configs", default=",".join(CONFIGS))
    a = p.parse_args()

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.ops import native

    res = {"card": card(), "shape": {"users": USERS, "items": ITEMS, "factors": K, "batch": BATCH,
                                    "data": "bench.py --gpus 1 micro-batches (seed 1000, packed64)"}}
    res["hbm_copy"] = hbm_ceiling()
    steps, sizes = bench_batches(native, dev)
    res["shape"]["micro_batches_per_step"] = len(sizes)
    model = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=0.01, seed=1234, item_blocking=True)
    row_bytes = model.items.stride * 4

    names = [c for c in a.configs.split(",") if c in CONFIGS]
    for c in names:                         # every configuration's kernels loaded and warm
        apply(model, CONFIGS[c])
        timed(model, steps, a.warmup, 0)
    ms = {c: [] for c in names}
    for r in range(a.rounds):
        order = names if r % 2 == 0 else names[::-1]
        for c in order:
            apply(model, CONFIGS[c])
            ms[c].append(timed(model, steps, a.steps, r))
    base = statistics.median(ms[names[0]])
    res["ab"] = {c: {"ms_per_step": v, "median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v),
                     "updates_per_s_median": BATCH / (statistics.median(v) * 1e-3),
                     "speedup_vs_" + names[0]: base / statistics.median(v)}
                 for c, v in ms.items()}
    res["ab_note"] = (f"{a.rounds} rounds x {a.steps} steps per configuration, configurations alternated "
                      "(reversed order every other round); device time per step from CUDA events")

    res["profiles"] = {}
    for c in names:
        apply(model, CONFIGS[c])
        prof = profile(model, steps, 4)
        fused = prof["kernels"].get("fused", {}).get("us_per_launch")
        bm = bytes_model(sizes[0], row_bytes, 8, 3 * 8 * sizes[0])   # hist reads, scatter reads + writes
        if fused:
            bm["fused_tb_per_s"] = (bm["user_rows_bytes"] + bm["item_rows_bytes"]
                                    + bm["records_read_by_fused_bytes"]) / (fused * 1e-6) / 1e12
        prof["bytes_model"] = bm
        res["profiles"][c] = prof
    model.check_finite()
    model.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({c: res["ab"][c]["median_ms"] for c in names}))


if __name__ == "__main__":
    main()
