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

``--window`` records the step window instead (``DeviceOnlineMF(step_window=8)``, fps_mf_window.cu), written to
``profiles/h100_mf_step_window.json`` by default: device times of the staging copies and of the drain for each
kernel variant (CUDA events and ``torch.profiler``), the bytes model of a windowed step next to them, TB/s against
the ``copy_`` ceiling, the drain's split into its build phase (scatter rounds) and its apply phase (chains) from
the kernel's own ``%globaltimer`` marks, and A/B rows of the windowed and the per-launch step alternated round by
round.
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
    if "mf_window" in n:
        return "drain"
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
        c = {"gpu_memset": "memset", "gpu_memcpy": "staging_copy"}.get(e["cat"]) or kernel_class(e["name"])
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


# FPS_MF_WINDOW_VARIANT at k = 64: (float4 per lane, user rows prefetched, CTAs/SM); see dispatch_window
WINDOW_VARIANTS = {"v4_p2_2cta": "0", "v1_p4_3cta": "2", "v1_p8_2cta": "1"}


def window_bytes_model(step, row_bytes):
    """Bytes one windowed step moves, computed from the step's records (packed64)."""
    rec = torch.cat(step)
    n = rec.numel()
    touched = int(torch.unique((rec >> 16) & 0x3FFFFF).numel())
    staging = 2 * 8 * n                        # D2D copy into the staging slots: read + write
    drain_records = 8 * n                      # the drain reads every staged record once
    slot_table = 3 * 8 * n                     # T entry: atomicExch, chain read, reset (may stay in L2)
    users = 2 * row_bytes * n                  # every user row read and written once
    items = 2 * row_bytes * touched            # every touched item row read and written once
    return {"records": n, "touched_item_rows": touched, "row_bytes": row_bytes,
            "staging_copy_bytes": staging, "drain_record_bytes": drain_records, "slot_table_bytes": slot_table,
            "user_rows_bytes": users, "item_rows_bytes": items,
            "drain_bytes": users + items + drain_records + slot_table,
            "chain_bytes": users + items + 2 * 8 * n,   # rows, and each T entry read and reset by the chain
            "per_launch_bytes": 2 * row_bytes * n * 2 + 8 * n,
            "note": "computed from shapes and the step's item ids; slot-table and bitmap traffic are upper bounds "
                    "(they may be served by L2)"}


def window_split(model, steps, n_steps):
    """Device time of the staging copies and of the drain of each step, separately (CUDA events), and the drain's
    build and apply phases (the kernel's %globaltimer marks, CTA 0 after each grid sync)."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    stage_ms, drain_ms, build_ms, apply_ms = [], [], [], []
    model._win_phase_ns = torch.zeros(4, dtype=torch.int64, device=model.cuda_device)
    for s in range(n_steps):
        model.stats.zero_()
        model._win_phase_ns.zero_()
        ev[0].record()
        for b in steps[s % len(steps)]:
            model._stage(b, None, None)
        ev[1].record()
        model._drain()
        ev[2].record()
        torch.cuda.synchronize()
        stage_ms.append(ev[0].elapsed_time(ev[1]))
        drain_ms.append(ev[1].elapsed_time(ev[2]))
        ph = model._win_phase_ns.tolist()
        build_ms.append(ph[0] * 1e-6)
        apply_ms.append(ph[1] * 1e-6)
    model._win_phase_ns = None
    return (statistics.median(stage_ms), statistics.median(drain_ms), statistics.median(build_ms),
            statistics.median(apply_ms))


def window_main(a, res, steps, sizes, DeviceOnlineMF):
    ref = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=0.01, seed=1234, step_window=0)
    win = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=0.01, seed=1234, step_window=8)
    row_bytes = win._items.stride * 4
    bm = window_bytes_model(steps[0], row_bytes)
    ceiling = res["hbm_copy"]["tb_per_s"]
    res["window"] = {"step_window": win.step_window, "bytes_model": bm, "variants": {}}
    arms = {"per_launch": (ref, None)}
    arms.update({"window_" + v: (win, code) for v, code in WINDOW_VARIANTS.items()})
    for m, code in arms.values():               # warm every kernel
        if code is not None:
            os.environ["FPS_MF_WINDOW_VARIANT"] = code
        timed(m, steps, a.warmup, 0)
    for v, code in WINDOW_VARIANTS.items():
        os.environ["FPS_MF_WINDOW_VARIANT"] = code
        stage, drain, build, chain = window_split(win, steps, a.steps)
        prof = profile(win, steps, 4)
        res["window"]["variants"][v] = {
            "staging_ms_per_step": stage, "drain_ms_per_step": drain,
            "build_ms_per_step": build, "chain_ms_per_step": chain,
            "chain_tb_per_s": bm["chain_bytes"] / (chain * 1e-3) / 1e12,
            "drain_tb_per_s": bm["drain_bytes"] / (drain * 1e-3) / 1e12,
            "drain_share_of_copy_ceiling": bm["drain_bytes"] / (drain * 1e-3) / 1e12 / ceiling,
            "staging_tb_per_s": bm["staging_copy_bytes"] / (stage * 1e-3) / 1e12,
            "profile": prof}
    ms = {c: [] for c in arms}
    names = list(arms)
    for r in range(a.rounds):
        for c in (names if r % 2 == 0 else names[::-1]):
            m, code = arms[c]
            if code is not None:
                os.environ["FPS_MF_WINDOW_VARIANT"] = code
            ms[c].append(timed(m, steps, a.steps, r))
    os.environ.pop("FPS_MF_WINDOW_VARIANT", None)
    base = statistics.median(ms["per_launch"])
    res["ab"] = {c: {"ms_per_step": v, "median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v),
                     "updates_per_s_median": BATCH / (statistics.median(v) * 1e-3),
                     "speedup_vs_per_launch": base / statistics.median(v)}
                 for c, v in ms.items()}
    res["ab_note"] = (f"{a.rounds} rounds x {a.steps} steps per arm, arms alternated (reversed order every other "
                      "round); device time per step from CUDA events, stats reset + staging + drain included")
    res["per_launch_profile"] = profile(ref, steps, 4)
    res["per_launch_profile"]["bytes_tb_per_s"] = bm["per_launch_bytes"] / (
        res["per_launch_profile"]["busy_us_per_step"] * 1e-6) / 1e12
    for m in (win, ref):
        m.check_finite()
        m.close()
    return {c: res["ab"][c]["median_ms"] for c in names}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=None)
    p.add_argument("--window", action="store_true", help="record the step window (see the module docstring)")
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--steps", type=int, default=40)
    p.add_argument("--warmup", type=int, default=4)
    p.add_argument("--configs", default=",".join(CONFIGS))
    a = p.parse_args()
    if a.out is None:
        a.out = os.path.join(REPO, "profiles", "h100_mf_step_window.json" if a.window
                             else "h100_mf_step_breakdown.json")

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    from fps_b200.models.mf.device import DeviceOnlineMF
    from fps_b200.ops import native

    res = {"card": card(), "shape": {"users": USERS, "items": ITEMS, "factors": K, "batch": BATCH,
                                    "data": "bench.py --gpus 1 micro-batches (seed 1000, packed64)"}}
    res["hbm_copy"] = hbm_ceiling()
    steps, sizes = bench_batches(native, dev)
    res["shape"]["micro_batches_per_step"] = len(sizes)
    if a.window:
        summary = window_main(a, res, steps, sizes, DeviceOnlineMF)
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps(summary))
        return
    model = DeviceOnlineMF(USERS, ITEMS, K, learning_rate=0.01, seed=1234, item_blocking=True,
                           step_window=0)
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
