#!/usr/bin/env python
"""Headline benchmark: matrix-factorisation updates/sec (BASELINE.json metric / config 2).

    python bench.py --gpus N --steps K --warmup W            # N=1
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W

Model/config: online SGD matrix factorisation, 10M users x 1M items, k=64, item vectors on the
parameter server sharded over the N GPUs (psParallelism=N), user vectors on the owning worker
(workerParallelism=N), synthetic uniform ratings, random-init factors.  One "step" = ``--batch``
ratings per GPU pushed through the fused pull+SGD+push kernel, as ceil(batch / min(items, local users))
conflict-free micro-batches (no user repeats within a step while the batch fits the local users, no item
within a micro-batch: at N=1 every launch updates each row at most once, so a step's result does not
depend on how the asynchronous kernel is scheduled); one
"update" = one (user, item, rating) SGD update (pull item, update user, push item delta).

Two measurements are printed on ONE JSON line by rank 0:
  value  -- device-timed (CUDA events, max over ranks), inputs already resident on the GPU;
  e2e    -- through the public API (`DeviceOnlineMF.fit_stream`): every step's ratings are
            copied from pinned host memory and the step's loss is read back to the host.

`--impl reference` would run the unmodified reference (Scala 2.11 / Flink 1.4 on a JVM); it is
not installable here (no setup.py/pyproject, no JVM, no sbt, no network), so it reports that.
"""
from __future__ import annotations

import argparse
import json
import os

import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REPO)


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=400)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--impl", default="fps_b200", choices=["fps_b200", "reference", "nccl"])
    p.add_argument("--users", type=int, default=10_000_000)
    p.add_argument("--items", type=int, default=1_000_000)
    p.add_argument("--factors", type=int, default=64)
    p.add_argument("--batch", type=int, default=4 * 1024 * 1024, help="ratings per GPU per step")
    p.add_argument("--lr", type=float, default=0.01)
    p.add_argument("--pull-limit", type=int, default=0, help="0 = hardware max rows in flight")
    p.add_argument("--host-buffers", type=int, default=6)
    p.add_argument("--format", default="packed64", choices=["packed64", "arrays"],
                   help="rating record format: packed64 = 8 B/update (user:26|item:22|fp16 rating), "
                        "arrays = int32 user, int32 item, fp32 rating (12 B/update)")
    p.add_argument("--item-cache", default="auto", choices=["auto", "on", "off"],
                   help="worker-side item cache + per-step delta merge (default: on when N > 1)")
    p.add_argument("--sync-every", type=int, default=4, help="item-cache: merge every k micro-batches")
    p.add_argument("--item-blocking", default="auto", choices=["auto", "on", "off"],
                   help="deal every micro-batch into <=16 MB item-table buckets before the fused kernel (L2 blocking)")
    p.add_argument("--update-rule", default="parity", choices=["parity", "plain"],
                   help="parity: the reference's e = sigmoid(r - u.v) (SGDUpdater.scala:8; always positive, so "
                        "the squared error drifts up by design); plain: e = r - u.v (textbook SGD, loss falls)")
    p.add_argument("--quality-updates-per-user", type=float, default=1200.0,
                   help="convergence gate (outside the timed regions): total update budget = this x users, the "
                        "same synthetic low-rank stream trained by the replica mode, the direct one-sided mode "
                        "and ONE worker alone, RMSE evaluated at 1/3 and at the full budget; 0 disables")
    p.add_argument("--quality-lr", type=float, default=0.05)
    p.add_argument("--quality-init", type=float, default=0.05)
    p.add_argument("--no-direct", action="store_true", help="skip the direct one-sided mode measurement (N > 1)")
    p.add_argument("--no-fp64", action="store_true",
                   help="skip the fp64 row (the reference's precision: Array[Double] factors)")
    p.add_argument("--no-numa-bind", action="store_true",
                   help="do not bind the process to the NUMA node of its GPU (utils/numa.py)")
    p.add_argument("--kernel", default=None, choices=[None, "tma", "reg"],
                   help="fused MF kernel variant (default: reg = register-staged loads at full occupancy)")
    p.add_argument("--dump-outputs", metavar="DIR", default=None,
                   help="after the timed steps, write what they computed to DIR/<name>.npy (see dump_outputs)")
    a = p.parse_args()
    if a.dump_outputs and a.impl != "fps_b200":
        p.error("--dump-outputs needs --impl fps_b200")
    return a


DUMP_SEED = 20251015
DUMP_BYTES_PER_TABLE = 24 << 20      # ids + vectors of one table; two tables + stats stay below 64 MB


def dump_outputs(directory, model, world, rank):
    """The model state the timed steps leave behind, as a caller of ``DeviceOnlineMF.step`` sees it:

    * ``stats.npy``         float64 [2]: (sum of squared errors, updates) of the last timed step;
    * ``user_ids.npy``      float64 [m]: a fixed, seeded sample of rank 0's users (sorted; ids < 2^53 are exact);
    * ``user_vectors.npy``  float32 [m, k]: their factor vectors;
    * ``item_ids.npy``      float64 [m']: a fixed, seeded sample of all items (sorted);
    * ``item_vectors.npy``  float32 [m', k]: their factor vectors, pulled from the parameter server.

    At most 24 MB of ids + vectors per table (48 MB in all), so runs of two builds can be compared row for row.
    At N=1 the micro-batches are conflict-free, so two runs with the same arguments write the same vectors
    (``stats`` up to the order of its fp32 atomic sums)."""
    import numpy as np
    import torch

    if rank != 0:
        return
    os.makedirs(directory, exist_ok=True)
    k = model.k
    m_max = max(1, DUMP_BYTES_PER_TABLE // (8 + 4 * k))      # float64 id + k float32 per row
    g = torch.Generator().manual_seed(DUMP_SEED)
    n_local = model.users.shape[0]
    slots = torch.randperm(n_local, generator=g)[:m_max].sort().values
    slots = slots[slots * world + rank < model.num_users]
    uvec = model.users[slots.to(model.cuda_device), :k]
    ids = torch.randperm(model.num_items, generator=g)[:m_max].sort().values
    ivec = model.items.pull(ids.to(device=model.cuda_device, dtype=torch.int32))[:, :k]
    out = {"stats": model.stats.double(), "user_ids": (slots * world + rank).double(), "user_vectors": uvec,
           "item_ids": ids.double(), "item_vectors": ivec}
    for name, t in out.items():
        np.save(os.path.join(directory, name + ".npy"), t.cpu().numpy())


class ClockSampler:
    """Sample SM clocks / throttle reasons with nvidia-smi during the timed region."""

    Q = ("timestamp,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx = gpu_index
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.idx), f"--query-gpu={self.Q}",
                 "--format=csv,noheader,nounits", "-lms", "50"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None

    def stop(self, windows=()):
        """Summarise samples that fall inside the timed ``windows`` [(t0, t1) wall-clock seconds]."""
        import datetime

        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            out, _ = self.proc.communicate(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            out, _ = self.proc.communicate()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        rows = []
        for line in out.strip().splitlines():
            f = [x.strip() for x in line.split(",")]
            if len(f) < 9:
                continue
            try:
                ts = datetime.datetime.strptime(f[0], "%Y/%m/%d %H:%M:%S.%f").timestamp()
                rows.append((ts, float(f[1]), float(f[2]), float(f[3]),
                             [n for n, v in zip(names, f[5:9]) if v.lower().startswith("active")]))
            except ValueError:
                continue
        inside = [r for r in rows if any(t0 - 0.05 <= r[0] <= t1 + 0.05 for t0, t1 in windows)]
        window = "timed regions"
        if not inside:
            inside, window = rows, "whole run (timed regions shorter than the sampling period)"
        reasons = sorted({n for r in inside for n in r[4]})
        return {"sm_mhz": statistics.median([r[1] for r in inside]) if inside else None,
                "sm_max_mhz": max([r[2] for r in inside]) if inside else None,
                "power_w_max": max([r[3] for r in inside]) if inside else None,
                "samples": len(inside), "window": window, "reasons": reasons}


def quality_gate(a, world, rank, dev, shared_gpu, DeviceOnlineMF, ERR_PLAIN, sync_list=None, checkpoints=None):
    """Same synthetic low-rank rating stream, same update budget, plain-residual SGD: N workers in
    replica mode, N workers in direct one-sided mode, and ONE worker alone; held-out RMSE of each
    (``checkpoints``: budgets, in updates per user, at which the RMSE is evaluated)."""
    import torch
    import torch.distributed as dist
    from fps_b200.utils.synthetic import lowrank_ratings

    cps = sorted(checkpoints or [a.quality_updates_per_user])
    steps_at = [max(8, int(c * a.users / (a.batch * world))) for c in cps]
    init = a.quality_init

    def batch_of(rid, step):
        g = torch.Generator(device=dev).manual_seed(7919 * step + rid + 1)
        u = torch.randint(0, a.users // world, (a.batch,), generator=g, device=dev, dtype=torch.int32) * world + rid
        i = torch.randint(0, a.items, (a.batch,), generator=g, device=dev, dtype=torch.int32)
        return u, i, lowrank_ratings(u, i)

    gh = torch.Generator(device=dev).manual_seed(99991)
    hu = torch.randint(0, a.users, (1 << 20,), generator=gh, device=dev, dtype=torch.int32)
    hi = torch.randint(0, a.items, (1 << 20,), generator=gh, device=dev, dtype=torch.int32)
    hr = lowrank_ratings(hu, hi)

    def rmse(model, w, r):
        mine = (hu % w) == r
        pred = model.predict(hu[mine], hi[mine])
        t = torch.stack([((hr[mine] - pred) ** 2).sum().double(), mine.sum().double()])
        if w > 1:
            if shared_gpu:
                h = t.cpu(); dist.all_reduce(h); t = h
            else:
                dist.all_reduce(t)
        return float((t[0] / t[1]).sqrt())

    def curve(model, w, r, batches_of_step):
        out, done = [], 0
        for n in steps_at:
            for s in range(done, n):
                for b in batches_of_step(s):
                    model.step(*b)
            done = n
            model.refresh()
            model.check_finite()
            out.append(rmse(model, w, r))
        return out

    kw = dict(learning_rate=a.quality_lr, range_min=-init, range_max=init, seed=4321, err_mode=ERR_PLAIN)
    out = {"update_rule": "plain residual e = r - u.v", "lr": a.quality_lr, "init": init,
           "data": "rank-8 synthetic ratings (utils/synthetic.py), std 0.5", "updates_per_user": cps,
           "steps_per_worker": steps_at, "updates": [n * a.batch * world for n in steps_at],
           "rmse_untrained": float(hr.std())}
    curves = {}
    if world > 1:
        runs = [("direct", False, a.sync_every)] if not getattr(a, "skip_direct_quality", False) else []
        runs += [("replica", True, a.sync_every)]
        runs += [(f"replica_sync{se}", True, se) for se in (sync_list or []) if se != a.sync_every]
        for mode, cache, se in runs:
            m = DeviceOnlineMF(a.users, a.items, a.factors, item_cache=cache, sync_every=se, **kw)
            curves[mode] = curve(m, world, rank, lambda s: [batch_of(rank, s)])
            m.barrier(); m.close(); del m
        groups = [dist.new_group([r]) for r in range(world)]
        solo = DeviceOnlineMF(a.users, a.items, a.factors, group=groups[rank], **kw) if rank == 0 else None
    else:
        solo = DeviceOnlineMF(a.users, a.items, a.factors, **kw)
    ref = torch.zeros(len(cps), dtype=torch.float64, device="cpu" if shared_gpu else dev)
    if rank == 0:
        c = curve(solo, 1, 0, lambda s: [batch_of(rid, s) for rid in range(world)])
        ref[:] = torch.tensor(c, dtype=torch.float64)
        solo.close()
    if world > 1:
        dist.all_reduce(ref)
    curves["single_worker"] = [float(x) for x in ref]
    single = curves["single_worker"]
    for k, v in curves.items():
        out["rmse_" + k] = v if len(cps) > 1 else v[0]
    if world > 1:
        out["sync_every"] = a.sync_every
        for k, v in curves.items():
            if k != "single_worker":
                ratio = [x / y for x, y in zip(v, single)]
                out[k + "_vs_single"] = ratio if len(cps) > 1 else ratio[0]
        r_last = curves["replica"][-1] / single[-1]
        d_last = (curves["direct"][-1] / single[-1]) if "direct" in curves else None
        out["within_2pct"] = bool(abs(r_last - 1) <= 0.02 and (d_last is None or abs(d_last - 1) <= 0.02))
    return out


def main():
    a = parse()
    if a.impl == "reference":
        if int(os.environ.get("RANK", "0")) == 0:      # under torch.distributed.run: one line, from rank 0
            print(json.dumps({"impl": "reference", "n_gpus": a.gpus, "unavailable":
                              "reference is Scala 2.11 / Apache Flink 1.4 (no setup.py/pyproject: pip "
                              "reports 'not installable'); image has no JVM, sbt or network"}), flush=True)
        return 0

    import torch
    import torch.distributed as dist

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != a.gpus and world > 1:
        raise SystemExit(f"--gpus {a.gpus} but WORLD_SIZE={world}")
    n_dev = torch.cuda.device_count()
    shared_gpu = world > 1 and (os.environ.get("FPS_SHARE_GPU") == "1" or n_dev < world)
    local_rank = local_rank % max(n_dev, 1) if shared_gpu else local_rank
    # torchrun does not place its children: put this worker (and the pinned buffers it allocates below) on the
    # NUMA node of its GPU, so the per-step H2D copies do not cross the inter-socket link (best effort, no-op
    # on a single-node box or with FPS_NUMA_BIND=0)
    numa_info = None
    if not a.no_numa_bind:
        try:
            from fps_b200.utils.numa import bind_to_gpu_node

            numa_info = bind_to_gpu_node(local_rank, min_cpus=8)   # fewer local CPUs: memory policy only
        except Exception as exc:      # placement is an optimisation, never a reason to fail
            numa_info = {"error": f"{type(exc).__name__}: {exc}"}
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    saved_stdout = os.dup(1)
    os.dup2(2, 1)          # NCCL prints its version banner on stdout; rank 0 must print ONE JSON line
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        if shared_gpu:     # functional runs only: ranks share a GPU, gloo control plane, CUDA-IPC data plane
            dist.init_process_group("gloo")
        else:
            dist.init_process_group("nccl", device_id=dev)

    def max_over_ranks(x: float) -> float:
        if world == 1:
            return float(x)
        t = torch.tensor([x], dtype=torch.float64, device="cpu" if shared_gpu else dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    from fps_b200.ops import native
    from fps_b200.models.mf.device import DeviceOnlineMF, ERR_PLAIN, ERR_SIGMOID

    if a.impl == "nccl":
        from fps_b200.parallel.nccl_baseline import NcclOnlineMF as Model
    else:
        Model = DeviceOnlineMF
    n_local_users = a.users // world  # every generated user id stays < users and owned by rank
    n_sub = -(-a.batch // min(a.items, n_local_users))   # conflict-free micro-batches per step (see below)
    cache = {"auto": None, "on": True, "off": False}[a.item_cache]
    extra = {} if a.impl == "nccl" else {"item_blocking": {"auto": None, "on": True, "off": False}[a.item_blocking]}
    model = Model(a.users, a.items, a.factors, learning_rate=a.lr, pull_limit=a.pull_limit,
                  seed=1234, err_mode=ERR_SIGMOID if a.update_rule == "parity" else ERR_PLAIN,
                  kernel=a.kernel, item_cache=cache,
                  # the replica policy counts step() calls: every row is still exchanged once per
                  # --sync-every steps, one slice per micro-batch
                  sync_every=a.sync_every * n_sub, **extra)

    # ---- synthetic ratings: users owned by this worker (user % W == rank), uniform items -------
    # A step's ratings come as conflict-free micro-batches (distinct users in the step -- in each micro-batch
    # when the batch exceeds the local users -- and distinct items in a micro-batch): the fused kernel then
    # updates every row at most once per launch, and what a step computes is a function of its inputs alone,
    # not of the order in which the asynchronous kernel's warps happen to run.
    g = torch.Generator().manual_seed(1000 + rank)
    sizes = [len(c) for c in torch.arange(a.batch).tensor_split(n_sub)]
    host = []           # host[b] = the micro-batches of one step
    for _ in range(a.host_buffers):
        step = []
        if a.batch <= n_local_users:
            step_users = torch.randperm(n_local_users, generator=g)[:a.batch].split(sizes)
        for j, n in enumerate(sizes):
            u = step_users[j] if a.batch <= n_local_users else torch.randperm(n_local_users, generator=g)[:n]
            u = u.to(torch.int32) * world + rank
            i = torch.randperm(a.items, generator=g)[:n].to(torch.int32)
            r = torch.rand(n, generator=g, dtype=torch.float32).half().float()  # fp16-exact ratings
            if a.format == "packed64" and a.impl == "fps_b200":
                step.append((native.pack_ratings(u, i, r).pin_memory(),))
            else:
                step.append((u.pin_memory(), i.pin_memory(), r.pin_memory()))
        host.append(step)
    devb = [[tuple(t.to(dev) for t in b) for b in step] for step in host]

    def run_step(m, s, reset_stats=False):
        if reset_stats:
            m.stats.zero_()    # the step's loss, as fit_stream reports it
        for b in devb[s % len(devb)]:
            m.step(*b)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- device-timed --------------------------------------------------------------------------
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    windows = []
    for s in range(a.warmup):
        run_step(model, s, reset_stats=True)
    if hasattr(model, "flush"):
        model.flush()          # warm-up covers every kernel of the timed region, the end-of-run merge included
    barrier()
    w0 = time.time()
    launches0 = native.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(a.steps):
        run_step(model, a.warmup + s, reset_stats=True)
    e_mid = torch.cuda.Event(enable_timing=True)
    e_mid.record()
    if hasattr(model, "flush"):
        model.flush()          # item-cache mode: the timed region includes every delta merge
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    merge_ms = e_mid.elapsed_time(e1)      # end-of-run merge of the replica mode (inside the timed region)
    launches = native.launch_count() - launches0
    windows.append((w0, time.time()))
    barrier()
    ms_max = max_over_ranks(ms)
    model.check_finite()
    if a.dump_outputs:
        dump_outputs(a.dump_outputs, model, world, rank)
        barrier()          # the other ranks' shards stay as the timed steps left them until rank 0 has read them

    # ---- end to end through the public API -----------------------------------------------------
    def stream(n):
        for s in range(n):
            yield from host[s % len(host)]

    for _ in model.fit_stream(stream(a.warmup)):
        pass
    barrier()
    w0 = time.time()
    t0 = time.perf_counter()
    e0.record()
    n_res = 0
    last = [0.0, 0.0]        # (sum of squared errors, updates) of the last step's micro-batches
    for sse, n in model.fit_stream(stream(a.steps)):
        if n_res % n_sub == 0:
            last = [0.0, 0.0]
        last[0] += sse; last[1] += n
        n_res += 1
    e1.record()
    torch.cuda.synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3
    windows.append((w0, time.time()))
    e2e_ms = max(e0.elapsed_time(e1), wall_ms)
    e2e_ms_max = max_over_ranks(e2e_ms)
    assert n_res == a.steps * n_sub
    h2d = sum(x.numel() * x.element_size() for b in host[0] for x in b)
    barrier()

    # ---- the north-star path on the record: direct one-sided mode (every update pulls its item row from
    #      the owner and pushes the delta back inside the fused kernel; no replica) -----------------------
    direct = None
    if world > 1 and a.impl == "fps_b200" and not a.no_direct and getattr(model, "item_cache", False):
        dm = DeviceOnlineMF(a.users, a.items, a.factors, learning_rate=a.lr, pull_limit=a.pull_limit,
                            seed=1234, err_mode=ERR_SIGMOID if a.update_rule == "parity" else ERR_PLAIN,
                            kernel=a.kernel, item_cache=False)
        for s in range(a.warmup):
            run_step(dm, s)
        barrier()
        w0 = time.time()
        e0.record()
        for s in range(a.steps):
            run_step(dm, a.warmup + s)
        e1.record()
        torch.cuda.synchronize()
        d_ms = max_over_ranks(e0.elapsed_time(e1))
        windows.append((w0, time.time()))
        dm.check_finite()
        barrier()
        dm.close()
        del dm
        direct = {"value": a.steps * a.batch * world / (d_ms / 1e3), "unit": "updates/s",
                  "ms_per_step": d_ms / a.steps,
                  "note": "item_cache off: per-update one-sided pull (peer LDG.128) + push (REDG.ADD.F32x4) "
                          "over NVLink inside the fused kernel; link bound for remote rows"}
    # ---- the reference's precision: fp64 tables and math (Vector.scala:8), direct one-sided mode -----------------
    fp64 = None
    if a.impl == "fps_b200" and not a.no_fp64:
        from fps_b200.models.mf.device_f64 import DeviceOnlineMFf64

        fm = DeviceOnlineMFf64(a.users, a.items, a.factors, learning_rate=a.lr, seed=1234,
                               err_mode=ERR_SIGMOID if a.update_rule == "parity" else ERR_PLAIN)
        for s in range(a.warmup):
            run_step(fm, s)
        barrier()
        w0 = time.time()
        e0.record()
        for s in range(a.steps):
            run_step(fm, a.warmup + s)
        e1.record()
        torch.cuda.synchronize()
        f_ms = max_over_ranks(e0.elapsed_time(e1))
        windows.append((w0, time.time()))
        fm.check_finite()
        barrier()
        fm.close()
        del fm
        fp64 = {"value": a.steps * a.batch * world / (f_ms / 1e3), "unit": "updates/s", "ms_per_step": f_ms / a.steps,
                "note": "fp64 tables and math like the reference (Array[Double]); 512-byte rows, "
                        "ld.global.v2.f64 pulls + red.global.add.f64 pushes; direct one-sided mode at N > 1"}
    clocks = sampler.stop(windows) if rank == 0 else None

    # ---- convergence gate (outside every timed region) ---------------------------------------------
    quality = None
    if a.impl == "fps_b200" and a.quality_updates_per_user > 0:
        try:
            quality = quality_gate(a, world, rank, dev, shared_gpu, DeviceOnlineMF, ERR_PLAIN,
                                   checkpoints=[a.quality_updates_per_user / 3, a.quality_updates_per_user])
        except Exception as exc:     # the headline line must be printed whatever happens here
            quality = {"error": f"{type(exc).__name__}: {exc}"}
        barrier()

    if rank == 0:
        total_updates = a.steps * a.batch * world
        value = total_updates / (ms_max / 1e3)
        e2e_value = total_updates / (e2e_ms_max / 1e3)
        out = {
            "metric": "matrix-factorization updates/sec (whole box, max over ranks)",
            "value": value, "unit": "updates/s", "n_gpus": world, "steps": a.steps,
            "warmup": a.warmup, "ms_per_step": ms_max / a.steps, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
            "impl": a.impl, "kernel": a.kernel or os.environ.get("FPS_MF_KERNEL", "reg"),
            "config": {"model": "online SGD MF 10Mx1M k=64 (psOnlineMF)", "users": a.users,
                       "items": a.items, "factors": a.factors,
                       "global_batch": a.batch * world, "per_gpu_batch": a.batch,
                       "micro_batches_per_step": n_sub,
                       "seq_len": None, "parallelism": f"workers{world}xps{world}",
                       "partition": "user%W on workers, item%G on PS shards",
                       "l2": "inputs larger than L2: 2.8 GB of factor tables accessed at random, "
                             f"{len(host)} distinct {h2d >> 20} MiB rating steps cycled",
                       "pull_limit": a.pull_limit or "hardware max rows in flight",
                       "item_cache": bool(getattr(model, "item_cache", False)),
                       "sync_every": a.sync_every,
                       "sync_every_note": "in steps; the replica policy runs per micro-batch with "
                                          f"sync_every={a.sync_every * n_sub} slices",
                       "item_blocking": (f"{model.block_buckets} buckets of {1 << model.block_shift} item rows, "
                                         "reordered inside the timed step (2 extra kernels)"
                                         if getattr(model, "item_blocking", False) else False),
                       "record_format": a.format if a.impl == "fps_b200" else "arrays",
                       "update_rule": ("reference parity e=sigmoid(r-u.v) (SGDUpdater.scala:8): e>0 always, so the "
                                       "reported mse drifts upward by design; --update-rule plain trains with "
                                       "e=r-u.v at the same speed" if a.update_rule == "parity"
                                       else "plain residual e=r-u.v"),
                       "precision_note": "fp32 tables and math (reference: fp64 on the JVM)",
                       "exchange": ({"ctas": model.replica.n_ctas, "stages": model.replica.stages,
                                     "sliced": model.replica.sliced, "own_shard_in_place": model.replica.own is not None,
                                     "kernel_ms": model.replica.timing_summary(),
                                     "final_merge_ms": merge_ms,
                                     "final_merge_note": "the timed region ends with a full (all slices, all "
                                                         "destinations) delta merge that is not overlapped with "
                                                         "training; rank 0's device time of it, included in value"}
                                    if getattr(model, "replica", None) is not None else None),
                       "host_placement": numa_info,
                       "quality": quality},
            "value_direct": direct,
            "value_fp64": fp64,
            "clocks": clocks,
            "e2e": {"value": e2e_value, "unit": "updates/s", "ms_per_step": e2e_ms_max / a.steps,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 8 * n_sub,
                    "last_step_mse": (last[0] / last[1]) if last[1] else None},
            "gpu_launches": launches,
        }
        sys.stdout.flush()
        os.dup2(saved_stdout, 1)
        print(json.dumps(out), flush=True)
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
