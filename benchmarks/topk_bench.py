#!/usr/bin/env python
"""Top-K scoring benchmark (K6): B queries pulled from the PS x N local items, k=64, K=100.
Reports device time per batch, TF32 tensor throughput of the two GEMM passes and the comparison with
torch (cuBLAS fp32 matmul + torch.topk) on the same data.

``--exclude 0,100,1000``: instead, per-query exclusion lists of E items (half the query's own exact
top-E, which drives theta down, half uniform ids).  For each E, plain and length-sorted tables, it
times ``topk(K, exclude=...)`` (and, separately, its exclusion-list normalisation), plain ``topk(K)``
and the over-fetch it replaces (``topk(K + E)`` and a device-side filter), checks that the exclusion result equals the over-fetch wherever that returns
K items, and counts the rows answered by the brute-force fallback.  One JSON line, with the card's
name and power limit read in the same run."""
import argparse
import json
import os

import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def t_ms(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=2048)
    ap.add_argument("--factors", type=int, default=64)
    ap.add_argument("--K", type=int, default=100)
    ap.add_argument("--skew", type=float, default=0.0,
                    help="> 0: log-normal item lengths with this sigma (popularity skew) instead of U[0.05, 2.05)")
    ap.add_argument("--pass1-fraction", type=float, default=0.0,
                    help="> 0: also time DeviceTopK(pass1_fraction=f) (theta from a prefix of the tiles)")
    ap.add_argument("--exclude", type=str, default=None,
                    help="comma list of E: time top-K with E excluded items per query (see module doc)")
    ap.add_argument("--out", type=str, default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    users = ShardedTable(a.users, a.factors, seed=1, init_range=(-1, 1))
    items = ShardedTable(a.items, a.factors, seed=2, init_range=(-1, 1))
    # LEMP-style: make item lengths heterogeneous so tile pruning has something to prune
    if a.skew > 0:
        items.local.mul_(torch.exp(torch.randn(items.local.shape[0], 1, device=dev) * a.skew))
    else:
        items.local.mul_(torch.rand(items.local.shape[0], 1, device=dev) * 2 + 0.05)
    tk = DeviceTopK(items.local)
    q = torch.randint(0, a.users, (a.queries,), device=dev)
    if a.exclude is not None:
        res = exclude_bench(a, users, items, q, [int(e) for e in a.exclude.split(",")])
        line = json.dumps(res)
        print(line)
        if a.out:
            with open(a.out, "w") as f:
                f.write(line + "\n")
        return
    tile_max = torch.empty((a.queries, tk.n_tiles), dtype=torch.float32, device=dev)
    ms_pass1 = t_ms(lambda: native.topk_mma(items.local, 1, q_ids=q, q_tab=users.table_c, tile_max=tile_max))
    ms_total = t_ms(lambda: tk.topk(a.K, q_ids=q, q_table=users), iters=5, warm=2)

    def torch_ref():
        u = users.pull(q)
        return torch.topk(u @ items.local[:, : a.factors].T, a.K, dim=1)

    ms_torch = t_ms(torch_ref, iters=5, warm=2)
    tkp = DeviceTopK(items.local, sort_by_length=True)       # LEMP LENGTH bound at tile granularity
    ms_pruned = t_ms(lambda: tkp.topk(a.K, q_ids=q, q_table=users), iters=5, warm=2)
    p1, p2 = tkp.last_tiles_scored
    ms_frac = None
    if a.pass1_fraction > 0:
        tkf = DeviceTopK(items.local, pass1_fraction=a.pass1_fraction)
        ms_frac = t_ms(lambda: tkf.topk(a.K, q_ids=q, q_table=users), iters=5, warm=2)
        ref_s, _ = tk.topk(a.K, q_ids=q, q_table=users)
        got_s, _ = tkf.topk(a.K, q_ids=q, q_table=users)
        assert torch.equal(ref_s, got_s), "pass1_fraction changed the result"
    for name, t in (("plain", tk), ("pruned", tkp)):       # per-stage breakdown (synchronising trace)
        t.trace = []; t._t0 = None
        t.topk(a.K, q_ids=q, q_table=users)
        print(name, " ".join(f"{lbl}={ms:.3f}" for lbl, ms in t.trace), file=sys.stderr)
        t.trace = None
    flops = 2.0 * a.queries * a.items * a.factors
    print(json.dumps({"queries": a.queries, "items": a.items, "factors": a.factors, "K": a.K,
                      "pass1_ms": ms_pass1, "pass1_tf32_TFLOPs": flops / ms_pass1 / 1e9,
                      "topk_total_ms": ms_total, "queries_per_s": a.queries / ms_total * 1e3,
                      "pass1_fraction": a.pass1_fraction, "pass1_fraction_total_ms": ms_frac,
                      "length_pruned_total_ms": ms_pruned, "tiles": tkp.n_tiles, "tiles_pass1": p1,
                      "tiles_pass2": p2, "skew": a.skew,
                      "torch_matmul_topk_ms": ms_torch, "speedup_vs_torch": ms_torch / ms_total}))


def gpu_info() -> dict:
    """Name and power limit of GPU 0, read with nvidia-smi (read-only query)."""
    import subprocess

    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power, clock = [x.strip() for x in out.strip().split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:            # the timing is still valid; say why the card is unnamed
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e.__class__.__name__})"}


def filter_overfetch(sc, rows, ex_sorted, K):
    """The approach exclusion replaces: drop the excluded ids from a longer list, keep the first K."""
    at = torch.searchsorted(ex_sorted, rows).clamp_max(ex_sorted.shape[1] - 1)
    keep = torch.gather(ex_sorted, 1, at) != rows
    n, L = rows.shape
    order = torch.where(keep, torch.arange(L, device=rows.device).expand(n, L), L)
    first = torch.sort(order, dim=1).values[:, :K]
    ok = first < L
    first = first.clamp_max(L - 1)
    return (torch.where(ok, torch.gather(sc, 1, first), -3.0e38),
            torch.where(ok, torch.gather(rows, 1, first), -1))


def exclude_bench(a, users, items, q, e_list):
    from fps_b200.models.mf.device_topk import DeviceTopK, normalize_exclude

    dev = q.device
    g = torch.Generator(device=dev).manual_seed(17)
    out = {"queries": a.queries, "items": a.items, "factors": a.factors, "K": a.K, **gpu_info(), "runs": []}
    for sort in (False, True):
        tk = DeviceTopK(items.local, sort_by_length=sort)
        for E in e_list:
            ex_sorted = None
            if E > 0:
                own = tk.topk(E, q_ids=q, q_table=users)[1][:, : E - E // 2]          # exact top of the query
                rand = torch.randint(0, a.items, (a.queries, E // 2), generator=g, device=dev)
                ex = torch.cat([own, rand], 1)
                ex_sorted = torch.sort(ex, dim=1).values.contiguous()
                off = torch.arange(a.queries + 1, device=dev) * E
                exclude = (off, ex.reshape(-1))
            else:
                exclude = None
            run_ex = lambda: tk.topk(a.K, q_ids=q, q_table=users, exclude=exclude)
            run_plain = lambda: tk.topk(a.K, q_ids=q, q_table=users)

            def run_old():
                sc, rows = tk.topk(a.K + E, q_ids=q, q_table=users)
                return (sc, rows) if ex_sorted is None else filter_overfetch(sc, rows, ex_sorted, a.K)

            s_ex, r_ex = run_ex()
            fallback, tiles = tk.last_fallback_rows, list(tk.last_tiles_scored)
            s_old, r_old = run_old()
            times = {"ex": [], "plain": [], "old": []}
            for _ in range(3):                           # alternate the variants, keep each one's best
                for name, fn in (("ex", run_ex), ("plain", run_plain), ("old", run_old)):
                    times[name].append(t_ms(fn, iters=10, warm=2))
            ms_ex, ms_plain, ms_old = min(times["ex"]), min(times["plain"]), min(times["old"])
            # the exclusion-list normalisation alone (sort, de-duplication, host syncs), part of exclude_ms
            ms_norm = None if exclude is None else t_ms(
                lambda: normalize_exclude(exclude[0], exclude[1], a.queries, a.items, tk.inv_perm, device=dev),
                iters=10, warm=2)
            full = (r_old >= 0).all(dim=1)               # rows the over-fetch answered completely
            mismatch = int((~(s_ex == s_old).all(dim=1) & full).sum())
            out["runs"].append({"sort_by_length": sort, "E": E, "exclude_ms": ms_ex, "plain_ms": ms_plain,
                                "overfetch_filter_ms": ms_old, "normalize_ms": ms_norm, "exclude_over_plain": ms_ex / ms_plain,
                                "exclude_over_overfetch": ms_ex / ms_old, "fallback_rows": fallback,
                                "overfetch_short_rows": int((~full).sum()),
                                "exclude_short_rows": int((r_ex < 0).any(dim=1).sum()),
                                "score_mismatch_rows": mismatch, "tiles": tk.n_tiles,
                                "tiles_scored": tiles, "ms_all": times})
            print(json.dumps(out["runs"][-1]), file=sys.stderr)
    return out


if __name__ == "__main__":
    main()
