#!/usr/bin/env python
"""Wide-row top-K benchmark: B queries pulled from a PS table x N local items, K=100, at row strides
128 (whole-tile kernel, the per-FLOP yardstick of the same run) and 132 .. 512 (K-streamed kernel),
with plain and length-sorted item tables.  Per stride it reports

* ms per ``DeviceTopK.topk`` (plain and length-sorted) and the tiles each pass scored;
* TF32 TFLOP/s of pass 1 (tile maxima) and pass 2 (candidates >= theta) over the whole table, from
  ``2 * B * N * stride`` and the kernel time, and the item bytes streamed from L2 to the SMs per second
  (every CTA row block reads the whole table: ``ceil(B / rows_per_cta) * N * stride * 4``);
* the rows answered by the brute-force fallback;
* cuBLAS fp32 matmul + ``torch.topk`` on the same data (chunked over queries), and how well the two
  result sets agree (share of the fp32 top-K ids found in the TF32 top-K, largest score difference).

Then it times ``DeviceSkipGram.most_similar`` (default 1024 words, K=10) on a 1M x 300 vocabulary
against normalised fp32 cuBLAS + ``torch.topk``.  One JSON line, with the card's name and power limit
read in the same run; ``--out`` also writes it to a file."""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from topk_bench import gpu_info, t_ms  # noqa: E402


def rows_per_cta(stride: int) -> int:
    """Query rows one CTA keeps resident (mirrors the launcher in csrc/fps_topk_mma.cu)."""
    kb = -(-stride // 32)
    if kb <= 4:
        return 128          # whole-tile kernel (2 x 128 for strides <= 64 with > 128 queries)
    return 128 if kb <= 10 else 64


def torch_topk(q, items, K, chunk):
    """cuBLAS fp32 matmul + torch.topk, ``chunk`` queries at a time."""
    vals, idx = [], []
    for a in range(0, q.shape[0], chunk):
        top = torch.topk(q[a:a + chunk] @ items.T, K, dim=1)
        vals.append(top.values); idx.append(top.indices)
    return torch.cat(vals), torch.cat(idx)


def agreement(rows, ref_idx, sc, ref_val):
    overlap = (ref_idx[:, :, None] == rows[:, None, :]).any(-1).float().mean().item()
    return overlap, (sc - ref_val).abs().max().item()


def stride_run(a, stride, dev):
    from fps_b200.models.mf.device_topk import DeviceTopK
    from fps_b200.ops import native
    from fps_b200.store.sharded_table import ShardedTable

    users = ShardedTable(a.users, stride, seed=1, init_range=(-1, 1))
    items = ShardedTable(a.items, stride, seed=2, init_range=(-1, 1))
    items.local.mul_(torch.rand(items.local.shape[0], 1, device=dev,
                                generator=torch.Generator(device=dev).manual_seed(3)) * 2 + 0.05)
    tab = items.local[: a.items]
    q = torch.randint(0, a.users, (a.queries,), device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    tk = DeviceTopK(tab)
    n_tiles = tk.n_tiles
    # ---- the two passes over the whole table, timed as kernels -----------------------------------
    tile_max = torch.empty((a.queries, n_tiles), dtype=torch.float32, device=dev)
    ms_p1 = t_ms(lambda: native.topk_mma(tab, 1, q_ids=q, q_tab=users.table_c, tile_max=tile_max))
    theta = native.row_kth_largest(tile_max, a.K)
    cap = 2048
    _, n_splits, _ = native.topk_geometry(tab, a.queries, 0, cap)
    cnt = torch.empty((a.queries, n_splits), dtype=torch.int32, device=dev)
    cs = torch.empty((a.queries, cap), dtype=torch.float32, device=dev)
    ci = torch.empty((a.queries, cap), dtype=torch.int32, device=dev)
    ms_p2 = t_ms(lambda: native.topk_mma(tab, 2, q_ids=q, q_tab=users.table_c, theta=theta, cand_count=cnt,
                                         cand_score=cs, cand_item=ci))
    flops = 2.0 * a.queries * a.items * stride
    item_bytes = math.ceil(a.queries / rows_per_cta(stride)) * a.items * stride * 4.0
    # ---- the pipeline, plain and length-sorted ---------------------------------------------------
    sc, rows = tk.topk(a.K, q_ids=q, q_table=users)
    fb_plain, tiles_plain = tk.last_fallback_rows, list(tk.last_tiles_scored)
    tkp = DeviceTopK(tab, sort_by_length=True)
    scp, rowsp = tkp.topk(a.K, q_ids=q, q_table=users)
    fb_sorted, tiles_sorted = tkp.last_fallback_rows, list(tkp.last_tiles_scored)
    assert torch.equal(sc, scp), "length-sorted table changed the scores"
    # ---- cuBLAS fp32 + torch.topk on the same data -----------------------------------------------
    u = users.pull(q)
    ref_val, ref_idx = torch_topk(u, tab, a.K, a.torch_chunk)
    overlap, max_diff = agreement(rows, ref_idx, sc, ref_val)
    overlap_s, _ = agreement(rowsp, ref_idx, scp, ref_val)
    times = {"plain": [], "sorted": [], "torch": []}
    for _ in range(3):                                   # alternate the variants, keep each one's best
        times["plain"].append(t_ms(lambda: tk.topk(a.K, q_ids=q, q_table=users), iters=5, warm=1))
        times["sorted"].append(t_ms(lambda: tkp.topk(a.K, q_ids=q, q_table=users), iters=5, warm=1))
        times["torch"].append(t_ms(lambda: torch_topk(users.pull(q), tab, a.K, a.torch_chunk), iters=3, warm=1))
    ms_plain, ms_sorted, ms_torch = min(times["plain"]), min(times["sorted"]), min(times["torch"])
    out = {"stride": stride, "kernel": "whole-tile" if stride <= 128 else "k-streamed",
           "rows_per_cta": rows_per_cta(stride), "tiles": n_tiles,
           "pass1_ms": ms_p1, "pass1_tf32_TFLOPs": flops / ms_p1 / 1e9,
           "pass2_ms": ms_p2, "pass2_tf32_TFLOPs": flops / ms_p2 / 1e9,
           "pass1_item_L2_GBps": item_bytes / ms_p1 / 1e6,
           "topk_ms": ms_plain, "tiles_scored": tiles_plain, "fallback_rows": fb_plain,
           "sorted_topk_ms": ms_sorted, "sorted_tiles_scored": tiles_sorted, "sorted_fallback_rows": fb_sorted,
           "torch_fp32_topk_ms": ms_torch, "speedup_vs_torch": ms_torch / ms_plain,
           "sorted_speedup_vs_torch": ms_torch / ms_sorted,
           "torch_id_overlap": overlap, "sorted_torch_id_overlap": overlap_s,
           "torch_max_score_diff": max_diff, "ms_all": times}
    print(json.dumps(out), file=sys.stderr)
    users.close(); items.close()
    del tk, tkp, tile_max, cs, ci
    torch.cuda.empty_cache()
    return out


def w2v_run(a, dev):
    from fps_b200.models.w2v import DeviceSkipGram

    sg = DeviceSkipGram(a.vocab, dim=300, seed=5)
    words = torch.randint(0, a.vocab, (a.words,), device=dev, generator=torch.Generator(device=dev).manual_seed(6))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    sc, ids = sg.most_similar(words, a.w2v_K)            # first call: builds the normalised snapshot
    e1.record(); torch.cuda.synchronize()
    ms_first = e0.elapsed_time(e1)
    ms = t_ms(lambda: sg.most_similar(words, a.w2v_K), iters=5, warm=1)
    w = sg.w_in.local[: a.vocab]                         # one rank: slot == word id
    wn = torch.nn.functional.normalize(w, dim=1)

    def ref():
        qn = wn[words]
        vals, idx = [], []
        for s in range(0, words.numel(), a.torch_chunk):
            cos = qn[s:s + a.torch_chunk] @ wn.T
            cos[torch.arange(cos.shape[0], device=dev), words[s:s + a.torch_chunk]] = float("-inf")
            top = torch.topk(cos, a.w2v_K, dim=1)
            vals.append(top.values); idx.append(top.indices)
        return torch.cat(vals), torch.cat(idx)

    ref_val, ref_idx = ref()
    ms_torch = t_ms(ref, iters=3, warm=1)
    overlap, max_diff = agreement(ids, ref_idx, sc, ref_val)
    out = {"vocab": a.vocab, "dim": 300, "words": a.words, "K": a.w2v_K, "most_similar_ms": ms,
           "most_similar_first_call_ms": ms_first, "torch_fp32_cosine_topk_ms": ms_torch,
           "speedup_vs_torch": ms_torch / ms, "torch_id_overlap": overlap, "torch_max_score_diff": max_diff,
           "self_in_list": int((ids == words[:, None]).any(dim=1).sum())}
    print(json.dumps(out), file=sys.stderr)
    sg.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=2048)
    ap.add_argument("--K", type=int, default=100)
    ap.add_argument("--strides", type=str, default="128,132,256,300,512")
    ap.add_argument("--torch-chunk", type=int, default=256, help="queries per cuBLAS matmul of the baseline")
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--words", type=int, default=1024)
    ap.add_argument("--w2v-K", type=int, default=10)
    ap.add_argument("--out", type=str, default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = False          # the baseline is true fp32
    res = {"queries": a.queries, "items": a.items, "users": a.users, "K": a.K, **gpu_info(), "runs": []}
    for s in [int(x) for x in a.strides.split(",")]:
        res["runs"].append(stride_run(a, s, dev))
    base = next((r for r in res["runs"] if r["stride"] == 128), None)
    if base is not None:                                   # cost of streaming K, per FLOP
        for r in res["runs"]:
            r["pass1_rate_vs_128"] = r["pass1_tf32_TFLOPs"] / base["pass1_tf32_TFLOPs"]
            r["pass2_rate_vs_128"] = r["pass2_tf32_TFLOPs"] / base["pass2_tf32_TFLOPs"]
    if a.words > 0:
        res["most_similar"] = w2v_run(a, dev)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
