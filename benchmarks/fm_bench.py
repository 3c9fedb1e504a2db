"""Factorization-machine step on one GPU: the fused CSR kernel (ops/csrc/fps_fm.cu) against a stock-PyTorch FM on the
same batches.

Shapes: 2^24 hashed features, 39 one-hot entries per example (one per field, Criteo's field count), 2^18 examples
per step, k = 15, 16, 31 and 63 (strides 16, 20, 32 and 64 floats), feature ids drawn per field uniformly or
Zipf-skewed (s = 1.1 over the field's ids, ranks mapped through a fixed permutation).

The PyTorch FM gathers the entries' rows into a leaf tensor, forms the linear term, ``s`` and ``sum x^2 v^2`` with
``embedding_bag``, takes the gradient of the summed logistic loss with autograd, and applies it with ``index_add_``;
``w0`` takes the batch-mean step like the kernel.  Before timing, both run one step on a batch with no shared rows
from the same table and must agree.  Timing: CUDA events, median of ``--rounds`` alternated rounds of ``--steps``
steps each.  The bytes model counts, per entry, one read and one write of the row (the pass-2 re-read is an L2 hit)
plus the entry's id, and per example its offset, label and prediction; its rate is reported beside a ``copy_`` of
1 GiB on the same card.  The card's name and power limit are read in the same run.

    python benchmarks/fm_bench.py [--out profiles/h100_fm_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NF = 1 << 24
FIELDS = 39
BATCH = 1 << 18
KS = (15, 16, 31, 63)
LR = 1e-4   # random labels and Zipf-hot rows: a small rate keeps the timed tables finite


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            "0"], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unknown"
    return name, q


def batches(dist, count, n, seed):
    """``count`` one-hot batches of ``n`` examples: (row_ptr, cols int32, labels) on the GPU."""
    rng = np.random.default_rng(seed)
    per = NF // FIELDS
    perm = rng.permutation(per)
    out = []
    for _ in range(count):
        if dist == "uniform":
            r = rng.integers(0, per, (n, FIELDS))
        else:
            r = perm[np.minimum(rng.zipf(1.1, (n, FIELDS)) - 1, per - 1)]
        cols = (r + np.arange(FIELDS) * per).astype(np.int32).reshape(-1)
        rp = (np.arange(n + 1, dtype=np.int64) * FIELDS)
        labels = rng.integers(0, 2, n).astype(np.float32)
        out.append(tuple(torch.from_numpy(a).cuda() for a in (rp, cols, labels)))
    return out


def torch_step(P, dim, rp, cols, labels):
    """Stock-PyTorch FM step on the [NF + 1, stride] table ``P`` (row NF: w0)."""
    n = labels.numel()
    E = P[cols.long(), :dim].requires_grad_()
    idx = torch.arange(E.shape[0], device=P.device)
    off = rp[:-1]
    lin = F.embedding_bag(idx, E[:, :1], off, mode="sum")[:, 0]
    V = E[:, 1:]
    s = F.embedding_bag(idx, V, off, mode="sum")
    sq = F.embedding_bag(idx, V * V, off, mode="sum")
    w0 = P[NF, 0]
    yhat = w0 + lin + 0.5 * (s * s - sq).sum(1)
    F.binary_cross_entropy_with_logits(yhat, labels, reduction="sum").backward()
    with torch.no_grad():
        g = torch.sigmoid(yhat) - labels
        P.index_add_(0, cols.long(), F.pad(E.grad, (0, P.shape[1] - dim)), alpha=-LR)
        P[NF, 0] -= LR * g.mean()
    return yhat.detach()


def bytes_model(n, nnz, stride):
    return nnz * (2 * stride * 4 + 4) + n * (8 + 4 + 4)


def copy_rate():
    a = torch.empty(1 << 28, dtype=torch.float32, device="cuda")
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(20):
        b.copy_(a)
    e.record()
    torch.cuda.synchronize()
    return 2 * a.numel() * 4 * 20 / (s.elapsed_time(e) * 1e-3) / 1e12


def agree(m, k):
    """One step of each on a batch with no shared rows, from the same table."""
    rng = np.random.default_rng(k)
    n = 4096
    cols = torch.from_numpy(rng.choice(NF, n * FIELDS, replace=False).astype(np.int32)).cuda()
    rp = torch.arange(n + 1, dtype=torch.int64, device="cuda") * FIELDS
    labels = torch.from_numpy(rng.integers(0, 2, n).astype(np.float32)).cuda()
    P = m.table.local.clone()
    ids = torch.cat([cols.long(), torch.tensor([NF], device="cuda")])
    before = P[ids].clone()
    pred_f = m.step_csr(rp, cols, None, labels)
    pred_t = torch_step(P, 1 + k, rp, cols, labels)
    torch.cuda.synchronize()
    dp = (pred_f - pred_t).abs().max().item()
    step_t = P[ids] - before
    dt = ((m.table.local[ids] - before) - step_t).abs().max().item() / step_t.abs().max().item()
    assert dp <= 1e-4 * (1 + pred_t.abs().max().item()) and dt <= 1e-3, (dp, dt)
    return dp, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                  "profiles", "h100_fm_bench.json"))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--torch-steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ks", default=",".join(map(str, KS)))
    ap.add_argument("--batch", type=int, default=BATCH)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fm_bench needs a CUDA device")
    import fps_b200  # noqa: F401
    from fps_b200.models.fm import DeviceFactorizationMachine

    torch.cuda.set_device(0)
    name, power = card()
    copy_tbs = copy_rate()
    data = {d: batches(d, 2, args.batch, 7 + i) for i, d in enumerate(("uniform", "zipf"))}
    rows = []
    for k in map(int, args.ks.split(",")):
        m = DeviceFactorizationMachine(NF, k, learning_rate=LR, init_range=(-0.01, 0.01), seed=1)
        stride = m.table.stride
        dp, dt = agree(m, k)
        for dist, bs in data.items():
            P = m.table.local.clone()
            ev = lambda: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            for rp, cols, labels in bs:          # warm-up of both
                m.step_csr(rp, cols, None, labels)
                torch_step(P, 1 + k, rp, cols, labels)
            torch.cuda.synchronize()
            fused, ref = [], []
            for _ in range(args.rounds):
                s, e = ev()
                s.record()
                for i in range(args.steps):
                    rp, cols, labels = bs[i % len(bs)]
                    m.step_csr(rp, cols, None, labels)
                e.record()
                torch.cuda.synchronize()
                fused.append(s.elapsed_time(e) / args.steps)
                s, e = ev()
                s.record()
                for i in range(args.torch_steps):
                    rp, cols, labels = bs[i % len(bs)]
                    torch_step(P, 1 + k, rp, cols, labels)
                e.record()
                torch.cuda.synchronize()
                ref.append(s.elapsed_time(e) / args.torch_steps)
            del P
            mf, mr = statistics.median(fused), statistics.median(ref)
            n = args.batch
            tbs = bytes_model(n, n * FIELDS, stride) / (mf * 1e-3) / 1e12
            row = dict(k=k, stride=stride, dist=dist, fused_ms=round(mf, 3), torch_ms=round(mr, 3),
                       fused_examples_per_s=round(n / (mf * 1e-3)), torch_examples_per_s=round(n / (mr * 1e-3)),
                       speedup=round(mr / mf, 2), bytes_model_tbs=round(tbs, 3),
                       bytes_model_of_copy=round(tbs / copy_tbs, 3), fused_rounds_ms=[round(x, 3) for x in fused],
                       torch_rounds_ms=[round(x, 3) for x in ref], agree_max_pred_diff=dp, agree_max_step_rel_diff=dt)
            print(json.dumps(row), flush=True)
            rows.append(row)
        finite = bool(torch.isfinite(m.table.local).all().item())
        for row in rows:
            if row["k"] == k:
                row["table_finite"] = finite
        m.close()
        torch.cuda.empty_cache()
    out = dict(card=name, power_limit_and_max_sm_clock=power, features=NF, fields=FIELDS, batch=args.batch,
               steps_per_round=args.steps, torch_steps_per_round=args.torch_steps, rounds=args.rounds,
               copy_tbs=round(copy_tbs, 3), rows=rows,
               note="multi-GPU throughput not measured")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(dict(card=name, power=power, copy_tbs=out["copy_tbs"])))


if __name__ == "__main__":
    main()
