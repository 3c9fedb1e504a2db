"""Field-aware FM step on one GPU: the fused CSR pair kernel (ops/csrc/fps_ffm.cu) against a stock-PyTorch FFM on the
same batches, with the FM kernel at the same k for context.

Shapes: 2^22 hashed features, 39 one-hot entries per example (one per field, Criteo's field count), 2^16 examples
per step, k = 4, 8 and 16 (rows of 4 + 39 kp floats), feature ids drawn per field uniformly or Zipf-skewed (s = 1.1
over the field's ids, ranks mapped through a fixed permutation).

The PyTorch FFM gathers the entries' rows into a leaf tensor, views each example's slabs as ``V[a, f]`` (entry a's
slab for field f), forms the pair term with the field-indexed transpose ``V[a, b] . V[b, a]`` over ``a < b``, takes
the gradient of the summed logistic loss with autograd, and applies it with ``index_add_``; ``w0`` takes the
batch-mean step like the kernel.  Before timing, both run one step on a batch with no shared slabs from the same
table and must agree.  Timing: CUDA events, median of ``--rounds`` alternated rounds.  The bytes model counts, per
pair, a read and a write of both slabs (the pass-2 re-read is an L2 hit), per entry a read and a write of ``w`` plus
its id and field, and per example its offset, label and prediction; its rate is reported beside a ``copy_`` of 1 GiB
on the same card.  The card's name and power limit are read in the same run.

    python benchmarks/ffm_bench.py [--out profiles/h100_ffm_bench.json]
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

NF = 1 << 22
FIELDS = 39
BATCH = 1 << 16
KS = (4, 8, 16)
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
    """``count`` one-hot batches of ``n`` examples: (row_ptr, cols int32, fields int32, labels) on the GPU."""
    rng = np.random.default_rng(seed)
    per = NF // FIELDS
    perm = rng.permutation(per)
    out = []
    fields = torch.arange(FIELDS, dtype=torch.int32).repeat(n).cuda()
    for _ in range(count):
        if dist == "uniform":
            r = rng.integers(0, per, (n, FIELDS))
        else:
            r = perm[np.minimum(rng.zipf(1.1, (n, FIELDS)) - 1, per - 1)]
        cols = (r + np.arange(FIELDS) * per).astype(np.int32).reshape(-1)
        rp = (np.arange(n + 1, dtype=np.int64) * FIELDS)
        labels = rng.integers(0, 2, n).astype(np.float32)
        rp_d, cols_d, labels_d = (torch.from_numpy(a).cuda() for a in (rp, cols, labels))
        out.append((rp_d, cols_d, fields, labels_d))
    return out


def torch_step(P, k, cols, labels):
    """Stock-PyTorch FFM step on the [NF + 1, stride] table ``P`` (row NF: w0); entry a of an example is field a."""
    n = labels.numel()
    kp = 4 * -(-k // 4)
    E = P[cols.long()].requires_grad_()
    w = E[:, 0].view(n, FIELDS)
    V = E[:, 4:].view(n, FIELDS, FIELDS, kp)                 # V[e, a, f]: entry a's slab for field f
    dots = (V * V.transpose(1, 2)).sum(-1)                   # [e, a, b] = V[a, b] . V[b, a]
    pairs = torch.triu(dots, diagonal=1).sum((1, 2))
    w0 = P[NF, 0]
    yhat = w0 + w.sum(1) + pairs
    F.binary_cross_entropy_with_logits(yhat, labels, reduction="sum").backward()
    with torch.no_grad():
        g = torch.sigmoid(yhat) - labels
        P.index_add_(0, cols.long(), E.grad, alpha=-LR)
        P[NF, 0] -= LR * g.mean()
    return yhat.detach()


def bytes_model(n, nnz, pairs, kp):
    return pairs * 4 * kp * 4 + nnz * (4 + 4 + 4 + 4) + n * (8 + 4 + 4)


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
    """One step of each on a batch with no shared slabs (distinct features), from the same table."""
    rng = np.random.default_rng(k)
    n = 1024
    cols = torch.from_numpy(rng.choice(NF, n * FIELDS, replace=False).astype(np.int32)).cuda()
    fields = torch.arange(FIELDS, dtype=torch.int32, device="cuda").repeat(n)
    rp = torch.arange(n + 1, dtype=torch.int64, device="cuda") * FIELDS
    labels = torch.from_numpy(rng.integers(0, 2, n).astype(np.float32)).cuda()
    P = m.table.local.clone()
    ids = torch.cat([cols.long(), torch.tensor([NF], device="cuda")])
    before = P[ids].clone()
    pred_f = m.step_csr(rp, cols, fields, None, labels)
    pred_t = torch_step(P, k, cols, labels)
    torch.cuda.synchronize()
    dp = (pred_f - pred_t).abs().max().item()
    step_t = P[ids] - before
    dt = ((m.table.local[ids] - before) - step_t).abs().max().item() / step_t.abs().max().item()
    assert dp <= 1e-4 * (1 + pred_t.abs().max().item()) and dt <= 1e-3, (dp, dt)
    del P
    return dp, dt


def timed(fn, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(steps):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                  "profiles", "h100_ffm_bench.json"))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--torch-steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ks", default=",".join(map(str, KS)))
    ap.add_argument("--batch", type=int, default=BATCH)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ffm_bench needs a CUDA device")
    import fps_b200  # noqa: F401
    from fps_b200.models.fm import DeviceFactorizationMachine, DeviceFieldAwareFM

    torch.cuda.set_device(0)
    name, power = card()
    copy_tbs = copy_rate()
    data = {d: batches(d, 2, args.batch, 7 + i) for i, d in enumerate(("uniform", "zipf"))}
    n = args.batch
    pairs = n * FIELDS * (FIELDS - 1) // 2
    rows = []
    for k in map(int, args.ks.split(",")):
        kp = 4 * -(-k // 4)
        m = DeviceFieldAwareFM(NF, FIELDS, k, learning_rate=LR, init_range=(-0.01, 0.01), seed=1)
        fm = DeviceFactorizationMachine(NF, k, learning_rate=LR, init_range=(-0.01, 0.01), seed=1)
        dp, dt = agree(m, k)
        for dist, bs in data.items():
            P = m.table.local.clone()
            step_f = lambda i: m.step_csr(bs[i % 2][0], bs[i % 2][1], bs[i % 2][2], None, bs[i % 2][3])
            step_t = lambda i: torch_step(P, k, bs[i % 2][1], bs[i % 2][3])
            step_fm = lambda i: fm.step_csr(bs[i % 2][0], bs[i % 2][1], None, bs[i % 2][3])
            for i in range(2):                      # warm-up of all three
                step_f(i), step_t(i), step_fm(i)
            torch.cuda.synchronize()
            fused, ref, fmk = [], [], []
            for _ in range(args.rounds):
                fused.append(timed(step_f, args.steps))
                ref.append(timed(step_t, args.torch_steps))
                fmk.append(timed(step_fm, args.steps))
            del P
            mf, mr, mk = (statistics.median(x) for x in (fused, ref, fmk))
            tbs = bytes_model(n, n * FIELDS, pairs, kp) / (mf * 1e-3) / 1e12
            row = dict(k=k, stride=m.table.stride, dist=dist, fused_ms=round(mf, 3), torch_ms=round(mr, 3),
                       fm_kernel_ms=round(mk, 3), fused_examples_per_s=round(n / (mf * 1e-3)),
                       torch_examples_per_s=round(n / (mr * 1e-3)), speedup=round(mr / mf, 2),
                       bytes_model_tbs=round(tbs, 3), bytes_model_of_copy=round(tbs / copy_tbs, 3),
                       fused_rounds_ms=[round(x, 3) for x in fused], torch_rounds_ms=[round(x, 3) for x in ref],
                       fm_kernel_rounds_ms=[round(x, 3) for x in fmk], agree_max_pred_diff=dp,
                       agree_max_step_rel_diff=dt)
            print(json.dumps(row), flush=True)
            rows.append(row)
        finite = bool(torch.isfinite(m.table.local).all().item())
        for row in rows:
            if row["k"] == k:
                row["table_finite"] = finite
        m.close()
        fm.close()
        torch.cuda.empty_cache()
    out = dict(card=name, power_limit_and_max_sm_clock=power, features=NF, fields=FIELDS, batch=args.batch,
               pairs_per_step=pairs, steps_per_round=args.steps, torch_steps_per_round=args.torch_steps,
               rounds=args.rounds, copy_tbs=round(copy_tbs, 3), rows=rows,
               note="multi-GPU throughput not measured")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(dict(card=name, power=power, copy_tbs=out["copy_tbs"])))


if __name__ == "__main__":
    main()
