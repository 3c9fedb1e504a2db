"""AdaGrad against SGD for the factorization machines (DESIGN §2.17), on one GPU, at the shapes of
benchmarks/fm_bench.py (2^24 features, 39 one-hot fields, 2^18 examples per step, k 15-63) and
benchmarks/ffm_bench.py (2^22 features, 39 fields, 2^16 examples per step, k 4-16), uniform and Zipf ids.

For each shape an SGD model and an AdaGrad model of the same table take steps on the same batches; their rounds
alternate, and each reports the median of ``--rounds`` rounds.  The bytes model is the SGD one of those benchmarks
with the accumulator traffic added: AdaGrad reads and reduces one ``H`` row per FM entry and two ``H`` slabs (and
one ``H_w``) per FFM pair, so it moves about twice the row bytes.  The card's name and power limit are read in the
same run.  Results go to ``--out`` (default profiles/h100_fm_adagrad_bench.json)."""
import argparse
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import ffm_bench  # noqa: E402
import fm_bench  # noqa: E402


def fm_bytes(n, nnz, stride, ada):
    return nnz * ((4 if ada else 2) * stride * 4 + 4) + n * (8 + 4 + 4)


def ffm_bytes(n, nnz, pairs, kp, ada):
    return pairs * (8 if ada else 4) * kp * 4 + nnz * (4 + 4 + 4 + 4 + (8 if ada else 0)) + n * (8 + 4 + 4)


def run(kind, ks, batch, steps, rounds, copy_tbs):
    from fps_b200.models.fm import DeviceFactorizationMachine, DeviceFieldAwareFM

    mod = fm_bench if kind == "fm" else ffm_bench
    data = {d: mod.batches(d, 2, batch, 7 + i) for i, d in enumerate(("uniform", "zipf"))}
    fields = mod.FIELDS
    rows = []
    for k in ks:
        models = {}
        for opt in ("sgd", "adagrad"):
            if kind == "fm":
                models[opt] = DeviceFactorizationMachine(mod.NF, k, learning_rate=mod.LR, init_range=(-0.01, 0.01),
                                                         seed=1, optimizer=opt)
            else:
                models[opt] = DeviceFieldAwareFM(mod.NF, fields, k, learning_rate=mod.LR, init_range=(-0.01, 0.01),
                                                 seed=1, optimizer=opt)
        for dist, bs in data.items():
            def stepper(m):
                if kind == "fm":
                    return lambda i: m.step_csr(bs[i % 2][0], bs[i % 2][1], None, bs[i % 2][2])
                return lambda i: m.step_csr(bs[i % 2][0], bs[i % 2][1], bs[i % 2][2], None, bs[i % 2][3])
            fns = {opt: stepper(m) for opt, m in models.items()}
            for i in range(2):
                for fn in fns.values():
                    fn(i)
            torch.cuda.synchronize()
            ms = {opt: [] for opt in fns}
            for _ in range(rounds):
                for opt, fn in fns.items():
                    ms[opt].append(ffm_bench.timed(fn, steps))
            med = {opt: statistics.median(v) for opt, v in ms.items()}
            n, nnz = batch, batch * fields
            row = dict(model=kind, k=k, stride=models["sgd"].table.stride, dist=dist)
            for opt in fns:
                if kind == "fm":
                    b = fm_bytes(n, nnz, models[opt].table.stride, opt == "adagrad")
                else:
                    b = ffm_bytes(n, nnz, n * fields * (fields - 1) // 2, 4 * -(-k // 4), opt == "adagrad")
                tbs = b / (med[opt] * 1e-3) / 1e12
                row.update({f"{opt}_ms": round(med[opt], 3), f"{opt}_rounds_ms": [round(x, 3) for x in ms[opt]],
                            f"{opt}_bytes_model_tbs": round(tbs, 3), f"{opt}_bytes_model_of_copy": round(tbs / copy_tbs, 3)})
            row["adagrad_over_sgd"] = round(med["adagrad"] / med["sgd"], 3)
            print(json.dumps(row), flush=True)
            rows.append(row)
        for opt, m in models.items():
            finite = bool(torch.isfinite(m.table.local).all().item())
            for row in rows:
                if row["model"] == kind and row["k"] == k:
                    row[f"{opt}_table_finite"] = finite
            m.close()
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(HERE), "profiles", "h100_fm_adagrad_bench.json"))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--fm-ks", default=",".join(map(str, fm_bench.KS)))
    ap.add_argument("--ffm-ks", default=",".join(map(str, ffm_bench.KS)))
    ap.add_argument("--fm-batch", type=int, default=fm_bench.BATCH)
    ap.add_argument("--ffm-batch", type=int, default=ffm_bench.BATCH)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fm_adagrad_bench needs a GPU")
    import fps_b200  # noqa: F401

    torch.cuda.set_device(0)
    name, power = ffm_bench.card()
    copy_tbs = ffm_bench.copy_rate()
    rows = run("fm", [int(k) for k in args.fm_ks.split(",") if k], args.fm_batch, args.steps, args.rounds, copy_tbs)
    rows += run("ffm", [int(k) for k in args.ffm_ks.split(",") if k], args.ffm_batch, args.steps, args.rounds,
                copy_tbs)
    out = dict(card=name, power_limit_and_max_sm_clock=power, fm_features=fm_bench.NF, ffm_features=ffm_bench.NF,
               fields=fm_bench.FIELDS, fm_batch=args.fm_batch, ffm_batch=args.ffm_batch, steps_per_round=args.steps,
               rounds=args.rounds, copy_tbs=round(copy_tbs, 3), rows=rows, note="multi-GPU throughput not measured")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(dict(card=name, power=power, copy_tbs=out["copy_tbs"])))


if __name__ == "__main__":
    main()
