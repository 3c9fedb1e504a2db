"""CPU model of the replica (sender-side combining) mode's staleness: N workers train their own replica of the
item table with mini-batched SGD and merge `replica - base` deltas every `sync_every` steps; held-out RMSE against
ONE worker on the same stream and update budget.  Pure torch on the host -- a quick way to explore the
quality side of the `sync_every` knob without a GPU.

    python benchmarks/replica_staleness_sim.py [--users 4096 --items 8192 --k 16 --lr 0.05 --updates 5242880]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fps_b200.utils.synthetic import lowrank_ratings  # noqa: E402


def run(nu, ni, k, lr, init, updates, batch, world, sync_every, mb=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    U = (torch.rand(nu, k, generator=g) * 2 - 1) * init
    V = (torch.rand(ni, k, generator=g) * 2 - 1) * init
    reps = [V.clone() for _ in range(world)]
    bases = [V.clone() for _ in range(world)]
    hu = torch.randint(0, nu, (200000,), generator=g)
    hi = torch.randint(0, ni, (200000,), generator=g)
    hr = lowrank_ratings(hu, hi)
    steps = updates // (batch * world)
    for s in range(steps):
        for w in range(world):
            u = torch.randint(0, nu // world, (batch,), generator=g) * world + w
            i = torch.randint(0, ni, (batch,), generator=g)
            r = lowrank_ratings(u, i)
            Vw = reps[w] if sync_every else V
            for a in range(0, batch, mb):
                uu, ii, rr = u[a:a + mb], i[a:a + mb], r[a:a + mb]
                pu, pv = U[uu], Vw[ii]
                e = (rr - (pu * pv).sum(1))[:, None] * lr
                U.index_add_(0, uu, e * pv)
                Vw.index_add_(0, ii, e * pu)
        if sync_every and (s + 1) % sync_every == 0:
            for w in range(world):
                V += reps[w] - bases[w]
            for w in range(world):
                reps[w] = V.clone()
                bases[w] = V.clone()
    if sync_every:
        for w in range(world):
            V += reps[w] - bases[w]
    return float(((hr - (U[hu] * V[hi]).sum(1)) ** 2).mean().sqrt())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--users", type=int, default=4096)
    p.add_argument("--items", type=int, default=8192)
    p.add_argument("--k", type=int, default=16)
    p.add_argument("--lr", type=float, default=0.05)
    p.add_argument("--init", type=float, default=0.3)
    p.add_argument("--updates", type=int, default=160 * 32768)
    p.add_argument("--batch", type=int, default=32768)
    a = p.parse_args()
    out = {"config": vars(a), "rmse": {}}
    single = run(a.users, a.items, a.k, a.lr, a.init, a.updates, a.batch, 1, 0)
    out["rmse"]["single_worker"] = single
    for world in (2, 4, 8):
        for se in (1, 2, 4, 8):
            r = run(a.users, a.items, a.k, a.lr, a.init, a.updates, a.batch, world, se)
            out["rmse"][f"N{world}_sync{se}"] = r
            out["rmse"][f"N{world}_sync{se}_vs_single"] = r / single
    print(json.dumps(out))


if __name__ == "__main__":
    main()
