"""Multi-rank check of the factorization machine in the direct mode, run under torchrun.

``bias=False``: each rank steps its own stream of batches over features no other rank uses (no feature shared inside
a batch either), with a barrier between steps; the table, read back from both shards, equals the one-rank fp64
replay of every batch within the replay's bound.  ``bias=True``: ``w0`` ends at its start value plus the sum of the
deltas each rank reports having pushed."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NF, K, STEPS, N = 4096, 12, 3, 128


def _batches(rank, world):
    """Per-rank batches over the features f with f % world == rank, every feature used once over all steps."""
    rng = np.random.default_rng(99)
    feats = rng.permutation(np.arange(1, NF - 1))
    out = []
    for r in range(world):
        mine = feats[feats % world == r]
        pos, lst = 0, []
        for s in range(STEPS):
            sizes = rng.integers(0, 4, N)
            rp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
            cols = mine[pos:pos + rp[-1]].astype(np.int64)
            pos += rp[-1]
            vals = rng.normal(0, 1, rp[-1]).astype(np.float32)
            labels = rng.integers(0, 2, N).astype(np.float32)
            lst.append((rp, cols, vals, labels))
        out.append(lst)
    return out


def _full_table(m, dev):
    ids = torch.arange(NF + 1, device=dev)
    return m.table.pull(ids).cpu().numpy().astype(np.float64)


def check(rank, world, dev, bias):
    from fps_b200.models.fm import DeviceFactorizationMachine
    from tests import fm_ref

    m = DeviceFactorizationMachine(NF, K, learning_rate=0.05, reg_factors=0.01, init_range=(-0.3, 0.3), bias=bias,
                                   seed=3)
    m.barrier()
    torch.cuda.synchronize()
    W = _full_table(m, dev)
    stride = m.table.stride
    W = np.pad(W, ((0, 0), (0, stride - W.shape[1])))
    batches = _batches(rank, world)
    t = lambda a: torch.from_numpy(a).to(dev)
    dist.barrier()   # every rank has read the starting table before any rank pushes to it
    for s in range(STEPS):
        rp, cols, vals, labels = batches[rank][s]
        m.step_csr(t(rp), t(cols), t(vals), t(labels))
        torch.cuda.synchronize()
        dist.barrier()
    m.check()
    got = _full_table(m, dev)
    dist.barrier()
    if not bias:
        T = None
        for s in range(STEPS):
            for r in range(world):
                rp, cols, vals, labels = batches[r][s]
                res = fm_ref.replay(W, rp, cols, vals, labels, num_features=NF, dim=1 + K, lr=0.05, reg_factors=0.01,
                                    bias=False, tol=T)
                W, T = res.table, res.tol
        err = np.abs(got - W[:, : 1 + K])
        assert (err <= fm_ref.MARGIN * T[:, : 1 + K]).all(), (err / np.maximum(T[:, : 1 + K], 1e-30)).max()
        assert got[NF, 0] == 0.0
    else:
        parts = [None] * world
        dist.all_gather_object(parts, m.bias_pushed)
        total = float(sum(parts))
        assert total != 0.0
        assert abs(got[NF, 0] - (W[NF, 0] + total)) <= 1e-6 * (1 + abs(total)), (got[NF, 0], W[NF, 0], total)
    dist.barrier()
    m.close()


def main():
    from tests.mp_util import init_dist
    rank, world, dev, shared = init_dist()
    for bias in (False, True):
        check(rank, world, dev, bias)
    dist.barrier()
    if rank == 0:
        print(f"MP_FM_CHECK_OK world={world} shared_gpu={int(shared)}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
