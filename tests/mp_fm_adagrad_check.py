"""Multi-rank check of the factorization machine with AdaGrad (DESIGN §2.17) in the direct mode, run under torchrun.

The batches of tests/mp_fm_check.py: each rank steps its own stream over features no other rank uses, with a
barrier between steps.  ``bias=False``: the table and the accumulators, read back from both shards, equal the
one-rank fp64 AdaGrad replay of every batch within the replay's bounds.  ``bias=True``: ``w0`` (which keeps the SGD
step) ends at its start value plus the sum of the deltas each rank reports having pushed."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.mp_fm_check import K, NF, STEPS, _batches, _full_table  # noqa: E402


def _full_acc(m, dev):
    """AdaGrad's H of every row, read back from both shards."""
    from fps_b200.ops import native

    ids = torch.arange(NF + 1, device=dev)
    out = torch.empty((NF + 1, m.table.dim), dtype=torch.float32, device=dev)
    native.pull_gather(m._acc_c, ids, out)
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.float64)


def check(rank, world, dev, bias):
    from fps_b200.models.fm import DeviceFactorizationMachine
    from tests import fm_ref

    m = DeviceFactorizationMachine(NF, K, learning_rate=0.05, reg_factors=0.01, init_range=(-0.3, 0.3), bias=bias,
                                   seed=3, optimizer="adagrad")
    m.barrier()
    torch.cuda.synchronize()
    stride = m.table.stride
    W = np.pad(_full_table(m, dev), ((0, 0), (0, stride - 1 - K)))
    H = np.pad(_full_acc(m, dev), ((0, 0), (0, stride - 1 - K)))
    batches = _batches(rank, world)
    t = lambda a: torch.from_numpy(a).to(dev)
    dist.barrier()   # every rank has read the starting table before any rank pushes to it
    for s in range(STEPS):
        rp, cols, vals, labels = batches[rank][s]
        m.step_csr(t(rp), t(cols), t(vals), t(labels))
        torch.cuda.synchronize()
        dist.barrier()
    m.check()
    got, got_h = _full_table(m, dev), _full_acc(m, dev)
    dist.barrier()
    if not bias:
        T, TH = None, None
        for s in range(STEPS):
            for r in range(world):
                rp, cols, vals, labels = batches[r][s]
                res = fm_ref.replay(W, rp, cols, vals, labels, num_features=NF, dim=1 + K, lr=0.05,
                                    reg_factors=0.01, bias=False, tol=T, acc=H, acc_tol=TH)
                W, T, H, TH = res.table, res.tol, res.acc, res.tol_acc
        d = 1 + K
        for name, a, b, tol in (("table", got, W, T), ("acc", got_h, H, TH)):
            err = np.abs(a - b[:, :d])
            assert (err <= fm_ref.MARGIN * tol[:, :d]).all(), (name, (err / np.maximum(tol[:, :d], 1e-30)).max())
        assert got[NF, 0] == 0.0 and (got_h[NF] == 0).all()
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
        print(f"MP_FM_ADAGRAD_CHECK_OK world={world} shared_gpu={int(shared)}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
