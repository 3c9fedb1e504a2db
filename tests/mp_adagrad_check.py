"""Multi-rank check of row-wise AdaGrad in the direct mode, run under torchrun: a conflict-free batch (distinct
users, distinct items) split by user over the ranks, item rows and item accumulators read from and reduced
into peer shards, equals the one-rank run of the whole batch -- for the pointwise and the BPR loss.  Rows
and accumulators are compared at the tolerances of mp_bpr_check.py (the pushes of different ranks land in
any order)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _item_acc(model, ni, dev):
    from tests.mp_util import all_gather_cat

    ids, acc = model._item_acc.dump_local()
    ids, acc = all_gather_cat(ids), all_gather_cat(acc)
    full = torch.zeros(ni, device=dev)
    full[ids.to(dev)] = acc.to(dev)
    return full


def direct_equals_solo(rank, world, dev, solo_group, loss):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from tests.mp_util import all_gather_cat

    nu, ni, k, b = 4096, 16384, 32, 2048
    g = torch.Generator().manual_seed(23)
    users = torch.randperm(nu, generator=g)[:b].to(dev)
    ij = torch.randperm(ni, generator=g)[:2 * b].to(dev)
    items, negs = ij[:b], ij[b:]
    ratings = torch.rand(b, generator=g).to(dev) + 0.5
    kw = dict(range_min=-0.5, range_max=0.5, learning_rate=0.05, seed=4, optimizer="adagrad", step_window=0)
    if loss == "bpr":
        kw.update(loss="bpr", regularization=0.01)

    def step(m, sel):
        extra = dict(negatives=negs[sel].int()[:, None].contiguous()) if loss == "bpr" else {}
        m.step(users[sel].int(), items[sel].int(), ratings[sel], **extra)

    multi = DeviceOnlineMF(nu, ni, k, item_cache=False, **kw)
    step(multi, (users % world) == rank)
    multi.barrier()
    got_items = multi.items.pull(torch.arange(ni, device=dev))[:, :k].clone()
    got_acc = _item_acc(multi, ni, dev)
    uid, uvec = multi.user_vectors()
    uacc = multi.accumulators[0][uid // world]
    uid, uvec, uacc = all_gather_cat(uid), all_gather_cat(uvec), all_gather_cat(uacc)
    multi.barrier()
    solo = DeviceOnlineMF(nu, ni, k, group=solo_group, **kw)
    if rank == 0:
        step(solo, torch.ones(b, dtype=torch.bool, device=dev))
        torch.cuda.synchronize()
        s_uacc, s_iacc = solo.accumulators
        assert (got_acc[items] > 0).all()
        torch.testing.assert_close(got_items, solo.items.local[:ni, :k], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(got_acc, s_iacc[:ni], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(uvec.to(dev), solo.users[uid.to(dev), :k], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(uacc.to(dev), s_uacc[uid.to(dev)], rtol=1e-5, atol=1e-6)
    solo.close()
    multi.close()


def main():
    from tests.mp_util import init_dist
    rank, world, dev, shared = init_dist()
    solo_groups = [dist.new_group([r]) for r in range(world)]
    for loss in ("pointwise", "bpr"):
        direct_equals_solo(rank, world, dev, solo_groups[rank], loss)
    dist.barrier()
    if rank == 0:
        print(f"MP_ADAGRAD_CHECK_OK world={world} shared_gpu={int(shared)}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
