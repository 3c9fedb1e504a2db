"""Multi-rank check of the WARP loss, run under torchrun: the lowrank_implicit set of tests/bpr_quality.py split by
user over the ranks, trained with candidates sampled in the kernel, in the direct mode (item rows read from and
pushed to their owners) and in the default replica mode (local item replicas).  Each run stays finite and beats an
untrained model on held-out AUC and recall@10.
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def train(rank, world, dev, lr, item_cache):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from tests import bpr_quality as Q
    from tests import warp_quality as W
    from tests.mp_util import all_gather_cat

    tu, ti, eu, ei = Q.data()
    mine = (tu % world) == rank
    u, i = tu[mine].int().to(dev), ti[mine].int().to(dev)
    batch = 128 // world
    n_steps = max(-(-int(((tu % world) == r).sum()) // batch) for r in range(world))
    m = DeviceOnlineMF(Q.NUM_USERS, Q.NUM_ITEMS, Q.K, range_min=-Q.INIT, range_max=Q.INIT, learning_rate=lr,
                       negative_sample_rate=W.T, seed=1, loss="warp", regularization=Q.REG, margin=W.MARGIN,
                       item_cache=item_cache)
    for _ in range(Q.EPOCHS):
        for s in range(n_steps):           # every rank takes part in every exchange round
            a = s * batch
            m.step(u[a:a + batch], i[a:a + batch], torch.ones(u[a:a + batch].numel(), device=dev))
    m.refresh()
    m.check_finite()
    V = m.items.pull(torch.arange(Q.NUM_ITEMS, device=dev))[:, :Q.K].clone()
    uid, uvec = m.user_vectors()
    uid, uvec = all_gather_cat(uid), all_gather_cat(uvec)
    U = torch.zeros(Q.NUM_USERS, Q.K, device=dev)
    U[uid] = uvec
    stats = all_gather_cat(m.stats[None]).sum(0).cpu()
    m.barrier()
    m.close()
    assert torch.isfinite(U).all() and torch.isfinite(V).all()
    return Q.metrics(U, V, (tu, ti), (eu, ei)), stats


def main():
    from tests.mp_util import init_dist
    from tests import warp_quality as W

    rank, world, dev, shared = init_dist()
    res = {}
    for mode, cache in (("direct", False), ("replica", True)):
        (auc, recall), stats = train(rank, world, dev, W.LR, cache)
        (auc0, recall0), _ = train(rank, world, dev, 0.0, cache)
        res[mode] = (round(auc, 4), round(recall, 4), round(auc0, 4))
        assert stats[3].item() > 0 and stats[2].item() >= stats[3].item(), stats
        assert auc > auc0 + 0.1 and recall > recall0 + 0.03, (mode, auc, recall, auc0, recall0)
    dist.barrier()
    if rank == 0:
        print(f"MP_WARP_CHECK_OK world={world} shared_gpu={int(shared)} (auc, recall, untrained auc)={res}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
