"""Multi-rank checks of the pairwise (BPR) loss, run under torchrun:

A. direct mode -- a conflict-free batch (distinct users, all positives and negatives distinct) split by
   user over the ranks, items pulled from and pushed to peer shards: the model equals the one-rank run of
   the whole batch (up to fp32 rounding: the dot products are summed in the same order, but the
   one-sided pushes of different ranks land in any order).
B. replica mode -- the same lowrank_implicit set trained with the same update budget by one worker and by
   N workers with local item replicas: held-out AUC within 2 %.
C. the online learner + generator with loss="bpr" on N ranks.
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def direct_equals_solo(rank, world, dev, solo_group):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from tests.mp_util import all_gather_cat

    nu, ni, k, b = 4096, 16384, 32, 2048
    g = torch.Generator().manual_seed(21)
    users = torch.randperm(nu, generator=g)[:b].to(dev)
    ij = torch.randperm(ni, generator=g)[:2 * b].to(dev)
    items, negs = ij[:b], ij[b:]
    ratings = torch.ones(b, device=dev)
    kw = dict(range_min=-0.5, range_max=0.5, learning_rate=0.05, seed=4, loss="bpr", regularization=0.01)
    multi = DeviceOnlineMF(nu, ni, k, item_cache=False, **kw)
    mine = (users % world) == rank
    multi.step(users[mine].int(), items[mine].int(), ratings[mine], negatives=negs[mine].int()[:, None].contiguous())
    multi.barrier()
    got_items = multi.items.pull(torch.arange(ni, device=dev))[:, :k].clone()
    uid, uvec = multi.user_vectors()
    uid, uvec = all_gather_cat(uid), all_gather_cat(uvec)
    stats = all_gather_cat(multi.stats[None]).sum(0)
    multi.barrier()
    solo = DeviceOnlineMF(nu, ni, k, group=solo_group, **kw)
    if rank == 0:
        solo.step(users.int(), items.int(), ratings, negatives=negs.int()[:, None].contiguous())
        torch.cuda.synchronize()
        torch.testing.assert_close(got_items, solo.items.local[:ni, :k], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(uvec, solo.users[uid, :k], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(stats, solo.stats, rtol=1e-4, atol=1.0)
    solo.close()
    multi.close()


def replica_auc(rank, world, dev, solo_group):
    from fps_b200.models.mf.device import DeviceOnlineMF
    from tests import bpr_quality as Q
    from tests.mp_util import all_gather_cat

    tu, ti, eu, ei = Q.data()
    kw = dict(range_min=-Q.INIT, range_max=Q.INIT, learning_rate=Q.LR, negative_sample_rate=1, seed=1,
              loss="bpr", regularization=Q.REG)
    parts = [((tu % world) == r) for r in range(world)]
    batch = 128 // world

    def batches(r):
        u, i = tu[parts[r]].int().to(dev), ti[parts[r]].int().to(dev)
        return [(u[a:a + batch], i[a:a + batch], torch.ones(min(batch, u.numel() - a), device=dev))
                for a in range(0, u.numel(), batch)]

    mine = batches(rank)
    n_steps = max(len(batches(r)) for r in range(world))
    m = DeviceOnlineMF(Q.NUM_USERS, Q.NUM_ITEMS, Q.K, item_cache=True, sync_every=2, **kw)
    for _ in range(Q.EPOCHS):
        for s in range(n_steps):
            if s < len(mine):
                m.step(*mine[s])
            else:                       # every rank takes part in every exchange round
                m.step(*(t[:0] for t in mine[0]))
    m.refresh()
    m.check_finite()
    V = m.items.pull(torch.arange(Q.NUM_ITEMS, device=dev))[:, :Q.K].clone()
    uid, uvec = m.user_vectors()
    uid, uvec = all_gather_cat(uid), all_gather_cat(uvec)
    U = torch.zeros(Q.NUM_USERS, Q.K, device=dev)
    U[uid] = uvec
    m.barrier()
    solo = DeviceOnlineMF(Q.NUM_USERS, Q.NUM_ITEMS, Q.K, group=solo_group, **kw)
    result = None
    if rank == 0:
        every = [batches(r) for r in range(world)]
        for _ in range(Q.EPOCHS):
            for s in range(n_steps):
                for r in range(world):
                    if s < len(every[r]):
                        solo.step(*every[r][s])
        torch.cuda.synchronize()
        auc_solo, _ = Q.metrics(solo.users[:, :Q.K], solo.items.local[:Q.NUM_ITEMS, :Q.K], (tu, ti), (eu, ei))
        auc_rep, _ = Q.metrics(U, V, (tu, ti), (eu, ei))
        result = (auc_rep, auc_solo)
        assert auc_solo >= Q.AUC_GATE, result
        assert auc_rep >= 0.98 * auc_solo, result
    solo.close()
    m.close()
    return result


def learner(rank, world, dev):
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.device_api import ps_online_learner_and_generator_device
    from tests import bpr_quality as Q

    tu, ti, _, _ = Q.data()
    recs = [Rating(int(u), int(i), 1.0, t) for t, (u, i) in enumerate(zip(tu[:3000].tolist(), ti[:3000].tolist()))]
    out = ps_online_learner_and_generator_device(recs, numFactors=16, rangeMin=-0.1, rangeMax=0.1, learningRate=0.2,
                                                 negativeSampleRate=2, K=10, batch_size=256, seed=2, loss="bpr",
                                                 regularization=0.01)
    if rank == 0:
        assert len(out) == len(recs)
        assert all(len(top) == 10 for _, _, _, top in out)
    assert torch.isfinite(out.items).all()
    out.model.close()


def main():
    from tests.mp_util import init_dist
    rank, world, dev, shared = init_dist()
    solo_groups = [dist.new_group([r]) for r in range(world)]
    direct_equals_solo(rank, world, dev, solo_groups[rank])
    q = replica_auc(rank, world, dev, solo_groups[rank])
    learner(rank, world, dev)
    dist.barrier()
    if rank == 0:
        print(f"MP_BPR_CHECK_OK world={world} shared_gpu={int(shared)} auc(replica, solo)={q}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
