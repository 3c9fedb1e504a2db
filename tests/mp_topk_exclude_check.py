"""Multi-rank top-K with per-query exclusion lists, run under torchrun: every rank drops the excluded
global item ids it owns, so the merged lists equal brute force over the gathered items with the
excluded columns masked; and the online learner (no learning, unbounded user memory) gives the same
lists on N ranks as on one."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from tests.mp_util import all_gather_cat, init_dist
    rank, world, dev, shared = init_dist()
    from fps_b200.models.mf.common import Rating
    from fps_b200.models.mf.device_topk import DeviceTopK, DistributedTopK
    from fps_b200.models.mf.topk import psOnlineLearnerAndGenerator
    from fps_b200.store.sharded_table import ShardedTable

    # ---- A: DistributedTopK(exclude=...) == brute force over the gathered items -----------------------
    nu, k, n_local, K, n_q = 5000, 32, 6000, 20, 300
    users = ShardedTable(nu, k, seed=3, init_range=(-1, 1))
    g = torch.Generator(device="cpu").manual_seed(200 + rank)
    local_items = (torch.randn(n_local, k, generator=g) * (0.2 + torch.rand(n_local, 1, generator=g))).to(dev)
    local_ids = torch.arange(n_local, device=dev) * world + rank
    q = torch.randint(0, nu, (n_q,), generator=torch.Generator().manual_seed(7)).to(dev)   # same on all ranks
    # the same TF32 scores the ranks compute, gathered column block by column block (rank-major)
    part = DeviceTopK(local_items).scores(q_ids=q, q_table=users)
    full = all_gather_cat(part.T.contiguous()).T.contiguous()
    gids = all_gather_cat(local_ids)
    # exclusion lists in global ids (identical on every rank): every third query drops its own exact
    # top-3K, the others random ids with duplicates and ids nobody owns
    rng = np.random.RandomState(9)
    top = gids[torch.topk(full, 3 * K, dim=1).indices].cpu().numpy()
    lists = []
    for r in range(n_q):
        if r % 3 == 0:
            lists.append(top[r].tolist())
        else:
            x = rng.randint(-5, world * n_local + 50, rng.randint(0, 3 * K)).tolist()
            lists.append(x + x[:3])
    off = torch.tensor(np.cumsum([0] + [len(x) for x in lists]), device=dev)
    flat = torch.tensor([i for x in lists for i in x], dtype=torch.int64, device=dev)
    col = {int(gid): c for c, gid in enumerate(gids.tolist())}
    masked = full.clone()
    for r, x in enumerate(lists):
        cols = [col[i] for i in x if i in col]
        if cols:
            masked[r, torch.tensor(cols, device=dev)] = float("-inf")
    sc, ids = DistributedTopK(users, local_items, local_ids).topk(q, K, exclude=(off, flat))
    ref = torch.topk(masked, K, dim=1)
    assert torch.equal(sc, ref.values)
    ref_ids = gids[ref.indices]
    same = (ids == ref_ids) | (sc == torch.roll(sc, 1, 1)) | (sc == torch.roll(sc, -1, 1))
    assert same.all()
    for r, x in enumerate(lists):
        assert not (set(ids[r].tolist()) & set(x)), r
    users.barrier()
    users.close()

    # ---- B: learner, learningRate=0, userMemory=-1: N ranks == 1 rank ------------------------------------
    rng = np.random.RandomState(3)
    n_users, n_items = 30, 400
    ratings = [Rating(1, i, 1.0, i) for i in range(0, 120, 3)]               # user 1 rates many items
    ratings += [Rating(int(rng.randint(n_users)), int(rng.randint(n_items)), 1.0, 200 + t) for t in range(150)]
    kw = dict(numFactors=16, K=10, userMemory=-1, learningRate=0.0, rangeMin=-1.0, rangeMax=1.0,
              batch_size=25, plain_residual=True, seed=5, backend="device", numUsers=n_users, numItems=n_items)
    solo_group = [dist.new_group([r]) for r in range(world)][rank]
    multi = psOnlineLearnerAndGenerator(ratings, **kw)
    solo = psOnlineLearnerAndGenerator(ratings, group=solo_group, **kw)
    if rank == 0:
        assert len(multi) == len(solo) == len(ratings)
        for (u, i, ts, a), (u2, i2, ts2, b) in zip(multi, solo):
            assert (u, i, ts) == (u2, i2, ts2) and len(a) == len(b) == 10
            assert [s for s, _ in a] == [s for s, _ in b]
            ties = {s for j, (s, _) in enumerate(b) if any(s == b[t][0] for t in (j - 1, j + 1) if 0 <= t < len(b))}
            assert all(x == y or s in ties for (s, x), (_, y) in zip(a, b))
    dist.barrier()
    solo.model.close()
    dist.barrier()
    multi.model.close()
    if rank == 0:
        print("MP_TOPK_EXCLUDE_CHECK_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
