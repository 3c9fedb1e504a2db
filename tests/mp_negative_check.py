"""Multi-rank check of ``negative_sampling="seen"``, run under torchrun: every rank trains on its own stream
(its users, and items from a range of its own) in the default replica mode; each rank's registry then holds
exactly its own stream's items in first-occurrence order, and the pointwise and BPR models stay finite."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(rank, world, dev, loss):
    from fps_b200.models.mf.device import DeviceOnlineMF

    nu, ni, k = 4000, 8000, 16
    m = DeviceOnlineMF(nu, ni, k, learning_rate=0.05, negative_sample_rate=2, user_memory=16,
                       negative_sampling="seen", loss=loss, seed=2)
    assert m.item_cache == (world > 1)
    g = torch.Generator().manual_seed(100 + rank)
    span = ni // world
    stream = []
    for n in (3000, 500, 4000):
        users = torch.randint(0, nu // world, (n,), generator=g) * world + rank
        items = torch.randint(0, span // 2, (n,), generator=g) + rank * span
        stream.append(items)
        m.step(users.int().to(dev), items.int().to(dev), torch.rand(n, generator=g).to(dev) + 0.5)
    m.barrier()
    m.check_finite()
    items = torch.cat(stream).numpy()
    _, idx = np.unique(items, return_index=True)
    np.testing.assert_array_equal(m.seen_items().cpu().numpy(), items[np.sort(idx)])
    assert float(m.stats[1].item()) > 7500
    m.close()


def main():
    from tests.mp_util import init_dist
    rank, world, dev, shared = init_dist()
    for loss in ("pointwise", "bpr"):
        run(rank, world, dev, loss)
        dist.barrier()
    if rank == 0:
        print(f"MP_NEGATIVE_CHECK_OK world={world} shared_gpu={int(shared)}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
