"""Multi-rank ``DeviceSkipGram.most_similar``, run under torchrun: after training on every rank (replica
deltas in flight), the collective query over the W_in shards gives the same lists as a one-rank model
loaded with the same weights."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from tests.mp_util import init_dist
    rank, world, dev, shared = init_dist()
    from fps_b200.models.w2v import DeviceSkipGram

    vocab, dim, K = 20000, 300, 10
    multi = DeviceSkipGram(vocab, dim=dim, learning_rate=0.05, negative=5, seed=11)
    g = torch.Generator(device=dev).manual_seed(100 + rank)           # every rank trains its own pairs
    for _ in range(10):
        c = torch.randint(0, vocab, (8192,), generator=g, device=dev, dtype=torch.int32)
        off = torch.randint(1, 4, (8192,), generator=g, device=dev, dtype=torch.int32)
        multi.step(c, (c + off) % vocab)
    words = torch.randint(0, vocab, (257,), generator=torch.Generator().manual_seed(7)).to(dev)  # same on all ranks
    sc, ids = multi.most_similar(words, K)
    assert sc.shape == ids.shape == (257, K)
    assert (ids != words[:, None]).all() and (ids >= 0).all()
    all_ids = torch.arange(vocab, device=dev)
    w = multi.w_in.pull(all_ids)                                       # deltas were flushed by the query

    solo_group = [dist.new_group([r]) for r in range(world)][rank]
    solo = DeviceSkipGram(vocab, dim=dim, group=solo_group, seed=11)
    solo.w_in.load(all_ids, w)
    s_sc, s_ids = solo.most_similar(words, K)
    # same rows, same TF32 products: equal lists up to the order of near-equal scores
    torch.testing.assert_close(sc, s_sc, rtol=0, atol=1e-5)
    near = (s_sc - torch.roll(s_sc, 1, 1)).abs() < 1e-5
    near |= (s_sc - torch.roll(s_sc, -1, 1)).abs() < 1e-5
    assert ((ids == s_ids) | near).all()
    dist.barrier()
    solo.close()
    dist.barrier()
    multi.close()
    if rank == 0:
        print("MP_W2V_NEIGHBOURS_CHECK_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
