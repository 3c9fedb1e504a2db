"""Multi-rank ``DeviceSkipGram.train_tokens(cbow=True)``, run under torchrun, in direct mode (rows read and pushed on
their owners) and in replica mode (local replicas, deltas exchanged in the background): every rank trains its own
part of a topic corpus, the counters add up, the tables stay finite and every rank reads the same rows after a
barrier."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from tests.mp_util import all_gather_cat, init_dist
    rank, world, dev, shared = init_dist()
    from fps_b200.models.w2v import DeviceSkipGram
    from fps_b200.utils.synthetic import topic_corpus

    vocab, topics = 4000, 40
    tok = topic_corpus(vocab, topics, 10, 8000, seed=1)                # the same corpus on every rank
    counts = np.bincount(tok[tok >= 0].numpy(), minlength=vocab).astype(np.float64)
    part = tok.view(-1, 11)[rank::world].reshape(-1).to(dev)          # every rank trains its own sentences
    for replica in (False, True):
        m = DeviceSkipGram(vocab, 128, learning_rate=0.05, negative=5, seed=7, replica_cache=replica,
                           word_counts=counts, noise_counts=counts)
        before_in = m.w_in.pull(torch.arange(vocab, device=dev)).clone()
        m.fit_tokens(part, epochs=2, batch_tokens=16384, cbow=True)
        m.barrier()
        m.check_finite()
        ts, st = m.token_stats.cpu(), m.stats.cpu()
        assert ts[0].item() == 2 * part.numel() and 0 < ts[1].item() < ts[0].item() and ts[2].item() > 0, ts
        assert 0 < st[1].item() <= ts[1].item() * 6, (st, ts)           # at most 1 + negative targets per center
        w = m.w_in.pull(torch.arange(vocab, device=dev))
        v = m.w_out.pull(torch.arange(vocab, device=dev))
        assert torch.isfinite(w).all() and (w != before_in).any() and torch.isfinite(v).all() and v.any()
        rows = all_gather_cat(torch.cat([w, v], 1)[None])
        assert all(torch.equal(rows[0], rows[r]) for r in range(world)), replica
        dist.barrier()
        m.close()
        dist.barrier()
    if rank == 0:
        print("MP_W2V_CBOW_CHECK_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
