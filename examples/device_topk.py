"""Top-K serving on an H100: user vectors on the parameter server, wgmma scoring against local items."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fps_b200.models.mf.device_topk import DeviceTopK
from fps_b200.store.sharded_table import ShardedTable

torch.cuda.set_device(0)
users = ShardedTable(100_000, 64, seed=1, init_range=(-1, 1))          # parameter server
items = ShardedTable(200_000, 64, seed=2, init_range=(-1, 1))          # this worker's items
queries = torch.randint(0, 100_000, (1024,), device="cuda")
scores, rows = DeviceTopK(items.local).topk(10, q_ids=queries, q_table=users, rescore=True)
print("user", int(queries[0]), "->", rows[0].tolist(), [round(s, 2) for s in scores[0].tolist()])

# LEMP-style LENGTH pruning: keep the item table sorted by vector length; with skewed lengths (popular
# items have long vectors) only a prefix of the table has to be scored.  Same results, same row numbers.
items.local.mul_(torch.exp(torch.randn(items.local.shape[0], 1, device="cuda")))
pruned = DeviceTopK(items.local, sort_by_length=True)
s2, r2 = pruned.topk(10, q_ids=queries, q_table=users)
p1, p2 = pruned.last_tiles_scored
print(f"length-sorted table: scored {p2} of {pruned.n_tiles} item tiles in pass 2; top-1 item of user "
      f"{int(queries[0])}: {int(r2[0, 0])}")
