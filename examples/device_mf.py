"""Fused online SGD matrix factorisation on an H100:  python examples/device_mf.py
   or  python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 examples/device_mf.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.distributed as dist
from fps_b200.models.mf.device import DeviceOnlineMF, ERR_PLAIN
from fps_b200.ops import native

world, rank = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0))
torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
if world > 1:
    dist.init_process_group("nccl")
nu, ni = 1_000_000, 100_000
mf = DeviceOnlineMF(nu, ni, 64, range_min=0.0, range_max=0.1, learning_rate=0.02, err_mode=ERR_PLAIN, seed=1)
g = torch.Generator().manual_seed(rank)
def batches(n, size=1 << 20):
    for _ in range(n):
        u = torch.randint(0, nu // world, (size,), generator=g, dtype=torch.int32) * world + rank   # users this worker owns
        i = torch.randint(0, ni, (size,), generator=g, dtype=torch.int32)
        r = ((u % 7 + i % 5).float() / 10).half().float()
        yield (native.pack_ratings(u, i, r).pin_memory(),)
for step, (sse, n) in enumerate(mf.fit_stream(batches(30))):
    if rank == 0 and step % 5 == 0:
        print(f"step {step:3d}  mse {sse / n:.4f}")
mf.barrier(); mf.close()
if world > 1:
    dist.destroy_process_group()
