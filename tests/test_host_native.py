"""Native host runtime (libfps_host.so): partitioner/packer and key interner."""
import numpy as np
import torch

from fps_b200.ops import host, native


def test_partition_pack_matches_torch_reference():
    g = torch.Generator().manual_seed(0)
    n, W = 100_003, 4
    u = torch.randint(0, 1 << 20, (n,), generator=g, dtype=torch.int32)
    i = torch.randint(0, 1 << 18, (n,), generator=g, dtype=torch.int32)
    r = torch.rand(n, generator=g) * 5
    parts = host.partition_pack(u, i, r, W, pin=False, threads=3)
    ref = native.pack_ratings(u, i, r)
    for w in range(W):
        sel = (u % W) == w
        assert torch.equal(parts[w], ref[sel])           # stable order, identical fp16 rounding
    assert sum(p.numel() for p in parts) == n


def test_native_interner():
    it = host.NativeInterner()
    a = it.map([10, -5, 10, 7])
    assert a.tolist() == [0, 1, 0, 2] and len(it) == 3
    assert it.map([7, 99], insert=False).tolist() == [2, -1]
    assert it.keys().tolist() == [10, -5, 7]


def test_kernel_library_builds_and_is_current():
    """nvcc cross-compiles every kernel for sm_90a (no GPU needed); a stale or broken build fails here."""
    from fps_b200.ops import build

    path = build.build_kernels()          # rebuilds when sources changed; raises on compile errors
    assert path.exists()
    srcs = sorted(build.CSRC.glob("*.cu")) + sorted(build.CSRC.glob("*.cuh")) + sorted(build.CSRC.glob("*.h"))
    assert not build._stale(path, srcs)
    import ctypes
    lib = ctypes.CDLL(str(path))
    for sym in ["fps_mf_sgd_fused", "fps_mf_sgd_tma", "fps_topk_mma", "fps_pa_step", "fps_sketch_update",
                "fps_server_loop_launch", "fps_client_issue", "fps_client_collect", "fps_replica_exchange", "fps_flush_policy",
                "fps_pull_gather", "fps_push_add", "fps_push_assign", "fps_pull_dot", "fps_init_rows",
                "fps_bloom_query", "fps_rings_preload"]:
        assert hasattr(lib, sym), sym
