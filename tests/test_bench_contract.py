"""CPU-side checks of ``bench.py``'s contract with the driver: the reference arm's one-line answer (also
under torch.distributed.run: rank 0 only) and the bookkeeping of the convergence gate (``config.quality``)."""
import json
import os
import subprocess
import sys
import types

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(env_extra):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--gpus", "2",
                        "--steps", "20", "--warmup", "5"], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, r.stderr
    return r.stdout.strip()


def test_reference_arm_prints_one_unavailable_line_from_rank_0_only():
    out = _run({"RANK": "0", "WORLD_SIZE": "2", "LOCAL_RANK": "0"})
    d = json.loads(out)
    assert d["impl"] == "reference" and "unavailable" in d and d["n_gpus"] == 2
    assert _run({"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}) == ""


def test_quality_gate_bookkeeping_with_a_stub_model():
    sys.path.insert(0, REPO)
    import bench

    class Stub:
        steps = 0

        def __init__(self, nu, ni, k, **kw):
            self.kw = kw

        def step(self, u, i, r):
            assert u.dtype == torch.int32 and u.numel() == 256 and float(r.abs().max()) < 4.0
            Stub.steps += 1

        def refresh(self): pass
        def check_finite(self): pass
        def predict(self, u, i): return torch.zeros(u.numel())
        def barrier(self): pass
        def close(self): pass

    a = types.SimpleNamespace(quality_updates_per_user=12.0, users=1000, items=500, factors=4, batch=256,
                              quality_lr=0.05, quality_init=0.05, sync_every=4)
    q = bench.quality_gate(a, 1, 0, torch.device("cpu"), False, Stub, 1, checkpoints=[4.0, 12.0])
    assert q["steps_per_worker"] == [15, 46] and Stub.steps == 46          # the curve continues, it does not restart
    assert q["updates"] == [15 * 256, 46 * 256]
    assert len(q["rmse_single_worker"]) == 2 and abs(q["rmse_single_worker"][0] - q["rmse_untrained"]) < 0.01


def test_dump_outputs_names_dtypes_size_and_fixed_sample(tmp_path):
    """``--dump-outputs``: float32 / float64 arrays, below 64 MB even at k = 1, the same seeded rows every time."""
    import numpy as np

    sys.path.insert(0, REPO)
    import bench

    def stub(k, n_users, n_items, world):
        g = torch.Generator().manual_seed(3)
        items = torch.rand((n_items, k), generator=g)
        return types.SimpleNamespace(k=k, num_users=n_users, num_items=n_items, cuda_device=torch.device("cpu"),
                                     users=torch.rand((-(-n_users // world), k), generator=g),
                                     items=types.SimpleNamespace(pull=lambda ids: items[ids.long()]),
                                     stats=torch.tensor([12.5, 256.0]), table=items)

    def dump(m, d, world, rank):
        bench.dump_outputs(str(tmp_path / d), m, world, rank)
        return {p.stem: np.load(p) for p in (tmp_path / d).glob("*.npy")}

    m = stub(1, 10_000_000, 8_000_000, 1)
    f = dump(m, "a", 1, 0)
    assert sum(p.stat().st_size for p in (tmp_path / "a").glob("*.npy")) <= 64 << 20
    assert f["stats"].dtype == np.float64 and f["stats"].tolist() == [12.5, 256.0]
    for t in ("user", "item"):
        assert f[t + "_ids"].dtype == np.float64 and f[t + "_vectors"].dtype == np.float32
        assert f[t + "_vectors"].shape == (f[t + "_ids"].size, 1) and np.all(np.diff(f[t + "_ids"]) > 0)
    np.testing.assert_array_equal(f["item_vectors"][:, 0], m.table[f["item_ids"].astype(np.int64), 0])
    m2 = stub(4, 1000, 500, 2)
    b, c = dump(m2, "b", 2, 0), dump(m2, "c", 2, 0)
    assert b.keys() == c.keys() and all(np.array_equal(b[n], c[n]) for n in b)
    assert b["user_ids"].size == 500 and np.all(b["user_ids"] % 2 == 0)
    assert dump(m2, "d", 2, 1) == {}                  # only rank 0 writes
