"""Launch the multi-rank device checks under torchrun.

With >= 2 GPUs every rank gets its own GPU (NCCL control plane, NVLink data plane).  On a single-GPU
box the same checks run with the ranks SHARING the GPU (gloo control plane; CUDA IPC maps the other
processes' shards exactly like peer GPUs), so the multi-rank logic -- fabric, one-sided pull/push,
replica exchange, distributed top-K -- is exercised by every ``pytest -m gpu`` run."""
import os
import subprocess
import tempfile

import pytest
import torch

from tests.mp_util import REPO, launch_cmd

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]    # torchrun children: their own 420 s limit applies first


def _run(script: str, world: int, port: int, ok: str, timeout: int = 420):
    env = dict(os.environ)
    if torch.cuda.device_count() < world:
        env["FPS_SHARE_GPU"] = "1"
    r = subprocess.run(launch_cmd(script, world, port), cwd=REPO, capture_output=True, text=True,
                       timeout=timeout, env=env)
    if r.returncode != 0 or ok not in r.stdout:      # keep the full transcript for post-mortems
        with open(os.path.join(tempfile.gettempdir(), f"fps_mp_fail_{script}.log"), "w") as f:
            f.write(r.stdout + "\n=== stderr ===\n" + r.stderr)
    err = [l for l in r.stderr.splitlines() if "Error" in l or "assert" in l.lower()]
    assert r.returncode == 0 and ok in r.stdout, "\n".join(err[:12]) + r.stdout[-1500:] + r.stderr[-1500:]
    return r.stdout


def _world(prefer: int = 4) -> int:
    n = torch.cuda.device_count()
    return 2 if n < prefer else prefer


def test_multi_rank_fabric_and_fused_step():
    _run("mp_device_check.py", _world(), 29617, "MP_DEVICE_CHECK_OK")


def test_multi_rank_distributed_topk():
    _run("mp_topk_check.py", 2, 29618, "MP_TOPK_CHECK_OK")


def test_multi_rank_replica_exchange_conservation_and_convergence():
    _run("mp_replica_check.py", _world(), 29619, "MP_REPLICA_CHECK_OK")


def test_multi_rank_online_learner_and_topk_generator():
    _run("mp_learner_check.py", _world(), 29620, "MP_LEARNER_CHECK_OK")
