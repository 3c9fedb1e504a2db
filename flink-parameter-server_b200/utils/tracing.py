"""Tracing / profiling helpers the reference lacks (SURVEY §5: only ``log.debug`` per message).

* :func:`nvtx_range` -- NVTX ranges around engine phases (visible in ncu / nsys timelines).
* :class:`DeviceTimer` -- CUDA-event timing of a region on the current stream (never wall clock).
* :func:`roofline` -- achieved fraction of the measured peaks in ``MEASURED_PEAKS.json``.
* :func:`sanitizer_cmd` -- the ``compute-sanitizer`` invocations used as race / memory checks for the
  control structures (rings, credit counters); the shard rows themselves are *intentionally* racy
  (Hogwild asynchronous SGD), so racecheck is scoped to the message-tier tests.
"""
from __future__ import annotations

import contextlib
import json
import os
from typing import Dict

import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@contextlib.contextmanager
def nvtx_range(name: str):
    on = torch.cuda.is_available()
    if on:
        torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        if on:
            torch.cuda.nvtx.range_pop()


class DeviceTimer:
    """``with DeviceTimer() as t: ...`` then ``t.ms`` (synchronises on exit)."""

    def __enter__(self):
        self.e0 = torch.cuda.Event(enable_timing=True)
        self.e1 = torch.cuda.Event(enable_timing=True)
        self.e0.record()
        return self

    def __exit__(self, *exc):
        self.e1.record()
        self.e1.synchronize()
        self.ms = self.e0.elapsed_time(self.e1)
        return False


def measured_peaks() -> Dict[str, float]:
    path = os.path.join(REPO, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            d = json.load(f)
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"], "source": "measured"}
    # H100 SXM data sheet (700 W card): HBM3 bandwidth and dense BF16 rate -- ceilings, not measurements
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "source": "H100 SXM data sheet"}


def roofline(bytes_moved: float, flops: float, ms: float, nvlink_bytes: float = 0.0) -> Dict[str, float]:
    """Achieved / bound for a kernel: bound = slowest of HBM bytes, NVLink bytes (450 GB/s/dir,
    the NVLink 4 data-sheet rate of an H100 SXM) and tensor FLOPs at the peaks of :func:`measured_peaks`."""
    p = measured_peaks()
    t_hbm = bytes_moved / (p["hbm_gbs"] * 1e9)
    t_link = nvlink_bytes / 450e9
    t_flop = flops / (p["bf16_tflops"] * 1e12)
    bound = max(t_hbm, t_link, t_flop)
    return {"ms": ms, "bound_ms": bound * 1e3, "fraction_of_roofline": bound * 1e3 / ms if ms > 0 else 0.0,
            "hbm_GBs": bytes_moved / ms / 1e6 if ms > 0 else 0.0, "peaks": p["source"]}


def sanitizer_cmd(tool: str = "racecheck", test: str = "tests/test_gpu_rings.py") -> str:
    return (f"compute-sanitizer --tool {tool} --error-exitcode 1 python -m pytest {test} -x -q "
            "-k 'credit or registered'")
