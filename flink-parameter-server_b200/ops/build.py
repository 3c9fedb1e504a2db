"""In-tree build of the fps_b200 native libraries.

Two shared objects are produced next to this file (git-ignored build products):

* ``libfps_kernels.so`` -- every hand-written sm_90a (H100) CUDA kernel + the symmetric-heap fabric,
  compiled by nvcc with ``-gencode arch=compute_90a,code=sm_90a -lineinfo`` and exposed through a
  plain C ABI (raw device pointers + ``cudaStream_t``), loaded with ``ctypes``.
* ``libfps_host.so`` -- the native host runtime (id interning, partitioner / batch packer,
  lock-free SPSC rings), compiled by g++.

The reference has no native code at all (SURVEY §2.9); these libraries are the GPU-native
replacement for its JVM hot loops.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

OPS_DIR = Path(__file__).resolve().parent
CSRC = OPS_DIR / "csrc"
KERNEL_LIB = OPS_DIR / "libfps_kernels.so"
HOST_LIB = OPS_DIR / "libfps_host.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; cannot build fps_b200 CUDA kernels")
    return cand


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _stale(lib: Path, srcs) -> bool:
    stamp = lib.with_suffix(".sha")
    if not lib.exists() or not stamp.exists():
        return True
    return stamp.read_text().strip() != _digest(srcs)


def build_kernels(force: bool = False, verbose: bool = False) -> Path:
    cu = sorted(CSRC.glob("*.cu"))
    hdr = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    if not force and not _stale(KERNEL_LIB, cu + hdr):
        return KERNEL_LIB
    build_dir = OPS_DIR / "build"
    build_dir.mkdir(exist_ok=True)
    objs = []
    procs = []
    for src in cu:
        obj = build_dir / (src.stem + ".o")
        cmd = [_nvcc(), *NVCC_FLAGS, "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src.name}:\n{out.decode()}")
        if verbose:
            sys.stderr.write(out.decode())
    link = [_nvcc(), "-shared", "-o", str(KERNEL_LIB), *map(str, objs), "-lcudart", "-lcuda"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout.decode()}")
    KERNEL_LIB.with_suffix(".sha").write_text(_digest(cu + hdr))
    return KERNEL_LIB


def build_host(force: bool = False) -> Path:
    cpp = sorted(CSRC.glob("*.cpp"))
    if not cpp:
        return HOST_LIB
    if not force and not _stale(HOST_LIB, cpp):
        return HOST_LIB
    cmd = ["g++", "-O3", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", str(HOST_LIB),
           *map(str, cpp)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError(f"g++ failed:\n{r.stdout.decode()}")
    HOST_LIB.with_suffix(".sha").write_text(_digest(cpp))
    return HOST_LIB


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_kernels(force=force, verbose=verbose)
    build_host(force=force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", KERNEL_LIB, HOST_LIB if HOST_LIB.exists() else "")
