"""Record-batch refusals of every binding that takes training records, and the ctypes mirrors of the kernel argument
blocks and the flush state against the C structs.  No GPU: the refusals come before any CUDA check, the layouts
are read from a host program compiled with nvcc."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

import fps_b200  # noqa: F401
from fps_b200.ops import build, native

BINDINGS = {
    "mf_sgd_fused": lambda u, i, r: native.mf_sgd_fused(u, i, r, None, 1, None, 0.1),
    "mf_sgd_fused_f64": lambda u, i, r: native.mf_sgd_fused_f64(u, i, r, None, 1, None, 0.1),
    "mf_bpr_fused": lambda u, i, r: native.mf_bpr_fused(u, i, r, None, None, 0.1),
    "mf_warp_fused": lambda u, i, r: native.mf_warp_fused(u, i, r, None, None, 0.1),
    "neg_sample": lambda u, i, r: native.neg_sample(u, i, r, 1, 8, None, None, 1),
    "neg_sample_seen": lambda u, i, r: native.neg_sample_seen(u, i, r, 1, None),
    "neg_sample_noise": lambda u, i, r: native.neg_sample_noise(u, i, r, 1, None, 0),
    "bucket_by_item": lambda u, i, r: native.bucket_by_item(u, i, r, 0, 1, None),
}


@pytest.fixture(autouse=True)
def _no_library(monkeypatch):
    """Every refusal must come before the kernel library is loaded."""
    def refuse():
        raise AssertionError("the kernel library was loaded before the records were refused")
    monkeypatch.setattr(native, "lib", refuse)


def _batch(n=4, dtype=torch.int32, n_items=None, n_ratings=None, item_dtype=None):
    return (torch.zeros(n, dtype=dtype), torch.zeros(n if n_items is None else n_items, dtype=item_dtype or dtype),
            torch.ones(n if n_ratings is None else n_ratings))


@pytest.mark.parametrize("name", sorted(BINDINGS))
@pytest.mark.parametrize("dtype", [torch.int32, torch.float64])
def test_packed_records_must_be_int64(name, dtype):
    with pytest.raises(TypeError, match="packed rating records must be an int64 tensor"):
        BINDINGS[name](torch.zeros(4, dtype=dtype), None, None)


@pytest.mark.parametrize("name", sorted(BINDINGS))
def test_id_dtypes_must_agree(name):
    with pytest.raises(TypeError, match="share an integer dtype"):
        BINDINGS[name](*_batch(item_dtype=torch.int64))


@pytest.mark.parametrize("name", sorted(BINDINGS))
@pytest.mark.parametrize("lengths", [dict(n_items=3), dict(n_ratings=3), dict(n_items=5), dict(n_ratings=5)],
                         ids=["short-items", "short-ratings", "long-items", "long-ratings"])
def test_record_lengths_must_agree(name, lengths):
    with pytest.raises(ValueError, match="same length"):
        BINDINGS[name](*_batch(**lengths))


@pytest.mark.parametrize("name", sorted(BINDINGS))
def test_ratings_must_be_float32(name):
    u, i, _ = _batch()
    with pytest.raises(TypeError, match="ratings must be"):
        BINDINGS[name](u, i, torch.ones(4, dtype=torch.float64))


# ---- ctypes mirrors of the argument blocks ---------------------------------------------------------------------

def _nvcc():
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if Path(cand).exists() else None


def _layout(tmp_path, header, lines):
    """Run a host program that includes ``header`` and prints ``lines`` (``key value`` pairs)."""
    src = tmp_path / "layout.cu"
    src.write_text(f'#include <cstddef>\n#include <cstdio>\n#include "{header}"\nint main() {{\n'
                   + "\n".join(lines) + "\n  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([_nvcc(), *build.NVCC_FLAGS, "-I", str(build.CSRC), str(src), "-o", str(exe)], check=True,
                   capture_output=True)
    return dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                        text=True).stdout.splitlines())


STRUCT_HEADER = {"MfArgs": "fps_mf_args.cuh", "BprArgs": "fps_mf_args.cuh", "ExchArgs": "fps_replica.cu",
                 "FlushPolicy": "fps_replica.cu", "BucketArgs": "fps_bucket.cu",
                 "W2vArgs": "fps_w2v_window.cu"}   # where each struct lives


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
@pytest.mark.parametrize("struct, mirror", [
    ("MfArgs", native.MfArgsC), ("BprArgs", native.BprArgsC), ("ExchArgs", native.ExchArgsC),
    ("FlushPolicy", native.FlushPolicyC), ("BucketArgs", native.BucketArgsC), ("W2vArgs", native.W2vArgsC)])
def test_args_mirror_matches_the_c_layout(tmp_path, struct, mirror):
    lines = [f'  printf("sizeof %zu\\n", sizeof({struct}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({struct}, {f}));' for f, _ in mirror._fields_]
    want = {f: str(getattr(mirror, f).offset) for f, _ in mirror._fields_}
    want["sizeof"] = str(C.sizeof(mirror))
    assert _layout(tmp_path, STRUCT_HEADER[struct], lines) == want


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_flush_state_words_match_the_c_layout(tmp_path):
    fields = {"pending": native.FLUSH_PENDING, "last_ns": native.FLUSH_LAST_NS, "flushes": native.FLUSH_COUNT,
              "mask": native.FLUSH_MASK}
    lines = ['  printf("sizeof %zu\\n", sizeof(FlushState));']
    lines += [f'  printf("{f} %zu\\n", offsetof(FlushState, {f}));' for f in fields]
    want = {f: str(8 * w) for f, w in fields.items()}
    want["sizeof"] = str(8 * native.FLUSH_STATE_WORDS)
    assert _layout(tmp_path, "fps_replica.cu", lines) == want
