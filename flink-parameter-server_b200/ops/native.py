"""ctypes bindings for ``libfps_kernels.so`` (hand-written sm_90a kernels + fabric).

Every wrapper takes torch CUDA tensors, validates them, and launches on the *current* torch
CUDA stream, so launches compose with torch streams, events and CUDA-graph capture.  There is
no PyTorch fallback on a GPU box: if the library is missing the ops raise.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import threading
from typing import Optional

import torch

from . import build as _build

FPS_MAX_SHARDS = 16
PART_HASH = 0
PART_RANGE = 1
PART_LUT = 2
LUT_OWNER_SHIFT = 40

_lib = None
_lib_lock = threading.Lock()
_launch_count = 0  # number of fps kernels launched by this process (bench "gpu_launches")


class ShardTableC(C.Structure):
    """Mirror of ``struct ShardTable`` (csrc/fps_common.cuh)."""

    _fields_ = [
        ("base", C.c_void_p * FPS_MAX_SHARDS),
        ("touched", C.c_void_p * FPS_MAX_SHARDS),
        ("rows_per_shard", C.c_longlong),
        ("div", C.c_longlong),
        ("num_shards", C.c_int),
        ("dim", C.c_int),
        ("stride", C.c_int),
        ("mode", C.c_int),
        ("shard_shift", C.c_int),
        ("pad_", C.c_int),
        ("lut", C.c_void_p),
    ]


class MfArgsC(C.Structure):
    """Mirror of ``struct MfArgs`` (csrc/fps_mf_args.cuh)."""

    _fields_ = [
        ("users", C.c_void_p),
        ("items", C.c_void_p),
        ("ratings", C.c_void_p),
        ("n_pos", C.c_longlong),
        ("neg_rate", C.c_int),
        ("num_items", C.c_longlong),
        ("seed", C.c_ulonglong),
        ("step", C.c_ulonglong),
        ("user_table", C.c_void_p),
        ("user_div", C.c_int),
        ("user_shift", C.c_int),
        ("lr", C.c_float),
        ("err_mode", C.c_int),
        ("format", C.c_int),
        ("stats", C.c_void_p),
        ("nan_flag", C.c_void_p),
        ("item_tab", ShardTableC),
        ("user_tab", ShardTableC),
        ("user_sharded", C.c_int),
        ("use_push_tab", C.c_int),
        ("push_tab", ShardTableC),
        ("l2_hints", C.c_int),
        ("pad2_", C.c_int),
        ("progress", C.c_void_p),
        ("out_ids", C.c_void_p),
        ("out_vecs", C.c_void_p),
        ("out_staged", C.c_void_p),
        ("out_cap", C.c_longlong),
        ("out_every", C.c_int),
        ("reserve_total", C.c_int),
        ("credits", C.c_void_p),
        ("item_acc", ShardTableC),
        ("user_acc_tab", ShardTableC),
        ("user_acc", C.c_void_p),
    ]


def available() -> bool:
    return _build.KERNEL_LIB.exists()


def lib() -> C.CDLL:
    """Load (building if needed) the kernel library.  Raises if it cannot be produced."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        path = _build.KERNEL_LIB
        if not path.exists() or os.environ.get("FPS_REBUILD") == "1":
            _build.build_kernels()
        l = C.CDLL(str(path))
        l.fps_error_string.restype = C.c_char_p
        l.fps_error_string.argtypes = [C.c_int]
        _lib = l
    return _lib


def launch_count() -> int:
    return _launch_count


def reset_launch_count() -> None:
    global _launch_count
    _launch_count = 0


def _check(code: int, what: str) -> None:
    if code != 0:
        msg = lib().fps_error_string(int(code))
        raise RuntimeError(f"fps_b200 native call {what} failed: [{code}] {msg.decode() if msg else ''}")


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


_sm_cache = {}


def sm_count(device: Optional[int] = None) -> int:
    dev = torch.cuda.current_device() if device is None else int(device)
    if dev not in _sm_cache:
        _sm_cache[dev] = torch.cuda.get_device_properties(dev).multi_processor_count
    return _sm_cache[dev]


def log2_or_neg(n: int) -> int:
    """log2(n) if n is a power of two, else -1 (kernels then use a real division)."""
    return n.bit_length() - 1 if n > 0 and (n & (n - 1)) == 0 else -1


def _id_bytes(ids: torch.Tensor) -> int:
    if ids.dtype == torch.int32:
        return 4
    if ids.dtype == torch.int64:
        return 8
    raise TypeError(f"ids must be int32 or int64, got {ids.dtype}")


def _req(t: torch.Tensor, name: str, dtype=None) -> None:
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")


def _req_vec4(t: torch.Tensor, name: str) -> None:
    """A ``[n, w]`` row buffer with ``w % 4 == 0`` is moved in 16-byte vectors by the row kernels, so its first
    element must sit on a 16-byte boundary.  A contiguous view with a storage offset that is not a multiple of 4
    floats would pass ``_req`` and reach the device as misaligned vector accesses."""
    if t.dim() == 2 and t.shape[1] % 4 == 0 and t.data_ptr() % 16 != 0:
        raise ValueError(f"{name}: rows {t.shape[1]} floats wide must start on a 16-byte boundary "
                         f"(storage offset {t.storage_offset()} floats); pass a copy or an aligned view")


def _bump(n: int = 1) -> None:
    global _launch_count
    _launch_count += n


# --------------------------------------------------------------------------------------------
# fabric
# --------------------------------------------------------------------------------------------
def heap_alloc(nbytes: int) -> int:
    out = C.c_void_p()
    _check(lib().fps_heap_alloc(C.c_size_t(nbytes), C.byref(out)), "heap_alloc")
    return int(out.value)


def heap_free(ptr: int) -> None:
    _check(lib().fps_heap_free(C.c_void_p(ptr)), "heap_free")


def ipc_get_handle(ptr: int) -> bytes:
    buf = (C.c_ubyte * 64)()
    _check(lib().fps_ipc_get_handle(C.c_void_p(ptr), buf), "ipc_get_handle")
    return bytes(buf)


def ipc_open_handle(handle: bytes) -> int:
    buf = (C.c_ubyte * 64).from_buffer_copy(handle)
    out = C.c_void_p()
    _check(lib().fps_ipc_open_handle(buf, C.byref(out)), "ipc_open_handle")
    return int(out.value)


def ipc_close(ptr: int) -> None:
    _check(lib().fps_ipc_close(C.c_void_p(ptr)), "ipc_close")


def enable_peer(dev: int, peer: int) -> None:
    _check(lib().fps_enable_peer(int(dev), int(peer)), f"enable_peer({dev},{peer})")


class _RawCudaBuffer:
    """Expose a raw device allocation through ``__cuda_array_interface__`` (zero-copy view)."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {
            "shape": tuple(shape),
            "typestr": typestr,
            "data": (int(ptr), False),
            "version": 3,
            "strides": None,
        }


_TYPESTR = {torch.float32: "<f4", torch.int32: "<i4", torch.int64: "<i8", torch.uint8: "|u1",
            torch.float16: "<f2", torch.int16: "<i2"}


def tensor_from_ptr(ptr: int, shape, dtype: torch.dtype, device: int) -> torch.Tensor:
    """Zero-copy torch view of raw device memory (the owner keeps the allocation alive)."""
    if dtype == torch.bfloat16:
        t = torch.as_tensor(_RawCudaBuffer(ptr, shape, "<i2"), device=torch.device("cuda", device))
        return t.view(torch.bfloat16)
    return torch.as_tensor(_RawCudaBuffer(ptr, shape, _TYPESTR[dtype]),
                           device=torch.device("cuda", device))


# --------------------------------------------------------------------------------------------
# kernels
# --------------------------------------------------------------------------------------------
def init_rows(rows: torch.Tensor, dim: int, shard: int, num_shards: int, mode: int, div: int,
              seed: int, lo: float, hi: float) -> None:
    _req(rows, "rows", torch.float32)
    n_rows, stride = rows.shape
    assert stride % 4 == 0
    _check(lib().fps_init_rows(C.c_void_p(rows.data_ptr()), C.c_longlong(n_rows), int(dim),
                               int(stride), int(shard), int(num_shards), int(mode),
                               C.c_longlong(div), C.c_ulonglong(seed & (2**64 - 1)),
                               C.c_float(lo), C.c_float(hi), _stream()), "init_rows")
    _bump()


MF_ERR_MODES = (0, 1, 2)   # the error rules of the pointwise step (fps_mf_args.cuh fps_mf_grad)


def _records(users, items, ratings):
    """Validate a batch of training records and return ``(packed, id_bytes)``.  ``items=None``: ``users`` holds
    packed64 records (:func:`pack_ratings`; the kernels decode their ids as int32).  Otherwise ``users``, ``items``
    and ``ratings`` are arrays of one length, with one int32 or int64 id dtype and float32 ratings.  The dtype and
    length refusals come before the CUDA checks."""
    if items is None:
        if users.dtype != torch.int64:
            raise TypeError("packed rating records must be an int64 tensor (see pack_ratings)")
        _req(users, "users")
        return True, 4
    if users.dtype != items.dtype:
        raise TypeError("users and items must share an integer dtype")
    id_bytes = _id_bytes(users)
    if ratings.dtype != torch.float32:
        raise TypeError(f"ratings must be {torch.float32}, got {ratings.dtype}")
    if items.numel() != users.numel() or ratings.numel() != users.numel():
        raise ValueError("users, items and ratings must have the same length")
    _req(users, "users"); _req(items, "items"); _req(ratings, "ratings")
    return False, id_bytes


def _shard_count(num_shards) -> None:
    """The device kernels keep per-shard state in arrays of ``FPS_MAX_SHARDS`` entries."""
    if not 1 <= int(num_shards) <= FPS_MAX_SHARDS:
        raise ValueError(f"num_shards must be in [1, {FPS_MAX_SHARDS}], got {num_shards}")


def _check_err_mode(err_mode) -> None:
    if int(err_mode) not in MF_ERR_MODES:
        raise ValueError(f"err_mode must be one of {MF_ERR_MODES}, got {err_mode!r}")


def _set_row_acc(a, name: str, acc, table, sharded: bool) -> None:
    """Row-wise AdaGrad accumulators of the ``name`` rows (``user`` / ``anchor``) of ``a``: a stride-1
    :class:`ShardTableC` in ``<name>_acc_tab`` when the row table is sharded, else a float32 tensor with one entry
    per row of ``table`` in ``<name>_acc``."""
    if sharded:
        if not isinstance(acc, ShardTableC) or int(acc.stride) != 1:
            raise ValueError(f"a sharded {name} table needs a stride-1 ShardTableC {name}_acc")
        setattr(a, f"{name}_acc_tab", acc)
        return
    if not torch.is_tensor(acc):
        raise ValueError(f"a worker-local {name} table needs a float32 {name}_acc tensor")
    _req(acc, f"{name}_acc", torch.float32)
    if acc.numel() < table.shape[0]:
        raise ValueError(f"{name}_acc must hold one accumulator per {name} row")
    setattr(a, f"{name}_acc", acc.data_ptr())


def mf_sgd_fused(users: torch.Tensor, items: torch.Tensor, ratings: torch.Tensor,
                 user_table, user_div: int, item_tab: ShardTableC, lr: float,
                 err_mode: int = 0, neg_rate: int = 0, num_items: int = 0, seed: int = 0,
                 step: int = 0, stats: Optional[torch.Tensor] = None,
                 nan_flag: Optional[torch.Tensor] = None, max_inflight_rows: int = 0,
                 kernel: Optional[str] = None, push_tab: Optional[ShardTableC] = None,
                 l2_hints: bool = False, reserve_total: int = 0,
                 progress: Optional[torch.Tensor] = None, output=None,
                 credits: Optional[torch.Tensor] = None, item_acc: Optional[ShardTableC] = None,
                 user_acc=None) -> None:
    """Fused pull + SGD + push (K1+K3+K2).

    ``item_acc`` / ``user_acc``: row-wise AdaGrad instead of SGD (DESIGN §2.10).  ``item_acc`` is a stride-1
    :class:`ShardTableC` of one fp32 accumulator per item row, partitioned like ``item_tab``; ``user_acc`` is
    a float32 ``[n_local]`` tensor, or a stride-1 :class:`ShardTableC` when ``user_table`` is one.  AdaGrad
    runs on the register-staged kernel only, without ``push_tab``, ``output`` or ``credits``.

    ``kernel="reg"`` (default): register-staged loads at full occupancy (csrc/fps_core.cu);
    ``kernel="tma"``: warp-specialised TMA/mbarrier pipeline (csrc/fps_mf_tma.cu) -- slower for
    256-byte rows, kept for large rows.
    ``items=None`` means ``users`` holds packed64 records (see :func:`pack_ratings`).

    ``err_mode``: 0 ``e = sigmoid(r - u.v)``, 1 ``e = r - u.v``, 2 ``e = r - sigmoid(u.v)``.  ``neg_rate > 0``
    draws that many negatives per record in the kernel, uniform over ``[0, num_items)`` and never the
    positive, so it needs ``num_items >= 2``.  ``reserve_total``: CTA slots the grid leaves free for a kernel running
    next to it (the replica exchange)."""
    _check_err_mode(err_mode)
    if int(neg_rate) > 0 and int(num_items) < 2:
        raise ValueError(f"sampled negatives need num_items >= 2, got {num_items}")
    packed, id_bytes = _records(users, items, ratings)
    user_sharded = isinstance(user_table, ShardTableC)
    if not user_sharded:
        _req(user_table, "user_table", torch.float32)
    if (user_table.stride if user_sharded else user_table.shape[1]) != item_tab.stride:
        raise ValueError("user table stride must equal item table stride")
    a = MfArgsC()
    a.users = users.data_ptr()
    a.items = None if packed else items.data_ptr()
    a.ratings = None if packed else ratings.data_ptr()
    a.format = 1 if packed else 0
    a.n_pos = users.numel(); a.neg_rate = int(neg_rate); a.num_items = int(max(num_items, 1))
    a.seed = seed & (2**64 - 1); a.step = int(step)
    if user_sharded:
        a.user_table = None; a.user_tab = user_table; a.user_sharded = 1
    else:
        a.user_table = user_table.data_ptr(); a.user_sharded = 0
    a.user_div = int(user_div)
    a.user_shift = log2_or_neg(int(user_div))
    a.lr = float(lr); a.err_mode = int(err_mode)
    a.stats = stats.data_ptr() if stats is not None else None
    a.nan_flag = nan_flag.data_ptr() if nan_flag is not None else None
    a.item_tab = item_tab
    if push_tab is not None:
        a.push_tab = push_tab; a.use_push_tab = 1
    a.l2_hints = 1 if l2_hints else 0
    variant = kernel or os.environ.get("FPS_MF_KERNEL", "reg")
    if packed or push_tab is not None or l2_hints or output is not None or credits is not None:
        variant = "reg"
    a.progress = progress.data_ptr() if progress is not None else None
    if credits is not None:    # device-side credit-counter pull limiter (int32 [credits, stalls])
        _req(credits, "credits", torch.int32)
        a.credits = credits.data_ptr()
    if output is not None:     # E5 worker output stream: (out_ids, out_vecs, staged counter, capacity, every)
        o_ids, o_vecs, o_staged, o_cap, o_every = output
        a.out_ids = o_ids.data_ptr(); a.out_vecs = o_vecs.data_ptr(); a.out_staged = o_staged.data_ptr()
        a.out_cap = int(o_cap); a.out_every = int(o_every)
    if item_acc is not None:
        if push_tab is not None or output is not None or credits is not None:
            raise ValueError("row-wise AdaGrad does not support push_tab, output or credits")
        if int(item_acc.stride) != 1:
            raise ValueError("item_acc must be a stride-1 accumulator table")
        a.item_acc = item_acc
        _set_row_acc(a, "user", user_acc, user_table, user_sharded)
        variant = "reg"
    elif user_acc is not None:
        raise ValueError("user_acc needs item_acc")
    a.reserve_total = max(0, int(reserve_total))
    rv = os.environ.get("FPS_MF_REG_VARIANT")
    if rv is not None:
        lib().fps_set_mf_reg_variant(int(rv))
    if variant == "tma":
        code = lib().fps_mf_sgd_tma(C.byref(a), id_bytes, int(max_inflight_rows),
                                    sm_count(users.device.index), _stream())
        if code != -1002:  # -1002: rows too large for the smem ring -> register-staged kernel
            _check(code, "mf_sgd_tma")
            _bump()
            return
    _check(lib().fps_mf_sgd_fused(C.byref(a), id_bytes, int(max_inflight_rows),
                                  sm_count(users.device.index), _stream()), "mf_sgd_fused")
    _bump()


WINDOW_MAX = 8   # micro-batches per drain (csrc/fps_mf_window.cu WIN_MAX)


class WinArgsC(C.Structure):
    """Mirror of ``struct WinArgs`` (csrc/fps_mf_window.cu)."""

    _fields_ = [
        ("stage", C.c_void_p), ("slot_bytes", C.c_longlong),
        ("n", C.c_longlong * WINDOW_MAX), ("fmt", C.c_int * WINDOW_MAX),
        ("n_slots", C.c_int), ("err_mode", C.c_int), ("lr", C.c_float), ("stride", C.c_int),
        ("user_table", C.c_void_p), ("item_table", C.c_void_p), ("rows", C.c_longlong),
        ("slots", C.c_void_p), ("user_bits", C.c_void_p), ("bm_words", C.c_longlong),
        ("ctl", C.c_void_p), ("stats", C.c_void_p), ("slot_stats", C.c_void_p), ("nan_flag", C.c_void_p),
        ("phase_ns", C.c_void_p),
    ]


def mf_window_drain(stage: torch.Tensor, slot_bytes: int, counts, formats, user_table: torch.Tensor,
                    item_table: torch.Tensor, lr: float, err_mode: int, slots: torch.Tensor,
                    user_bits: torch.Tensor, ctl: torch.Tensor, stats: torch.Tensor, slot_stats: torch.Tensor,
                    nan_flag: torch.Tensor, phase_ns: Optional[torch.Tensor] = None,
                    num_sms: Optional[int] = None) -> None:
    """Apply the micro-batches staged in ``stage`` (slot j at byte ``j * slot_bytes``: ``counts[j]`` records,
    ``formats[j]`` 1 = packed64, 0 = int32 users | int32 items | fp32 ratings) in order, in one cooperative
    launch (csrc/fps_mf_window.cu).  Conflict-free runs of micro-batches are applied item-major with the tables
    bitwise equal to one :func:`mf_sgd_fused` launch per micro-batch.  ``slots``: int64 ``[>= n, rows]``
    filled with -1, left so; ``user_bits``: int32 bitmap over the user rows; ``ctl``: int32 ``[2 * WINDOW_MAX]``;
    ``slot_stats``: float32 ``[>= n, 2]`` receives each micro-batch's (sum sq err, updates), ``stats`` the totals
    (``DeviceOnlineMF`` reads only the totals; the per-micro-batch sums serve callers that report per micro-batch).
    ``phase_ns``: optional int64 ``[4]``; the drain adds its build and apply nanoseconds to ``[0]`` and ``[1]`` and
    the windows it applied to ``[2]`` (``[3]`` is scratch).  ``num_sms``: SMs the cooperative grid is sized for
    (default: the device's); a smaller grid runs more rounds of every grid-stride loop and computes the same
    tables bitwise, since each item's chain is applied by one lane-group in micro-batch order."""
    n = len(counts)
    if not 0 < n <= WINDOW_MAX or len(formats) != n:
        raise ValueError(f"1..{WINDOW_MAX} staged micro-batches expected, got {n}")
    if num_sms is not None and int(num_sms) < 1:
        raise ValueError(f"num_sms must be >= 1, got {num_sms!r}")
    for t, name in ((stage, "stage"), (user_table, "user_table"), (item_table, "item_table"), (slots, "slots"),
                    (user_bits, "user_bits"), (ctl, "ctl"), (stats, "stats"), (slot_stats, "slot_stats"),
                    (nan_flag, "nan_flag")):
        _req(t, name)
    if user_table.shape[1] != item_table.shape[1]:
        raise ValueError("user table stride must equal item table stride")
    if user_bits.numel() * 32 < user_table.shape[0] or slots.numel() < n * item_table.shape[0]:
        raise ValueError("user bitmap or slot table too small")
    if slot_stats.numel() < 2 * n or ctl.numel() < 2 * WINDOW_MAX:
        raise ValueError("slot_stats / ctl too small")
    a = WinArgsC()
    a.stage = stage.data_ptr(); a.slot_bytes = int(slot_bytes)
    for j in range(n):
        a.n[j] = int(counts[j]); a.fmt[j] = int(formats[j])
    a.n_slots = n; a.err_mode = int(err_mode); a.lr = float(lr); a.stride = int(item_table.shape[1])
    a.user_table = user_table.data_ptr(); a.item_table = item_table.data_ptr(); a.rows = int(item_table.shape[0])
    a.slots = slots.data_ptr(); a.user_bits = user_bits.data_ptr(); a.bm_words = user_bits.numel()
    a.ctl = ctl.data_ptr(); a.stats = stats.data_ptr(); a.slot_stats = slot_stats.data_ptr()
    a.nan_flag = nan_flag.data_ptr()
    if phase_ns is not None:
        _req(phase_ns, "phase_ns", torch.int64)
        if phase_ns.numel() < 4:
            raise ValueError("phase_ns too small")
        a.phase_ns = phase_ns.data_ptr()
    rv = os.environ.get("FPS_MF_WINDOW_VARIANT")
    if rv is not None:
        lib().fps_set_mf_window_variant(int(rv))
    if num_sms is None:
        num_sms = sm_count(stage.device.index)
    _check(lib().fps_mf_window_drain(C.byref(a), int(num_sms), _stream()), "mf_window_drain")
    _bump()


class BprArgsC(C.Structure):
    """Mirror of ``struct BprArgs`` (csrc/fps_mf_args.cuh)."""

    _fields_ = [
        ("users", C.c_void_p), ("items", C.c_void_p), ("ratings", C.c_void_p), ("negatives", C.c_void_p),
        ("n_pos", C.c_longlong), ("n_neg", C.c_int), ("format", C.c_int),
        ("num_items", C.c_longlong), ("seed", C.c_ulonglong), ("step", C.c_ulonglong),
        ("lr", C.c_float), ("reg", C.c_float),
        ("anchor_table", C.c_void_p), ("anchor_div", C.c_int), ("anchor_shift", C.c_int),
        ("anchor_sharded", C.c_int), ("cand_sharded", C.c_int), ("anchor_tab", ShardTableC),
        ("cand_table", C.c_void_p), ("cand_div", C.c_int), ("cand_shift", C.c_int), ("cand_tab", ShardTableC),
        ("use_push_tab", C.c_int), ("stride", C.c_int), ("push_tab", ShardTableC),
        ("stats", C.c_void_p), ("nan_flag", C.c_void_p), ("reserve_total", C.c_int), ("pad_", C.c_int),
        ("anchor_acc_tab", ShardTableC), ("cand_acc", ShardTableC), ("anchor_acc", C.c_void_p),
        ("rank_items", C.c_longlong), ("margin", C.c_float), ("pad2_", C.c_int),
    ]


def _pairwise_args(users, items, ratings, anchor_table, cand_table, lr, reg, negatives, n_neg, num_items, seed,
                   step, anchor_div, cand_div, stats, n_stats, nan_flag, push_tab, reserve_total):
    """The validated :class:`BprArgsC` of :func:`mf_bpr_fused` / :func:`mf_warp_fused`, and the id width of the
    records (:func:`_records`)."""
    packed, id_bytes = _records(users, items, ratings)
    id_dtype = torch.int32 if id_bytes == 4 else torch.int64
    n_pos = users.numel()
    a = BprArgsC()
    strides = []
    for name, tab, div in (("anchor", anchor_table, anchor_div), ("cand", cand_table, cand_div)):
        if isinstance(tab, ShardTableC):
            setattr(a, f"{name}_tab", tab); setattr(a, f"{name}_sharded", 1)
            strides.append(int(tab.stride))
        else:
            _req(tab, f"{name}_table", torch.float32)
            setattr(a, f"{name}_table", tab.data_ptr())
            setattr(a, f"{name}_div", int(div)); setattr(a, f"{name}_shift", log2_or_neg(int(div)))
            strides.append(int(tab.shape[1]))
    if strides[0] != strides[1]:
        raise ValueError("anchor table stride must equal candidate table stride")
    a.stride = strides[0]
    if push_tab is not None:
        if not a.cand_sharded:
            raise ValueError("push_tab needs a ShardTable cand_table")
        if int(push_tab.stride) != a.stride:
            raise ValueError("push table stride must equal candidate table stride")
        a.push_tab = push_tab; a.use_push_tab = 1
    if negatives is not None:
        _req(negatives, "negatives", id_dtype)
        if negatives.dim() != 2 or negatives.shape[0] != n_pos:
            raise ValueError(f"negatives must be [{n_pos}, n]")
        a.negatives = negatives.data_ptr(); a.n_neg = int(negatives.shape[1])
    else:
        if int(n_neg) < 1:
            raise ValueError("n_neg must be >= 1 when negatives are sampled")
        if int(num_items) < 2:
            raise ValueError(f"sampled negatives need num_items >= 2, got {num_items}")
        a.n_neg = int(n_neg)
    if stats is not None:
        _req(stats, "stats", torch.float32)
        if stats.numel() < n_stats:
            raise ValueError(f"stats must hold {n_stats} floats")
        a.stats = stats.data_ptr()
    if nan_flag is not None:
        _req(nan_flag, "nan_flag", torch.int32)
        a.nan_flag = nan_flag.data_ptr()
    a.users = users.data_ptr()
    a.items = None if packed else items.data_ptr()
    a.ratings = None if packed else ratings.data_ptr()
    a.format = 1 if packed else 0
    a.n_pos = n_pos; a.num_items = int(max(num_items, 1))
    a.seed = seed & (2**64 - 1); a.step = int(step)
    a.lr = float(lr); a.reg = float(reg); a.reserve_total = int(reserve_total)
    return a, id_bytes


def mf_bpr_fused(users: torch.Tensor, items: Optional[torch.Tensor], ratings: Optional[torch.Tensor],
                 anchor_table, cand_table, lr: float, reg: float = 0.0, *,
                 negatives: Optional[torch.Tensor] = None, n_neg: int = 1, num_items: int = 0,
                 seed: int = 0, step: int = 0, anchor_div: int = 1, cand_div: int = 1,
                 stats: Optional[torch.Tensor] = None, nan_flag: Optional[torch.Tensor] = None,
                 max_inflight_rows: int = 0, push_tab: Optional[ShardTableC] = None,
                 reserve_total: int = 0, anchor_acc=None, cand_acc: Optional[ShardTableC] = None) -> None:
    """Fused pairwise (BPR) pull + SGD + push, one ``(anchor, positive, negative)`` triple per update
    (csrc/fps_mf_bpr.cu).  ``users`` are the anchor ids, ``items`` the positive candidates; records with
    ``rating <= 0`` are skipped.  ``items=None``: ``users`` holds packed64 records (:func:`pack_ratings`).

    ``anchor_table`` / ``cand_table``: a worker-local ``[rows, stride]`` float32 tensor (row of id =
    ``id // anchor_div`` / ``id // cand_div``) or a :class:`ShardTableC`.  ``push_tab`` (with a
    ShardTable ``cand_table``) receives the candidate deltas instead of ``cand_table``.

    ``negatives``: ``[n_pos, n]`` ids of the same dtype as ``users`` (int32 for packed64), ``-1`` voids a
    triple.  Without it ``n_neg`` negatives per positive are drawn in the kernel, uniform over
    ``[0, num_items)`` and never the positive.  ``stats`` (float32 ``[3]``) accumulates the softplus loss
    sum, the number of triples and the number with ``x > 0``.  ``max_inflight_rows`` caps the grid so that
    at most that many rows are being pulled at once (3 per lane-group).  ``reserve_total``: CTA slots
    the grid leaves free for a kernel running next to it (the replica exchange).

    ``cand_acc`` / ``anchor_acc``: row-wise AdaGrad instead of SGD (DESIGN §2.10).  ``cand_acc`` is a stride-1
    :class:`ShardTableC` of candidate accumulators (``cand_table`` must then be a ShardTableC, without
    ``push_tab``); ``anchor_acc`` a float32 ``[rows]`` tensor, or a stride-1 ShardTableC when ``anchor_table``
    is one."""
    a, id_bytes = _pairwise_args(users, items, ratings, anchor_table, cand_table, lr, reg, negatives, n_neg, num_items,
                                 seed, step, anchor_div, cand_div, stats, 3, nan_flag, push_tab, reserve_total)
    if cand_acc is not None:
        if not a.cand_sharded or push_tab is not None:
            raise ValueError("row-wise AdaGrad needs a ShardTableC cand_table and no push_tab")
        if int(cand_acc.stride) != 1:
            raise ValueError("cand_acc must be a stride-1 accumulator table")
        a.cand_acc = cand_acc
        _set_row_acc(a, "anchor", anchor_acc, anchor_table, bool(a.anchor_sharded))
    elif anchor_acc is not None:
        raise ValueError("anchor_acc needs cand_acc")
    _check(lib().fps_mf_bpr_fused(C.byref(a), id_bytes, int(max_inflight_rows),
                                  sm_count(users.device.index), _stream()), "mf_bpr_fused")
    _bump()


WARP_TRIAL_BLOCKS = (1, 2, 4, 8)   # candidates a lane-group pulls at once in fps_mf_warp (0 = per-geometry default)


def mf_warp_fused(users: torch.Tensor, items: Optional[torch.Tensor], ratings: Optional[torch.Tensor],
                  anchor_table, cand_table, lr: float, reg: float = 0.0, *, margin: float = 1.0,
                  rank_items: int = 0, negatives: Optional[torch.Tensor] = None, n_neg: int = 1,
                  num_items: int = 0, seed: int = 0, step: int = 0, anchor_div: int = 1, cand_div: int = 1,
                  stats: Optional[torch.Tensor] = None, nan_flag: Optional[torch.Tensor] = None,
                  max_inflight_rows: int = 0, push_tab: Optional[ShardTableC] = None, reserve_total: int = 0,
                  trial_block: int = 0) -> None:
    """Fused WARP (Weighted Approximate-Rank Pairwise) step (csrc/fps_mf_warp.cu, DESIGN §2.12): for each positive
    ``(anchor, item)`` with ``rating > 0``, its candidates are examined in order until one violates
    ``u . (v_i - v_j) < margin``; with ``n`` the live candidates examined up to it, the triple gets one hinge update
    with ``g = lr * ln(max(1, (rank_items - 1) // n))``.  No violator: nothing is written.  The arguments are those
    of :func:`mf_bpr_fused`: ``negatives`` ``[n_pos, T]`` are the candidates in order (``-1`` or the positive = void),
    else ``T = n_neg`` are drawn in the kernel, candidate ``t`` bitwise BPR's negative ``t``.

    ``rank_items``: the ``N`` of the rank estimate (``0`` = ``num_items``).  ``stats`` (float32 ``[4]``) accumulates
    ``sum L * (margin - x)`` over the updated positives, the positives updated, the live candidates examined and the
    positives considered.  ``max_inflight_rows`` caps the grid at ``2 + trial_block`` rows per lane-group.
    ``trial_block`` (one of :data:`WARP_TRIAL_BLOCKS`, ``0`` = the default of the row width) changes the speed only:
    the result is bitwise the same for all."""
    if not math.isfinite(float(margin)):
        raise ValueError(f"margin must be finite, got {margin!r}")
    if int(trial_block) not in (0,) + WARP_TRIAL_BLOCKS:
        raise ValueError(f"trial_block must be 0 or one of {WARP_TRIAL_BLOCKS}, got {trial_block!r}")
    a, id_bytes = _pairwise_args(users, items, ratings, anchor_table, cand_table, lr, reg, negatives, n_neg, num_items,
                                 seed, step, anchor_div, cand_div, stats, 4, nan_flag, push_tab, reserve_total)
    a.margin = float(margin)
    a.rank_items = int(rank_items) if int(rank_items) > 0 else int(a.num_items)
    _check(lib().fps_mf_warp_fused(C.byref(a), id_bytes, int(trial_block),
                                   int(max_inflight_rows), sm_count(users.device.index), _stream()), "mf_warp_fused")
    _bump()


def init_rows_f64(rows: torch.Tensor, dim: int, shard: int, num_shards: int, mode: int, div: int, seed: int,
                  lo: float, hi: float) -> None:
    """Philox init-by-id of fp64 rows ``[n, stride_doubles]`` (53-bit uniforms)."""
    _req(rows, "rows", torch.float64)
    _check(lib().fps_init_rows_f64(C.c_void_p(rows.data_ptr()), C.c_longlong(rows.shape[0]), int(dim),
                                   int(rows.shape[1]), int(shard), int(num_shards), int(mode), C.c_longlong(div),
                                   C.c_ulonglong(seed & (2**64 - 1)), C.c_double(lo), C.c_double(hi), _stream()),
           "init_rows_f64")
    _bump()


def mf_sgd_fused_f64(users: torch.Tensor, items: Optional[torch.Tensor], ratings: Optional[torch.Tensor],
                     user_table: torch.Tensor, user_div: int, item_tab: ShardTableC, lr: float,
                     err_mode: int = 0, stats: Optional[torch.Tensor] = None,
                     nan_flag: Optional[torch.Tensor] = None) -> None:
    """fp64 fused pull + SGD + push (csrc/fps_mf_f64.cu): ``user_table`` is float64 ``[n, k_pad]``, the shards
    of ``item_tab`` hold doubles (stride counted in 4-byte cells).  ``items=None``: packed64 records.
    ``err_mode`` as for :func:`mf_sgd_fused`."""
    _check_err_mode(err_mode)
    packed, id_bytes = _records(users, items, ratings)
    _req(user_table, "user_table", torch.float64)
    if user_table.shape[1] * 2 != item_tab.stride:
        raise ValueError("user table width must equal the item row width")
    a = MfArgsC()
    a.users = users.data_ptr()
    a.items = None if packed else items.data_ptr()
    a.ratings = None if packed else ratings.data_ptr()
    a.format = 1 if packed else 0
    a.n_pos = users.numel(); a.num_items = 1
    a.user_table = user_table.data_ptr(); a.user_div = int(user_div); a.user_shift = log2_or_neg(int(user_div))
    a.lr = float(lr); a.err_mode = int(err_mode)
    a.stats = stats.data_ptr() if stats is not None else None
    a.nan_flag = nan_flag.data_ptr() if nan_flag is not None else None
    a.item_tab = item_tab
    _check(lib().fps_mf_sgd_fused_f64(C.byref(a), id_bytes,
                                      sm_count(users.device.index), _stream()), "mf_sgd_fused_f64")
    _bump()


class NegArgsC(C.Structure):
    """Mirror of ``struct NegArgs`` (csrc/fps_sampler.cu)."""

    _fields_ = [
        ("users", C.c_void_p), ("items", C.c_void_p), ("ratings", C.c_void_p),
        ("n_pos", C.c_longlong), ("neg_rate", C.c_int), ("format", C.c_int),
        ("num_items", C.c_longlong), ("seed", C.c_ulonglong), ("step", C.c_ulonglong),
        ("seen", C.c_void_p), ("seen_pos", C.c_void_p), ("memory", C.c_int), ("user_div", C.c_int),
        ("max_tries", C.c_int), ("pad_", C.c_int),
        ("out_users", C.c_void_p), ("out_items", C.c_void_p), ("out_ratings", C.c_void_p),
    ]


def neg_sample(users: torch.Tensor, items: Optional[torch.Tensor], ratings: Optional[torch.Tensor],
               neg_rate: int, num_items: int, seen: torch.Tensor, seen_pos: torch.Tensor, user_div: int,
               seed: int = 0, step: int = 0, max_tries: int = 32):
    """K5: expand a micro-batch with ``neg_rate`` rating-0 negatives per rating, none of which is in
    the user's recent-items memory ``seen`` ([n_local_users, userMemory] int32 ring, updated in
    place).  Returns ``(users, items, ratings)`` int32/int32/float32 of length ``n*(1+neg_rate)``;
    a negative that could not be found in ``max_tries`` draws has user == -1 (skipped downstream).
    ``items=None``: ``users`` holds packed64 records."""
    packed, id_bytes = _records(users, items, ratings)
    _req(seen, "seen", torch.int32); _req(seen_pos, "seen_pos", torch.int32)
    n = users.numel()
    per = 1 + int(neg_rate)
    dev = users.device
    ou = torch.empty(n * per, dtype=torch.int32, device=dev)
    oi = torch.empty(n * per, dtype=torch.int32, device=dev)
    orat = torch.empty(n * per, dtype=torch.float32, device=dev)
    a = NegArgsC()
    a.users = users.data_ptr()
    a.items = None if packed else items.data_ptr()
    a.ratings = None if packed else ratings.data_ptr()
    a.n_pos = n; a.neg_rate = int(neg_rate); a.format = 1 if packed else 0
    a.num_items = int(max(num_items, 1)); a.seed = seed & (2**64 - 1); a.step = int(step)
    a.seen = seen.data_ptr(); a.seen_pos = seen_pos.data_ptr(); a.memory = int(seen.shape[1])
    a.user_div = int(user_div); a.max_tries = int(max_tries)
    a.out_users = ou.data_ptr(); a.out_items = oi.data_ptr(); a.out_ratings = orat.data_ptr()
    _check(lib().fps_neg_sample(C.byref(a), id_bytes,
                                sm_count(dev.index), _stream()), "neg_sample")
    _bump()
    return ou, oi, orat


class NegDomainArgsC(C.Structure):
    """Mirror of ``struct NegDomainArgs`` (csrc/fps_negatives.cu)."""

    _fields_ = [
        ("users", C.c_void_p), ("items", C.c_void_p), ("ratings", C.c_void_p),
        ("n_pos", C.c_longlong), ("neg_rate", C.c_int), ("format", C.c_int),
        ("seed", C.c_ulonglong), ("step", C.c_ulonglong), ("max_tries", C.c_int),
        ("memory", C.c_int), ("seen", C.c_void_p), ("seen_pos", C.c_void_p), ("user_div", C.c_int),
        ("cta_cap", C.c_int), ("num_items", C.c_longlong), ("order", C.c_void_p), ("count", C.c_void_p),
        ("first_pos", C.c_void_p), ("scratch", C.c_void_p), ("cta_new", C.c_void_p),
        ("cdf", C.c_void_p), ("vocab", C.c_longlong), ("last_nonzero", C.c_longlong),
        ("out_users", C.c_void_p), ("out_items", C.c_void_p), ("out_ratings", C.c_void_p),
    ]


def _neg_domain_args(users, items, ratings, neg_rate: int, seed: int, step: int, max_tries: int):
    packed, id_bytes = _records(users, items, ratings)
    if int(neg_rate) < 0:
        raise ValueError("neg_rate must be >= 0")
    n, per, dev = users.numel(), 1 + int(neg_rate), users.device
    out = (torch.empty(n * per, dtype=torch.int32, device=dev), torch.empty(n * per, dtype=torch.int32, device=dev),
           torch.empty(n * per, dtype=torch.float32, device=dev))
    a = NegDomainArgsC()
    a.users = users.data_ptr()
    a.items = None if packed else items.data_ptr()
    a.ratings = None if packed else ratings.data_ptr()
    a.n_pos = n; a.neg_rate = int(neg_rate); a.format = 1 if packed else 0
    a.seed = seed & (2**64 - 1); a.step = int(step); a.max_tries = int(max_tries)
    a.out_users, a.out_items, a.out_ratings = (t.data_ptr() for t in out)
    return a, out, id_bytes


def seen_registry(num_items: int, device) -> tuple:
    """Empty seen-items registry of :func:`neg_sample_seen` for ids ``[0, num_items)``: ``(order, count,
    first_pos)`` = int32 ``[num_items]`` ids in first-occurrence order, int32 ``[1]`` how many, and int32
    ``[num_items]`` per-item state (``-1`` registered, ``2**31 - 1`` not seen)."""
    n = max(int(num_items), 1)
    return (torch.zeros(n, dtype=torch.int32, device=device), torch.zeros(1, dtype=torch.int32, device=device),
            torch.full((n,), 2**31 - 1, dtype=torch.int32, device=device))


def neg_sample_seen(users: torch.Tensor, items: Optional[torch.Tensor], ratings: Optional[torch.Tensor],
                    neg_rate: int, registry: tuple, seen: Optional[torch.Tensor] = None,
                    seen_pos: Optional[torch.Tensor] = None, user_div: int = 1, seed: int = 0, step: int = 0,
                    max_tries: int = 32):
    """:func:`neg_sample` with negatives drawn from the items this worker has seen so far
    (PSOnlineMatrixFactorizationWorker.scala:61-88; csrc/fps_negatives.cu).  ``registry`` (from
    :func:`seen_registry`) holds them in first-occurrence order and is advanced past the micro-batch in place.

    Record ``p`` draws from ``D_p`` = the registry before the batch plus the batch's items first seen at
    positions ``< p`` (its own first-seen item is not in its domain), ``max(0, min(|D_p| - |ring_p|, neg_rate))``
    negatives, each uniform over ``D_p`` and none the positive or in the user's recent-items ring ``seen``
    (``[n_local_users, userMemory]`` int32, updated in place as :func:`neg_sample` does; ``None`` = no ring,
    ``|ring_p| = 0``).  Returns ``(users, items, ratings)`` int32/int32/float32 of length ``n*(1+neg_rate)``:
    the positive, then its negatives; the slots not drawn, and draws that found nothing admissible in
    ``max_tries`` tries, have user == -1.  ``items=None``: ``users`` holds packed64 records.  Item ids outside
    ``[0, num_items)`` are never registered.  The output depends on ``seed``, ``step`` and the stream only."""
    a, out, id_bytes = _neg_domain_args(users, items, ratings, neg_rate, seed, step, max_tries)
    order, count, first_pos = registry
    _req(order, "order", torch.int32); _req(count, "count", torch.int32); _req(first_pos, "first_pos", torch.int32)
    if order.numel() != first_pos.numel():
        raise ValueError("registry order and first_pos must have the same length")
    if seen is not None:
        _req(seen, "seen", torch.int32); _req(seen_pos, "seen_pos", torch.int32)
        a.seen, a.seen_pos, a.memory = seen.data_ptr(), seen_pos.data_ptr(), int(seen.shape[1])
    n, dev = users.numel(), users.device
    cta_cap = sm_count(dev.index) * 8
    scratch = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    cta_new = torch.empty(cta_cap, dtype=torch.int32, device=dev)
    a.user_div = int(user_div); a.cta_cap = cta_cap; a.num_items = order.numel()
    a.order, a.count, a.first_pos = order.data_ptr(), count.data_ptr(), first_pos.data_ptr()
    a.scratch, a.cta_new = scratch.data_ptr(), cta_new.data_ptr()
    _check(lib().fps_neg_sample_seen(C.byref(a), id_bytes, sm_count(dev.index), _stream()), "neg_sample_seen")
    _bump()
    return out


def noise_cdf(counts: torch.Tensor, power: float) -> torch.Tensor:
    """fp64 inverse CDF ``cdf[i] = sum_{j <= i} w_j`` of the noise weights ``w = counts ** power`` (``w = 0``
    where ``counts == 0``), built on the device by left-to-right sums, so a word of weight 0 has exactly its
    predecessor's prefix.  ``counts``: float64 CUDA tensor of non-negative finite values."""
    _req(counts, "counts", torch.float64)
    n = counts.numel()
    cdf = torch.empty(n, dtype=torch.float64, device=counts.device)
    totals = torch.empty(-(-n // 256), dtype=torch.float64, device=counts.device)
    _check(lib().fps_noise_cdf(C.c_void_p(counts.data_ptr()), C.c_longlong(n), C.c_double(float(power)),
                               C.c_void_p(cdf.data_ptr()), C.c_void_p(totals.data_ptr()), _stream()), "noise_cdf")
    _bump(3)
    return cdf


def neg_sample_noise(users: torch.Tensor, items: Optional[torch.Tensor], ratings: Optional[torch.Tensor],
                     neg_rate: int, cdf: torch.Tensor, last_nonzero: int, seed: int = 0, step: int = 0,
                     max_tries: int = 32):
    """:func:`neg_sample` with negatives drawn from fixed weights (skip-gram's unigram noise;
    csrc/fps_negatives.cu): a 53-bit Philox uniform, scaled by the total weight, then an upper-bound binary
    search of ``cdf`` (:func:`noise_cdf`), rejecting the positive ``items[p]``.  ``last_nonzero``: the last id
    of positive weight.  Returns ``(users, items, ratings)`` int32/int32/float32 of length ``n*(1+neg_rate)``;
    a negative that was the positive in all ``max_tries`` draws has user == -1.  Words of weight 0 are never
    drawn.  ``items=None``: ``users`` holds packed64 records."""
    a, out, id_bytes = _neg_domain_args(users, items, ratings, neg_rate, seed, step, max_tries)
    _req(cdf, "cdf", torch.float64)
    if not 0 <= int(last_nonzero) < cdf.numel():
        raise ValueError("last_nonzero must index cdf")
    a.cdf, a.vocab, a.last_nonzero = cdf.data_ptr(), cdf.numel(), int(last_nonzero)
    _check(lib().fps_neg_sample_noise(C.byref(a), id_bytes, sm_count(users.device.index), _stream()),
           "neg_sample_noise")
    _bump()
    return out


class W2vArgsC(C.Structure):
    """Mirror of ``struct W2vArgs`` (csrc/fps_w2v_window.cu)."""

    _fields_ = [
        ("tokens", C.c_void_p), ("n_tokens", C.c_longlong), ("vocab", C.c_longlong), ("keep_p", C.c_void_p),
        ("seed", C.c_ulonglong), ("step", C.c_ulonglong),
        ("seq", C.c_void_p), ("pos", C.c_void_p), ("n_comp", C.c_void_p), ("cta_cnt", C.c_void_p),
        ("cta_cap", C.c_int), ("stride", C.c_int), ("token_stats", C.c_void_p),
        ("w_in", ShardTableC), ("w_out", ShardTableC),
        ("window", C.c_int), ("negative", C.c_int), ("max_tries", C.c_int), ("lr", C.c_float),
        ("cdf", C.c_void_p), ("last_nonzero", C.c_longlong), ("stats", C.c_void_p), ("nan_flag", C.c_void_p),
        ("reserve_total", C.c_int), ("cbow", C.c_int),
    ]


def w2v_scratch(n_tokens: int, device) -> tuple:
    """Device scratch of :func:`w2v_subsample` for calls of up to ``n_tokens`` tokens: ``(seq, pos, n_comp,
    cta_cnt)`` int32 ``[n_tokens]``, ``[n_tokens]``, ``[1]`` and ``[8 * SMs]``.  Reusable from call to call."""
    n = max(int(n_tokens), 1)
    dev = torch.device(device)
    return (torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
            torch.zeros(1, dtype=torch.int32, device=dev),
            torch.empty(sm_count(dev.index) * 8, dtype=torch.int32, device=dev))


def w2v_subsample(tokens: torch.Tensor, vocab: int, keep_p: Optional[torch.Tensor] = None, *, seed: int = 0,
                  step: int = 0, token_stats: Optional[torch.Tensor] = None, scratch: Optional[tuple] = None) -> tuple:
    """Frequent-word subsampling and compaction of one token call (csrc/fps_w2v_window.cu, DESIGN §2.13), in one
    cooperative launch with no host synchronisation.

    ``tokens``: 1-D int32 or int64 CUDA tensor; ``-1`` marks a sentence boundary, and so does any other id outside
    ``[0, vocab)`` (counted as dropped).  Word ``w`` at call position ``i`` is kept iff the 53-bit Philox uniform
    keyed ``(i, 0, 0, step; seed)`` is ``< keep_p[w]`` (float64 ``[vocab]``; ``None`` keeps every word).  The kept
    words and every boundary, in order, form the compacted sequence.

    Returns ``(seq, pos, n_comp)``: int32 compacted sequence (``-1`` = boundary), the call position of each
    entry, and an int32 ``[1]`` device tensor holding the compacted length; only the first ``n_comp`` entries are
    written.  ``scratch`` (:func:`w2v_scratch`, large enough) is used instead of fresh buffers.  ``token_stats``
    (int64 ``[4]``) accumulates the tokens, the kept words and, at index 3, the dropped ids."""
    _req(tokens, "tokens")
    idb = _id_bytes(tokens)
    n = tokens.numel()
    if scratch is None:
        scratch = w2v_scratch(n, tokens.device)
    seq, pos, n_comp, cta_cnt = scratch
    for t, name in ((seq, "seq"), (pos, "pos"), (n_comp, "n_comp"), (cta_cnt, "cta_cnt")):
        _req(t, name, torch.int32)
    if seq.numel() < n or pos.numel() < n:
        raise ValueError(f"scratch holds {seq.numel()} entries, the call has {n} tokens")
    if n >= 2**31 - 1:
        raise ValueError("a token call must hold fewer than 2**31 - 1 tokens")
    a = W2vArgsC()
    a.tokens, a.n_tokens, a.vocab = tokens.data_ptr(), n, int(vocab)
    if keep_p is not None:
        _req(keep_p, "keep_p", torch.float64)
        if keep_p.numel() != int(vocab):
            raise ValueError("keep_p must hold one probability per word")
        a.keep_p = keep_p.data_ptr()
    a.seed = seed & (2**64 - 1); a.step = int(step)
    a.seq, a.pos, a.n_comp, a.cta_cnt = seq.data_ptr(), pos.data_ptr(), n_comp.data_ptr(), cta_cnt.data_ptr()
    a.cta_cap = cta_cnt.numel()
    if token_stats is not None:
        _req(token_stats, "token_stats", torch.int64)
        a.token_stats = token_stats.data_ptr()
    if n == 0:
        n_comp.zero_()
        return seq, pos, n_comp
    _check(lib().fps_w2v_subsample(C.byref(a), idb, sm_count(tokens.device.index), _stream()), "w2v_subsample")
    _bump()
    return seq, pos, n_comp


def w2v_window_fused(seq: torch.Tensor, pos: torch.Tensor, n_comp: torch.Tensor, w_in: ShardTableC,
                     w_out: ShardTableC, lr: float, *, window: int = 5, negative: int = 5, vocab: int,
                     seed: int = 0, step: int = 0, cdf: Optional[torch.Tensor] = None, last_nonzero: int = 0,
                     max_tries: int = 32, stats: Optional[torch.Tensor] = None,
                     token_stats: Optional[torch.Tensor] = None, nan_flag: Optional[torch.Tensor] = None,
                     reserve_total: int = 0, cbow: bool = False) -> None:
    """Fused center-window skip-gram negative-sampling step (csrc/fps_w2v_window.cu, DESIGN §2.13) over the
    compacted sequence of :func:`w2v_subsample`; one lane-group per kept center, the grid sized without reading
    ``n_comp`` on the host.  ``cbow=True`` trains CBOW instead (DESIGN §2.14), described below.

    The center at call position ``i`` draws a radius ``r = 1 + h mod window`` (``h`` keyed ``(i, 1, 0, step)``);
    its contexts are the entries up to ``r`` positions to either side, stopping at a boundary, in increasing
    position.  Each context ``q`` trains the context word (label 1), then ``negative`` noise words (label 0),
    uniform over ``[0, vocab)`` or from ``cdf`` (:func:`noise_cdf`, ``last_nonzero`` its last word of positive
    weight), keyed ``(i, 2 | slot << 8, j | try << 8, step)``; a draw equal to the context word is redrawn up to
    ``max_tries`` times, then voided.  With ``u = W_in[center]`` as pulled and ``D = 0``, per target
    ``d = (u + D) . v``, ``g = lr (label - sigmoid(d))``; ``g (u + D)`` is pushed to ``W_out[t]`` at once, ``g v``
    summed into the context's ``e``, and ``D += e`` after the context.  ``D`` is pushed to ``W_in[center]`` once.

    ``w_in`` / ``w_out``: :class:`ShardTableC` of the same stride, at most 512 floats.  ``stats`` (float32 ``[2]``)
    accumulates ``sum -log sigmoid(+-d)`` and the targets trained, ``token_stats`` (int64 ``[4]``) the contexts at
    index 2, ``nan_flag`` is set by a non-finite ``d``.  ``reserve_total``: CTA slots left free for the replica
    exchange running next to it.

    CBOW, per kept center with ``cw >= 1`` contexts (the same windows): ``h`` is the mean of the contexts'
    ``W_in`` rows as pulled.  The targets are the center word (label 1), then ``negative`` noise words drawn as
    those of context slot 0 but rejected against the center word.  Per target ``d = h . v``,
    ``g = lr (label - sigmoid(d))``; ``g h`` is pushed to ``W_out[t]`` at once and ``g v`` summed into ``e``.  ``e``
    is then pushed, unscaled, to ``W_in`` of every context, once per occurrence (word2vec.c's rule: each context row
    moves by ``-lr * cw`` times the loss gradient with respect to that row).  A center with no context trains nothing;
    ``token_stats[2]`` counts the contexts."""
    if not isinstance(cbow, bool):
        raise ValueError(f"cbow must be True or False, got {cbow!r}")
    for t, name in ((seq, "seq"), (pos, "pos"), (n_comp, "n_comp")):
        _req(t, name, torch.int32)
    if int(w_in.stride) != int(w_out.stride):
        raise ValueError("w_in and w_out must have the same stride")
    if not 1 <= int(window) < 2**23:
        raise ValueError(f"window must be in [1, 2**23), got {window!r}")
    if not 0 <= int(negative) <= 255:
        raise ValueError(f"negative must be in [0, 255], got {negative!r}")
    if not 1 <= int(max_tries) < 2**23:
        raise ValueError(f"max_tries must be in [1, 2**23), got {max_tries!r}")
    a = W2vArgsC()
    a.n_tokens, a.vocab = seq.numel(), int(vocab)
    a.seq, a.pos, a.n_comp = seq.data_ptr(), pos.data_ptr(), n_comp.data_ptr()
    a.w_in, a.w_out, a.stride = w_in, w_out, int(w_in.stride)
    a.window, a.negative, a.max_tries, a.lr = int(window), int(negative), int(max_tries), float(lr)
    a.seed = seed & (2**64 - 1); a.step = int(step)
    if cdf is not None:
        _req(cdf, "cdf", torch.float64)
        if cdf.numel() != int(vocab) or not 0 <= int(last_nonzero) < cdf.numel():
            raise ValueError("cdf must hold one prefix per word and last_nonzero must index it")
        a.cdf, a.last_nonzero = cdf.data_ptr(), int(last_nonzero)
    if stats is not None:
        _req(stats, "stats", torch.float32)
        a.stats = stats.data_ptr()
    if token_stats is not None:
        _req(token_stats, "token_stats", torch.int64)
        a.token_stats = token_stats.data_ptr()
    if nan_flag is not None:
        _req(nan_flag, "nan_flag", torch.int32)
        a.nan_flag = nan_flag.data_ptr()
    a.reserve_total, a.cbow = int(reserve_total), int(cbow)
    _check(lib().fps_w2v_window_fused(C.byref(a), sm_count(seq.device.index), _stream()), "w2v_window_fused")
    _bump()


class BucketArgsC(C.Structure):
    """Mirror of ``struct BucketArgs`` (csrc/fps_bucket.cu)."""

    _fields_ = [
        ("users", C.c_void_p), ("items", C.c_void_p), ("ratings", C.c_void_p), ("n", C.c_longlong),
        ("format", C.c_int), ("id_bytes", C.c_int), ("shift", C.c_int), ("n_buckets", C.c_int),
        ("scratch", C.c_void_p), ("out_users", C.c_void_p), ("out_items", C.c_void_p),
        ("out_ratings", C.c_void_p),
        ("rps", C.c_longlong), ("num_shards", C.c_int), ("shard_shift", C.c_int),
        ("pending", C.c_void_p),
    ]


BUCKET_MAX = 64


def bucket_by_item(users: torch.Tensor, items: Optional[torch.Tensor], ratings: Optional[torch.Tensor],
                   shift: int, n_buckets: int, scratch: torch.Tensor, num_shards: int = 1,
                   rows_per_shard: int = 0, pending: Optional[torch.Tensor] = None):
    """Reorder a micro-batch by ``row(item) >> shift`` (L2 blocking of the item table, one cooperative
    kernel in csrc/fps_bucket.cu); ``row`` is the row of the owner-major table the fused kernel reads
    (``(item % num_shards) * rows_per_shard + item // num_shards``; plain ``item`` for one shard).
    ``items=None``: ``users`` holds packed64 records.  ``scratch``: int32 device tensor of
    ``2 * BUCKET_MAX`` elements.  ``pending``: optional int64 ``[num_shards]`` device counters that
    receive the number of records per destination shard (feed of the device-side flush policy).
    Returns the reordered ``(users, items, ratings)`` (new tensors).  ``num_shards`` outside
    ``[1, FPS_MAX_SHARDS]`` is refused before any CUDA check."""
    _shard_count(num_shards)
    packed, id_bytes = _records(users, items, ratings)
    _req(scratch, "scratch", torch.int32)
    a = BucketArgsC()
    a.users = users.data_ptr(); a.n = users.numel()
    ou = torch.empty_like(users)
    oi = orat = None
    a.out_users = ou.data_ptr()
    a.format = 1 if packed else 0; a.id_bytes = id_bytes
    if not packed:
        oi, orat = torch.empty_like(items), torch.empty_like(ratings)
        a.items = items.data_ptr(); a.ratings = ratings.data_ptr()
        a.out_items = oi.data_ptr(); a.out_ratings = orat.data_ptr()
    a.shift = int(shift); a.n_buckets = int(n_buckets); a.scratch = scratch.data_ptr()
    a.num_shards = int(num_shards); a.shard_shift = log2_or_neg(a.num_shards)
    a.rps = int(rows_per_shard)
    if pending is not None:
        _req(pending, "pending", torch.int64)
        a.pending = pending.data_ptr()
    _check(lib().fps_bucket_by_item(C.byref(a), sm_count(users.device.index), _stream()), "bucket_by_item")
    _bump()
    return ou, oi, orat


PACK_USER_BITS, PACK_ITEM_BITS = 26, 22
PACK_ITEM_SHIFT = 16                                 # below it: the fp16 rating
PACK_USER_SHIFT = PACK_ITEM_SHIFT + PACK_ITEM_BITS   # 38 (csrc/fps_common.cuh FPS_REC_*)


def pack_ratings(users: torch.Tensor, items: torch.Tensor, ratings: torch.Tensor) -> torch.Tensor:
    """Pack ``(user, item, rating)`` into one int64 per rating: ``user:26 | item:22 | fp16 rating:16``
    -- 8 bytes per update over PCIe instead of 12.  Limits: user < 2^26, item < 2^22."""
    if int(users.max()) >= 1 << PACK_USER_BITS or int(items.max()) >= 1 << PACK_ITEM_BITS:
        raise ValueError("ids exceed the packed64 record range (user < 2^26, item < 2^22)")
    r16 = ratings.to(torch.float16).view(torch.int16).to(torch.int64) & 0xFFFF
    return (users.to(torch.int64) << PACK_USER_SHIFT) | (items.to(torch.int64) << PACK_ITEM_SHIFT) | r16


def pull_gather(tab: ShardTableC, ids: torch.Tensor, out: torch.Tensor, touch: bool = False,
                max_inflight_rows: int = 0, credits: Optional[torch.Tensor] = None) -> None:
    """``out[i] = table[ids[i]]`` (one-sided gather, K1).  Pull limiter: ``credits`` (int32 ``[2]``
    device tensor, ``credits[0]`` = pullLimit) is the device-side credit counter -- a lane-group takes a
    credit before it touches the owner and returns it when the answer is stored; ``credits[1]`` counts
    stalls.  Without it ``max_inflight_rows`` caps the grid (static limiter).  An ``out`` whose width is a
    multiple of 4 is stored in 16-byte vectors and must start on a 16-byte boundary (``ValueError`` otherwise)."""
    _req(ids, "ids"); _req(out, "out", torch.float32)
    assert out.shape[0] == ids.numel() and out.shape[1] <= tab.stride
    _req_vec4(out, "out")
    if credits is not None:
        _req(credits, "credits", torch.int32)
    _check(lib().fps_pull_gather(C.byref(tab), C.c_void_p(ids.data_ptr()), _id_bytes(ids),
                                 C.c_longlong(ids.numel()), C.c_void_p(out.data_ptr()),
                                 int(out.shape[1]), int(bool(touch)), sm_count(ids.device.index),
                                 int(max_inflight_rows),
                                 C.c_void_p(credits.data_ptr() if credits is not None else None),
                                 _stream()), "pull_gather")
    _bump()


def push_add(tab: ShardTableC, ids: torch.Tensor, delta: torch.Tensor, scale: float = 1.0,
             touch: bool = False, nan_flag: Optional[torch.Tensor] = None) -> None:
    """``table[ids[i]] += scale * delta[i]`` (K2).  A ``delta`` whose width is a multiple of 4 is read in 16-byte
    vectors and must start on a 16-byte boundary (``ValueError`` otherwise)."""
    _req(ids, "ids"); _req(delta, "delta", torch.float32)
    assert delta.shape[0] == ids.numel() and delta.shape[1] <= tab.stride
    _req_vec4(delta, "delta")
    _check(lib().fps_push_add(C.byref(tab), C.c_void_p(ids.data_ptr()), _id_bytes(ids),
                              C.c_longlong(ids.numel()), C.c_void_p(delta.data_ptr()),
                              int(delta.shape[1]), C.c_float(scale), int(bool(touch)),
                              C.c_void_p(nan_flag.data_ptr() if nan_flag is not None else None),
                              sm_count(ids.device.index), _stream()), "push_add")
    _bump()


def push_assign(tab: ShardTableC, ids: torch.Tensor, values: torch.Tensor, touch: bool = False) -> None:
    """table[ids[i]] = values[i] (model load); one-sided vector stores to the owning shard."""
    _req(ids, "ids"); _req(values, "values", torch.float32)
    assert values.shape[0] == ids.numel() and values.shape[1] <= tab.stride
    _check(lib().fps_push_assign(C.byref(tab), C.c_void_p(ids.data_ptr()), _id_bytes(ids),
                                 C.c_longlong(ids.numel()), C.c_void_p(values.data_ptr()),
                                 int(values.shape[1]), int(bool(touch)), sm_count(ids.device.index),
                                 _stream()), "push_assign")
    _bump()


def push_add_fetch(tab: ShardTableC, ids: torch.Tensor, delta: torch.Tensor) -> torch.Tensor:
    """table[ids[i]] += delta[i] and return the value AFTER each update (the ``(id, newValue)`` PS output
    of SimplePSLogic.scala:16-25); returning atomics, one per element."""
    _req(ids, "ids"); _req(delta, "delta", torch.float32)
    assert delta.shape[0] == ids.numel() and delta.shape[1] <= tab.stride
    out = torch.empty((ids.numel(), tab.dim), dtype=torch.float32, device=ids.device)
    _check(lib().fps_push_add_fetch(C.byref(tab), C.c_void_p(ids.data_ptr()), _id_bytes(ids),
                                    C.c_longlong(ids.numel()), C.c_void_p(delta.data_ptr()),
                                    int(delta.shape[1]), C.c_void_p(out.data_ptr()), int(out.shape[1]),
                                    sm_count(ids.device.index), _stream()), "push_add_fetch")
    _bump()
    return out


def local_table(t: torch.Tensor, dim: int) -> ShardTableC:
    """A single-shard ShardTable over a local ``[rows, stride]`` tensor (row index == id)."""
    _req(t, "table", torch.float32)
    tc = ShardTableC()
    tc.base[0] = t.data_ptr()
    tc.rows_per_shard = t.shape[0]; tc.div = t.shape[0]; tc.num_shards = 1
    tc.dim = int(dim); tc.stride = t.shape[1]; tc.mode = PART_HASH; tc.shard_shift = 0
    return tc


class CtrArgsC(C.Structure):
    """Mirror of ``struct CtrArgs`` (csrc/fps_ctr.cu)."""

    _fields_ = [("rows", C.c_void_p), ("labels", C.c_void_p), ("batch", C.c_longlong), ("fields", C.c_int),
                ("emb", C.c_int), ("stride", C.c_int), ("W1", C.c_void_p), ("W1T", C.c_void_p),
                ("b1", C.c_void_p), ("w2", C.c_void_p), ("b2", C.c_void_p), ("gW1", C.c_void_p),
                ("gb1", C.c_void_p), ("gw2", C.c_void_p), ("gb2", C.c_void_p), ("d_rows", C.c_void_p),
                ("loss", C.c_void_p), ("prob", C.c_void_p), ("lr", C.c_float), ("train", C.c_int)]


CTR_HIDDEN = 256


def ctr_step(rows: torch.Tensor, labels: torch.Tensor, fields: int, emb: int, weights: dict, grads: dict,
             d_rows: Optional[torch.Tensor], loss: torch.Tensor, lr: float, train: bool = True,
             prob: Optional[torch.Tensor] = None) -> None:
    """Fused wide-&-deep tower: forward, BCE, backward, dense SGD (mean gradient) and the row gradients
    (``-lr * dLoss/drow``, ready to push) in one kernel + a small apply kernel.  ``weights``: W1 [IN, 256],
    W1T [256, IN], b1 [256], w2 [256], b2 [1]; ``grads``: same shapes minus W1T.  ``rows`` is ``[B * fields,
    stride]`` with ``stride >= emb + 1`` (column ``emb`` is the wide weight); ``d_rows`` (train) has the shape of
    ``rows``, ``prob`` (optional) ``B`` elements, ``loss`` two.  Any other shape is a ``ValueError`` before
    anything is launched.  csrc/fps_ctr.cu."""
    _req(rows, "rows", torch.float32); _req(labels, "labels", torch.float32); _req(loss, "loss", torch.float32)
    fields, emb = int(fields), int(emb)
    B, IN = labels.numel(), fields * emb
    if fields < 1 or emb < 1 or IN > CTR_HIDDEN:
        raise ValueError(f"fields ({fields}) and emb ({emb}) must be >= 1 with fields * emb <= {CTR_HIDDEN}")
    if rows.dim() != 2 or rows.shape[0] != B * fields or rows.shape[1] < emb + 1:
        raise ValueError(f"rows must be [B * fields, >= emb + 1] = [{B * fields}, >= {emb + 1}], "
                         f"got {list(rows.shape)}")
    if loss.numel() != 2:
        raise ValueError(f"loss must hold 2 floats, got {loss.numel()}")
    shapes = {"W1": (IN, CTR_HIDDEN), "W1T": (CTR_HIDDEN, IN), "b1": (CTR_HIDDEN,), "w2": (CTR_HIDDEN,), "b2": (1,)}
    for k, shp in shapes.items():
        _req(weights[k], k, torch.float32)
        if tuple(weights[k].shape) != shp:
            raise ValueError(f"weights[{k!r}] must be {list(shp)}, got {list(weights[k].shape)}")
    if prob is not None:
        _req(prob, "prob", torch.float32)
        if prob.numel() != B:
            raise ValueError(f"prob must hold B = {B} floats, got {prob.numel()}")
    if train:
        _req(d_rows, "d_rows", torch.float32)
        if d_rows.shape != rows.shape:
            raise ValueError(f"d_rows must have the shape of rows {list(rows.shape)}, got {list(d_rows.shape)}")
        for k in ("W1", "b1", "w2", "b2"):
            _req(grads[k], f"grads[{k!r}]", torch.float32)
            if tuple(grads[k].shape) != shapes[k]:
                raise ValueError(f"grads[{k!r}] must be {list(shapes[k])}, got {list(grads[k].shape)}")
    a = CtrArgsC()
    a.rows = rows.data_ptr(); a.labels = labels.data_ptr(); a.batch = B
    a.fields, a.emb, a.stride = fields, emb, int(rows.shape[1])
    for k in shapes:
        setattr(a, k, weights[k].data_ptr())
    if train:
        a.gW1, a.gb1, a.gw2, a.gb2 = (grads[k].data_ptr() for k in ("W1", "b1", "w2", "b2"))
        a.d_rows = d_rows.data_ptr()
    a.loss = loss.data_ptr()
    a.prob = prob.data_ptr() if prob is not None else None
    a.lr = float(lr); a.train = int(bool(train))
    _check(lib().fps_ctr_step(C.byref(a), C.c_void_p(weights["W1"].data_ptr()),
                              C.c_void_p(weights["W1T"].data_ptr()), C.c_void_p(weights["b1"].data_ptr()),
                              C.c_void_p(weights["w2"].data_ptr()), C.c_void_p(weights["b2"].data_ptr()),
                              sm_count(rows.device.index), _stream()), "ctr_step")
    _bump(2 if train else 1)


class OutPolicyC(C.Structure):
    """Mirror of ``struct OutPolicy`` (csrc/fps_output.cu)."""

    _fields_ = [("count_max", C.c_ulonglong), ("interval_ns", C.c_ulonglong), ("n_new", C.c_ulonglong),
                ("staging_cap", C.c_ulonglong), ("ring_cap", C.c_ulonglong), ("require_all", C.c_int),
                ("force", C.c_int)]


OUT_STATE_WORDS = 8     # int64 words of ``struct OutState``


def output_step(state: torch.Tensor, s_ids: torch.Tensor, s_vecs: torch.Tensor, ring_ids: torch.Tensor,
                ring_vecs: torch.Tensor, host_tail: torch.Tensor, host_head: torch.Tensor, *, n_new: int,
                count_max: int = 0, interval_ns: int = 0, require_all: bool = False,
                force: bool = False) -> None:
    """Device-side count / timer flush policy of the worker output stream followed by the flush kernel
    (staging area -> ring in pinned host memory, tail published with ``st.release.sys``).  The ring and
    the head / tail words are pinned host tensors (mapped); csrc/fps_output.cu."""
    _req(state, "state", torch.int64); _req(s_ids, "s_ids", torch.int64); _req(s_vecs, "s_vecs", torch.float32)
    for t, nm in ((ring_ids, "ring_ids"), (ring_vecs, "ring_vecs"), (host_tail, "host_tail"), (host_head, "host_head")):
        if t.is_cuda or not t.is_pinned():
            raise ValueError(f"{nm} must be a pinned host tensor")
    p = OutPolicyC()
    p.count_max = int(count_max); p.interval_ns = int(interval_ns); p.n_new = int(n_new)
    p.staging_cap = int(s_ids.numel()); p.ring_cap = int(ring_ids.numel())
    p.require_all = int(bool(require_all)); p.force = int(bool(force))
    _check(lib().fps_output_step(C.byref(p), C.c_void_p(state.data_ptr()), C.c_void_p(s_ids.data_ptr()),
                                 C.c_void_p(s_vecs.data_ptr()), int(s_vecs.shape[1]),
                                 C.c_void_p(ring_ids.data_ptr()), C.c_void_p(ring_vecs.data_ptr()),
                                 C.c_void_p(host_tail.data_ptr()), C.c_void_p(host_head.data_ptr()),
                                 sm_count(state.device.index), _stream()), "output_step")
    _bump(2)


class FlushPolicyC(C.Structure):
    """Mirror of ``struct FlushPolicy`` (csrc/fps_replica.cu)."""

    _fields_ = [("count_max", C.c_ulonglong), ("interval_ns", C.c_ulonglong),
                ("add_uniform", C.c_ulonglong), ("require_all", C.c_int), ("force", C.c_int),
                ("num_dest", C.c_int), ("pad_", C.c_int)]


FLUSH_STATE_WORDS = 3 * FPS_MAX_SHARDS + 1   # int64 words of ``struct FlushState``
FLUSH_PENDING, FLUSH_LAST_NS, FLUSH_COUNT, FLUSH_MASK = 0, FPS_MAX_SHARDS, 2 * FPS_MAX_SHARDS, 3 * FPS_MAX_SHARDS


def flush_policy(state: torch.Tensor, num_dest: int, count_max: int = 0, interval_ns: int = 0,
                 require_all: bool = False, force: bool = False, add_uniform: int = 0) -> None:
    """Device-side CountLogic / TimerLogic (CountLogic.scala:5-29, TimerLogic.scala:6-51) for the
    per-destination send buffers of a replica: decides ON THE GPU which destinations to flush now
    (messages buffered >= ``count_max`` and/or ``globaltimer`` deadline ``interval_ns`` passed, OR /
    AND) and leaves the bit mask in ``state`` (int64 ``[FLUSH_STATE_WORDS]``) for the exchange kernel.
    ``num_dest`` outside ``[1, FPS_MAX_SHARDS]`` and a short ``state`` are refused before any CUDA check."""
    if not 1 <= int(num_dest) <= FPS_MAX_SHARDS:
        raise ValueError(f"num_dest must be in [1, {FPS_MAX_SHARDS}], got {num_dest}")
    if state.numel() < FLUSH_STATE_WORDS:
        raise ValueError(f"state must hold {FLUSH_STATE_WORDS} int64 words, got {state.numel()}")
    _req(state, "state", torch.int64)
    p = FlushPolicyC()
    p.count_max = int(count_max); p.interval_ns = int(interval_ns); p.add_uniform = int(add_uniform)
    p.require_all = int(bool(require_all)); p.force = int(bool(force)); p.num_dest = int(num_dest)
    _check(lib().fps_flush_policy(C.byref(p), C.c_void_p(state.data_ptr()), _stream()), "flush_policy")
    _bump()


class ExchArgsC(C.Structure):
    """Mirror of ``struct ExchArgs`` (csrc/fps_replica.cu)."""

    _fields_ = [("master", ShardTableC), ("cache", C.c_void_p), ("base", C.c_void_p),
                ("rps", C.c_longlong), ("slot_lo", C.c_longlong), ("slot_hi", C.c_longlong),
                ("state", C.c_void_p), ("mask_override", C.c_uint), ("n_stages", C.c_int),
                ("chunk_rows", C.c_int), ("sequential", C.c_int), ("slices", C.c_int),
                ("slice_offset", C.c_int), ("skip_mask", C.c_uint), ("pad_", C.c_int)]


def replica_exchange(master: ShardTableC, cache: torch.Tensor, base: torch.Tensor, *,
                     state: Optional[torch.Tensor] = None, mask: int = 0, n_ctas: int = 32,
                     n_stages: int = 4, slot_lo: int = 0, slot_hi: Optional[int] = None,
                     sequential: bool = False, slices: int = 1, slice_offset: int = 0,
                     skip_mask: int = 0) -> None:
    """One delta exchange between an owner-major replica and its master shards for the destinations
    flagged in ``state`` (written by :func:`flush_policy`) or in ``mask``: push ``replica - base``
    (REDG over NVLink), fold ``master - base`` into the replica, ``base <- master + pushed delta``.
    TMA bulk reads through a shared-memory ring; ``n_ctas`` CTAs.  csrc/fps_replica.cu.

    Each flagged destination moves its slots ``[slot_lo, slot_hi)``; with ``state`` and ``slices > 1``, one
    ``ceil((slot_hi - slot_lo) / slices)``-slot slice of them, slice ``(flushes[o] + o + slice_offset) %
    slices``, in both the TMA kernel and the kernel for rows wider than 2048 floats.  An empty range is a
    no-op.  ``n_stages <= 0`` means 4, more than 8 means 8.  Refused before any CUDA check: a shard count
    outside ``[1, FPS_MAX_SHARDS]``, a row stride that is not a positive multiple of 4 floats, and
    ``slot_lo < 0`` or ``slot_hi > rows_per_shard``."""
    _shard_count(master.num_shards)
    rps = int(master.rows_per_shard)
    if master.stride < 4 or master.stride % 4:
        raise ValueError(f"master stride must be a positive multiple of 4 floats, got {master.stride}")
    slot_hi = rps if slot_hi is None else int(slot_hi)
    if int(slot_lo) < 0 or slot_hi > rps:
        raise ValueError(f"slot range [{slot_lo}, {slot_hi}) is outside [0, {rps}]")
    _req(cache, "cache", torch.float32); _req(base, "base", torch.float32)
    assert cache.shape == base.shape and cache.shape[1] == master.stride
    assert cache.shape[0] == rps * master.num_shards
    a = ExchArgsC()
    a.master = master; a.cache = cache.data_ptr(); a.base = base.data_ptr(); a.rps = rps
    a.slot_lo = int(slot_lo); a.slot_hi = slot_hi
    if state is not None:
        _req(state, "state", torch.int64)
        a.state = state.data_ptr()
    a.mask_override = int(mask) & 0xFFFFFFFF
    a.n_stages = int(n_stages); a.sequential = int(bool(sequential))
    a.slices = max(1, int(slices)); a.slice_offset = int(slice_offset); a.skip_mask = int(skip_mask) & 0xFFFFFFFF
    _check(lib().fps_replica_exchange(C.byref(a), int(n_ctas), _stream()), "replica_exchange")
    _bump()


def segment_table(t: torch.Tensor, master: ShardTableC, alias: Optional[int] = None) -> ShardTableC:
    """ShardTable over a LOCAL owner-major ``[num_shards * rps, stride]`` tensor: the same
    ``id -> (owner, slot)`` map as ``master``, every "shard" in local HBM (a worker replica).
    ``alias=o``: segment ``o`` is the master shard itself (the worker's own shard is trained in place)."""
    _req(t, "table", torch.float32)
    n = int(master.num_shards)
    rps = int(master.rows_per_shard)
    assert t.shape[0] == n * rps and t.shape[1] == master.stride
    tc = ShardTableC()
    for o in range(n):
        tc.base[o] = master.base[o] if o == alias else t.data_ptr() + o * rps * t.shape[1] * 4
    tc.rows_per_shard = rps; tc.div = master.div; tc.num_shards = n
    tc.dim = master.dim; tc.stride = master.stride; tc.mode = master.mode
    tc.shard_shift = master.shard_shift
    return tc


def pull_dot(tab: ShardTableC, ids: torch.Tensor, local: torch.Tensor, score: torch.Tensor) -> None:
    _req(ids, "ids"); _req(local, "local", torch.float32); _req(score, "score", torch.float32)
    assert local.shape[0] == ids.numel() == score.numel()
    _check(lib().fps_pull_dot(C.byref(tab), C.c_void_p(ids.data_ptr()), _id_bytes(ids),
                              C.c_longlong(ids.numel()), C.c_void_p(local.data_ptr()),
                              int(local.shape[1]), C.c_void_p(score.data_ptr()),
                              sm_count(ids.device.index), _stream()), "pull_dot")
    _bump()


class TopkArgsC(C.Structure):
    """Mirror of ``struct TopkArgs`` (csrc/fps_topk_mma.cu)."""

    _fields_ = [
        ("q_ids", C.c_void_p),
        ("q_local", C.c_void_p),
        ("q_tab", ShardTableC),
        ("n_queries", C.c_int),
        ("n_items", C.c_int),
        ("stride", C.c_int),
        ("n_tiles", C.c_int),
        ("tiles_per_split", C.c_int),
        ("n_splits", C.c_int),
        ("mode", C.c_int),
        ("n_stages", C.c_int),
        ("out_scores", C.c_void_p),
        ("out_ld", C.c_longlong),
        ("tile_max", C.c_void_p),
        ("theta", C.c_void_p),
        ("cand_count", C.c_void_p),
        ("cand_score", C.c_void_p),
        ("cand_item", C.c_void_p),
        ("cand_cap", C.c_int),
        ("seg_cap", C.c_int),
        ("tile_lo", C.c_int),
        ("pad_", C.c_int),
        ("tile_limit", C.c_void_p),
    ]


TOPK_TILE = 128
# widest row the scoring kernel takes: strides up to 128 floats keep whole item tiles in shared memory,
# wider ones (up to 512) stream the items by 32-float K block (csrc/fps_topk_mma.cu)
TOPK_MAX_STRIDE = 512


def check_topk_stride(stride: int) -> None:
    """Raise ``ValueError`` for rows wider than the top-K scoring kernel supports."""
    if int(stride) > TOPK_MAX_STRIDE:
        raise ValueError(f"device top-K supports rows of at most {TOPK_MAX_STRIDE} floats "
                         f"(stride {int(stride)}); the kernel keeps the query block in shared memory")


def topk_geometry(items: torch.Tensor, n_queries: int, tile_lo: int = 0, cand_cap: int = 0):
    """``(n_tiles, n_splits, seg_cap)`` the scoring kernel will use for this problem: every query row
    is handled by ``n_splits`` CTAs, each owning ``seg_cap = cand_cap // n_splits`` candidate slots."""
    check_topk_stride(items.shape[1])
    a = TopkArgsC()
    a.n_queries = int(n_queries); a.n_items, a.stride = items.shape
    a.mode = -1; a.tile_lo = int(tile_lo); a.cand_cap = int(cand_cap)
    _check(lib().fps_topk_mma(C.byref(a), C.c_void_p(items.data_ptr()), 4,
                              sm_count(items.device.index), _stream()), "topk_geometry")
    return a.n_tiles, a.n_splits, a.seg_cap


def topk_mma(items: torch.Tensor, mode: int, *, q_ids: Optional[torch.Tensor] = None,
             q_tab: Optional[ShardTableC] = None, q_local: Optional[torch.Tensor] = None,
             out_scores: Optional[torch.Tensor] = None, tile_max: Optional[torch.Tensor] = None,
             theta: Optional[torch.Tensor] = None, cand_count: Optional[torch.Tensor] = None,
             cand_score: Optional[torch.Tensor] = None, cand_item: Optional[torch.Tensor] = None,
             tile_lo: int = 0, tile_limit: Optional[torch.Tensor] = None) -> None:
    """wgmma scoring kernel (K6): queries (pulled from ``q_tab`` by id, or ``q_local``) x local
    ``items`` with a mode-dependent epilogue.  Only tiles ``tile_lo <= t < min(n_tiles, tile_limit[0])``
    are scored (``tile_limit``: optional int32 device scalar).  Mode 2 fills per-split candidate
    segments: ``cand_count`` is ``[n_q, n_splits]`` (see :func:`topk_geometry`).  Rows of up to
    ``TOPK_MAX_STRIDE`` = 512 floats; wider ones raise ``ValueError``.  csrc/fps_topk_mma.cu."""
    check_topk_stride(items.shape[1])
    _req(items, "items", torch.float32)
    n_items, stride = items.shape
    a = TopkArgsC()
    if q_ids is not None:
        _req(q_ids, "q_ids")
        a.q_ids = q_ids.data_ptr(); a.q_tab = q_tab; n_q = q_ids.numel(); idb = _id_bytes(q_ids)
        if q_tab.stride != stride:
            raise ValueError("query table stride must equal item table stride")
    else:
        _req(q_local, "q_local", torch.float32)
        if q_local.shape[1] != stride:
            raise ValueError("q_local stride must equal item table stride")
        a.q_ids = None; a.q_local = q_local.data_ptr(); n_q = q_local.shape[0]; idb = 4
    a.n_queries = n_q; a.n_items = n_items; a.stride = stride; a.mode = int(mode)
    a.tile_lo = int(tile_lo)
    if tile_limit is not None:
        _req(tile_limit, "tile_limit", torch.int32)
        a.tile_limit = tile_limit.data_ptr()
    n_tiles = (n_items + TOPK_TILE - 1) // TOPK_TILE
    if mode == 0:
        _req(out_scores, "out_scores", torch.float32)
        a.out_scores = out_scores.data_ptr(); a.out_ld = out_scores.stride(0)
    elif mode == 1:
        _req(tile_max, "tile_max", torch.float32)
        if tuple(tile_max.shape) != (n_q, n_tiles):
            raise ValueError(f"tile_max must be [{n_q}, {n_tiles}]")
        a.tile_max = tile_max.data_ptr()
    else:
        _req(theta, "theta", torch.float32); _req(cand_count, "cand_count", torch.int32)
        _req(cand_score, "cand_score", torch.float32); _req(cand_item, "cand_item", torch.int32)
        a.theta = theta.data_ptr(); a.cand_count = cand_count.data_ptr()
        a.cand_score = cand_score.data_ptr(); a.cand_item = cand_item.data_ptr()
        a.cand_cap = cand_score.shape[1]
        _, n_splits, _ = topk_geometry(items, n_q, tile_lo, a.cand_cap)
        if tuple(cand_count.shape) != (n_q, n_splits):
            raise ValueError(f"cand_count must be [{n_q}, {n_splits}] (topk_geometry)")
    _check(lib().fps_topk_mma(C.byref(a), C.c_void_p(items.data_ptr()), idb,
                              sm_count(items.device.index), _stream()), "topk_mma")
    _bump()


def row_kth_largest(x: torch.Tensor, K: int, counts: Optional[torch.Tensor] = None,
                    n_cols: Optional[int] = None, k_per_row: Optional[torch.Tensor] = None) -> torch.Tensor:
    """K-th largest value of every row of ``x`` [n, L] (only the first ``n_cols`` columns if given);
    rows with fewer than ``K`` valid entries (``counts[row] < K``) give -3e38.  ``k_per_row`` (int32
    [n]) replaces ``K`` row by row.  Radix select, csrc/fps_select.cu."""
    _req(x, "x", torch.float32)
    n = x.shape[0]
    if counts is not None:
        _req(counts, "counts", torch.int32)
    if k_per_row is not None:
        _req(k_per_row, "k_per_row", torch.int32)
        if k_per_row.shape != (n,) or k_per_row.device != x.device:
            raise ValueError(f"k_per_row must be [{n}] on {x.device}")
    out = torch.empty(n, dtype=torch.float32, device=x.device)
    cols = int(x.shape[1] if n_cols is None else min(n_cols, x.shape[1]))
    _check(lib().fps_row_kth(C.c_void_p(x.data_ptr()), C.c_longlong(x.stride(0)), int(n),
                             cols, C.c_void_p(counts.data_ptr() if counts is not None else None),
                             int(K), C.c_void_p(k_per_row.data_ptr() if k_per_row is not None else None),
                             C.c_void_p(out.data_ptr()), _stream()), "row_kth")
    _bump()
    return out


def row_topk(scores: torch.Tensor, items: torch.Tensor, K: int, counts: Optional[torch.Tensor] = None,
             exclude: Optional[tuple] = None):
    """Sorted (descending) top-``K`` ``(score, item)`` of every row of the candidate arrays
    ``scores`` / ``items`` [n, cap] (int32 items); ``counts[row]`` limits the valid prefix.  Missing
    entries are ``(-3e38, -1)``; equal scores are ordered by ascending item.  ``exclude=(offsets,
    ex_items)``: int32 CSR, ``offsets`` [n + 1]; row ``r``'s excluded items ``ex_items[offsets[r]:
    offsets[r+1]]`` must be sorted ascending (see ``models.mf.device_topk.normalize_exclude``).
    Candidates whose item is excluded are dropped before the selection; rows left with fewer than ``K``
    get the missing-entry tail.  The kernel clamps every offset into ``[0, len(ex_items)]``, so a
    malformed CSR filters wrongly but never reads outside ``ex_items``."""
    _req(scores, "scores", torch.float32); _req(items, "items", torch.int32)
    if scores.shape != items.shape or scores.stride(0) != items.stride(0):
        raise ValueError("scores and items must have the same shape and row stride")
    if counts is not None:
        _req(counts, "counts", torch.int32)
    n = scores.shape[0]
    ex_off = ex_items = None
    ex_total = 0
    if exclude is not None:
        ex_off, ex_items = exclude
        _req(ex_off, "exclude offsets", torch.int32); _req(ex_items, "exclude items", torch.int32)
        if ex_off.shape != (n + 1,) or ex_items.dim() != 1:
            raise ValueError(f"exclude must be (offsets [{n + 1}], items [E]) int32")
        if ex_off.device != scores.device or ex_items.device != scores.device:
            raise ValueError(f"exclude must be on {scores.device}")
        ex_total = ex_items.numel()
        if ex_total == 0:                  # a non-null pointer selects the filtering kernel; never read
            ex_items = torch.zeros(1, dtype=torch.int32, device=scores.device)
    out_s = torch.empty((n, K), dtype=torch.float32, device=scores.device)
    out_i = torch.empty((n, K), dtype=torch.int32, device=scores.device)
    _check(lib().fps_row_topk(C.c_void_p(scores.data_ptr()), C.c_void_p(items.data_ptr()),
                              C.c_longlong(scores.stride(0)), int(n), int(scores.shape[1]),
                              C.c_void_p(counts.data_ptr() if counts is not None else None), int(K),
                              C.c_void_p(ex_off.data_ptr() if ex_off is not None else None),
                              C.c_void_p(ex_items.data_ptr() if ex_items is not None else None),
                              int(ex_total),
                              C.c_void_p(out_s.data_ptr()), C.c_void_p(out_i.data_ptr()), _stream()),
           "row_topk")
    _bump()
    return out_s, out_i


class PaArgsC(C.Structure):
    """Mirror of ``struct PaArgs`` (csrc/fps_pa.cu)."""

    _fields_ = [
        ("row_ptr", C.c_void_p), ("col_idx", C.c_void_p), ("values", C.c_void_p),
        ("labels", C.c_void_p), ("pred", C.c_void_p), ("loss", C.c_void_p), ("cost", C.c_void_p),
        ("n", C.c_longlong), ("binary", C.c_int), ("num_labels", C.c_int), ("algo", C.c_int),
        ("aggressiveness", C.c_float), ("nan_flag", C.c_void_p), ("tab", ShardTableC),
    ]


PA_ALGOS = {"PA": 0, "PAI": 1, "PAII": 2, "PB": 3, "ML": 4}
PA_UNLABELLED = -(2 ** 31)


def pa_step(tab: ShardTableC, row_ptr: torch.Tensor, col_idx: torch.Tensor, values: torch.Tensor,
            labels: torch.Tensor, pred: torch.Tensor, *, binary: bool, num_labels: int, algo: str,
            aggressiveness: float = 0.0, cost: Optional[torch.Tensor] = None,
            loss: Optional[torch.Tensor] = None, nan_flag: Optional[torch.Tensor] = None) -> None:
    """Fused passive-aggressive step over a CSR micro-batch (K7).  See csrc/fps_pa.cu."""
    _req(row_ptr, "row_ptr", torch.int64); _req(col_idx, "col_idx"); _req(values, "values", torch.float32)
    _req(labels, "labels", torch.int32); _req(pred, "pred", torch.int32)
    a = PaArgsC()
    a.row_ptr = row_ptr.data_ptr(); a.col_idx = col_idx.data_ptr(); a.values = values.data_ptr()
    a.labels = labels.data_ptr(); a.pred = pred.data_ptr()
    a.loss = loss.data_ptr() if loss is not None else None
    a.cost = cost.data_ptr() if cost is not None else None
    a.n = labels.numel(); a.binary = int(binary); a.num_labels = int(num_labels)
    a.algo = PA_ALGOS[algo]; a.aggressiveness = float(aggressiveness)
    a.nan_flag = nan_flag.data_ptr() if nan_flag is not None else None
    a.tab = tab
    _check(lib().fps_pa_step(C.byref(a), _id_bytes(col_idx), sm_count(values.device.index), _stream()),
           "pa_step")
    _bump()


class FmArgsC(C.Structure):
    """Mirror of ``struct FmArgs`` (csrc/fps_fm.cu)."""

    _fields_ = [
        ("row_ptr", C.c_void_p), ("cols", C.c_void_p), ("vals", C.c_void_p), ("labels", C.c_void_p),
        ("pred", C.c_void_p), ("stats", C.c_void_p), ("nan_flag", C.c_void_p), ("bad_id", C.c_void_p),
        ("n", C.c_longlong), ("nnz", C.c_longlong), ("num_features", C.c_longlong),
        ("dim", C.c_int), ("loss", C.c_int), ("lr", C.c_float), ("reg_linear", C.c_float),
        ("reg_factors", C.c_float), ("predict_only", C.c_int), ("bias", C.c_int), ("pad_", C.c_int),
        ("bias_acc", C.c_void_p), ("bias_done", C.c_void_p), ("tab", ShardTableC),
        ("reserve_total", C.c_int), ("max_ctas", C.c_int), ("acc", ShardTableC),
    ]


FM_LOSSES = {"logistic": 0, "squared": 1}
FM_MAX_DIM = 512   # widest row of the fused kernel: 1 + k floats


def fm_state(device) -> tuple:
    """Per-model device state of :func:`fm_step`'s ``w0`` rule: ``(bias_acc, bias_done)``, float64 ``[4]`` (sum of
    ``g``, labelled examples, the last ``w0`` delta, the sum of every ``w0`` delta pushed) and int32 ``[1]`` (the
    launch counter).  The kernel leaves the first two words and the counter at zero after every launch."""
    dev = torch.device(device)
    return torch.zeros(4, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)


def _check_fm_acc(acc, tab) -> None:
    """An AdaGrad accumulator table must have the parameter table's geometry: ``H`` of element ``(id, col)`` sits at
    the row's slot and column (DESIGN §2.17)."""
    if acc is None:
        return
    if not isinstance(acc, ShardTableC):
        raise TypeError(f"acc must be a ShardTableC or None, got {type(acc).__name__}")
    if not acc.base[0]:
        raise ValueError("acc has no shard 0 (a null base pointer would select plain SGD)")
    geo = ("stride", "dim", "rows_per_shard", "div", "num_shards", "mode")
    mine, theirs = tuple(int(getattr(acc, f)) for f in geo), tuple(int(getattr(tab, f)) for f in geo)
    if mine != theirs:
        raise ValueError(f"the accumulator table's geometry (stride, dim, rows_per_shard, div, shards, mode) {mine} "
                         f"differs from the parameter table's {theirs}")


def _fm_common_args(a, tab, bias, bias_state, predict_only, stats, nan_flag, bad_id, reserve_total, max_ctas,
                    acc=None):
    """The fields :class:`FmArgsC` and :class:`FfmArgsC` share: the ``w0`` state, the counters, the grid and the
    AdaGrad accumulators."""
    a.predict_only, a.bias = int(bool(predict_only)), int(bool(bias))
    if bias and not predict_only:
        bias_acc, done = bias_state
        _req(bias_acc, "bias_acc", torch.float64); _req(done, "bias_done", torch.int32)
        a.bias_acc, a.bias_done = bias_acc.data_ptr(), done.data_ptr()
    for t, name, dt in ((stats, "stats", torch.float32), (nan_flag, "nan_flag", torch.int32),
                        (bad_id, "bad_id", torch.int32)):
        if t is not None:
            _req(t, name, dt)
            setattr(a, name, t.data_ptr())
    a.tab = tab
    a.reserve_total, a.max_ctas = int(reserve_total), int(max_ctas)
    if acc is not None:
        a.acc = acc


def fm_step(tab: ShardTableC, row_ptr: torch.Tensor, cols: torch.Tensor, vals: Optional[torch.Tensor],
            labels: Optional[torch.Tensor], pred: torch.Tensor, *, num_features: int, loss: str = "logistic",
            lr: float = 0.05, reg_linear: float = 0.0, reg_factors: float = 0.0, bias: bool = True,
            bias_state: Optional[tuple] = None, predict_only: bool = False, stats: Optional[torch.Tensor] = None,
            nan_flag: Optional[torch.Tensor] = None, bad_id: Optional[torch.Tensor] = None,
            reserve_total: int = 0, max_ctas: int = 0, acc: Optional[ShardTableC] = None) -> None:
    """Fused factorization-machine step over a CSR micro-batch (csrc/fps_fm.cu, DESIGN §2.15): one launch.

    ``tab``: the model's :class:`ShardTableC`, rows ``[w | v_1 .. v_k | 0]`` of ``dim = 1 + k`` floats, id
    ``num_features`` the bias row (``w0`` in column 0).  ``row_ptr`` int64 ``[n + 1]``, ``cols`` int32 or int64,
    ``vals`` float32 of the same length or ``None`` (one-hot: every value 1), ``labels`` float32 ``[n]`` (NaN:
    predict only; ``None`` with ``predict_only``).  ``pred`` float32 ``[n]`` receives ``yhat`` from before each
    example's own update.  ``loss``: ``"logistic"`` (labels in {0, 1}) or ``"squared"``.  ``stats`` (float32
    ``[2]``) accumulates the loss and the labelled examples; ``nan_flag`` is set by a non-finite delta, ``bad_id``
    by an entry outside ``[0, num_features)`` (skipped).  With ``bias``, ``bias_state`` (:func:`fm_state`) carries
    the per-launch ``w0`` step: ``w0 -= lr * sum g / n_labelled``, pushed by the last CTA.  ``max_ctas`` > 0 caps
    the grid.  ``acc``: a :class:`ShardTableC` of ``tab``'s geometry holding AdaGrad's ``H`` per element (DESIGN
    §2.17); the feature rows then step by ``-lr * gam / sqrt(1 + H + gam^2)`` and ``H += gam^2``, where ``gam`` is
    the SGD gradient with its L2 term (``w0`` keeps the SGD rule; ``predict_only`` leaves ``H`` alone).  ``None``:
    plain SGD.  Every dtype, length and argument refusal comes before the library loads."""
    if loss not in FM_LOSSES:
        raise ValueError(f"loss must be one of {sorted(FM_LOSSES)}, got {loss!r}")
    _check_fm_acc(acc, tab)
    if row_ptr.dtype != torch.int64:
        raise TypeError(f"row_ptr must be {torch.int64}, got {row_ptr.dtype}")
    if cols.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"cols must be int32 or int64, got {cols.dtype}")
    if vals is not None:
        if vals.dtype != torch.float32:
            raise TypeError(f"vals must be {torch.float32}, got {vals.dtype}")
        if vals.numel() != cols.numel():
            raise ValueError("cols and vals must have the same length")
    n = row_ptr.numel() - 1
    if n < 0:
        raise ValueError("row_ptr must hold n + 1 offsets")
    if labels is None:
        if not predict_only:
            raise ValueError("a training step needs labels (predict_only=True predicts without)")
    else:
        if labels.dtype != torch.float32:
            raise TypeError(f"labels must be {torch.float32}, got {labels.dtype}")
        if labels.numel() != n:
            raise ValueError(f"labels must hold one entry per example: {labels.numel()} != {n}")
    if pred.dtype != torch.float32:
        raise TypeError(f"pred must be {torch.float32}, got {pred.dtype}")
    if pred.numel() != n:
        raise ValueError(f"pred must hold one entry per example: {pred.numel()} != {n}")
    if float(reg_linear) < 0 or float(reg_factors) < 0:
        raise ValueError("reg_linear and reg_factors must be >= 0")
    if int(num_features) < 0:
        raise ValueError(f"num_features must be >= 0, got {num_features}")
    if n >= 2 ** 31 - 1:
        raise ValueError("a micro-batch must hold fewer than 2**31 - 1 examples")
    if bias and not predict_only and bias_state is None:
        raise ValueError("bias=True needs bias_state (see fm_state)")
    _req(row_ptr, "row_ptr"); _req(cols, "cols"); _req(pred, "pred")
    if vals is not None:
        _req(vals, "vals")
    if labels is not None:
        _req(labels, "labels")
    a = FmArgsC()
    a.row_ptr, a.cols, a.pred = row_ptr.data_ptr(), cols.data_ptr(), pred.data_ptr()
    a.vals = vals.data_ptr() if vals is not None else None
    a.labels = labels.data_ptr() if labels is not None else None
    a.n, a.nnz, a.num_features = n, cols.numel(), int(num_features)
    a.dim, a.loss = int(tab.dim), FM_LOSSES[loss]
    a.lr, a.reg_linear, a.reg_factors = float(lr), float(reg_linear), float(reg_factors)
    _fm_common_args(a, tab, bias, bias_state, predict_only, stats, nan_flag, bad_id, reserve_total, max_ctas, acc)
    if n == 0:
        return
    _check(lib().fps_fm_step(C.byref(a), _id_bytes(cols), sm_count(pred.device.index), _stream()), "fm_step")
    _bump()


class FfmArgsC(C.Structure):
    """Mirror of ``struct FfmArgs`` (csrc/fps_ffm.cu)."""

    _fields_ = [
        ("row_ptr", C.c_void_p), ("cols", C.c_void_p), ("fields", C.c_void_p), ("vals", C.c_void_p),
        ("labels", C.c_void_p), ("pred", C.c_void_p), ("stats", C.c_void_p), ("nan_flag", C.c_void_p),
        ("bad_id", C.c_void_p), ("n", C.c_longlong), ("nnz", C.c_longlong), ("num_features", C.c_longlong),
        ("num_fields", C.c_int), ("k", C.c_int), ("loss", C.c_int), ("lr", C.c_float), ("reg_linear", C.c_float),
        ("reg_factors", C.c_float), ("predict_only", C.c_int), ("bias", C.c_int),
        ("bias_acc", C.c_void_p), ("bias_done", C.c_void_p), ("tab", ShardTableC),
        ("reserve_total", C.c_int), ("max_ctas", C.c_int), ("acc", ShardTableC),
    ]


FFM_MAX_FACTORS = 64
FFM_MAX_FIELDS = 256


def ffm_stride(num_fields: int, num_factors: int) -> int:
    """Row length of the field-aware FM: ``[w | 0 0 0]`` and one slab of ``round_up(k, 4)`` floats per field."""
    return 4 + int(num_fields) * 4 * -(-int(num_factors) // 4)


def ffm_step(tab: ShardTableC, row_ptr: torch.Tensor, cols: torch.Tensor, fields: torch.Tensor,
             vals: Optional[torch.Tensor], labels: Optional[torch.Tensor], pred: torch.Tensor, *, num_features: int,
             num_fields: int, num_factors: int, loss: str = "logistic", lr: float = 0.05, reg_linear: float = 0.0,
             reg_factors: float = 0.0, bias: bool = True, bias_state: Optional[tuple] = None,
             predict_only: bool = False, stats: Optional[torch.Tensor] = None,
             nan_flag: Optional[torch.Tensor] = None, bad_id: Optional[torch.Tensor] = None,
             reserve_total: int = 0, max_ctas: int = 0, acc: Optional[ShardTableC] = None) -> None:
    """Fused field-aware FM step over a CSR micro-batch (csrc/fps_ffm.cu, DESIGN §2.16): one launch.

    ``tab``: the model's :class:`ShardTableC`, rows ``[w | 0 0 0 | V_0 | .. | V_F-1]`` of
    :func:`ffm_stride` floats, one slab of ``round_up(num_factors, 4)`` floats per field; id ``num_features`` is
    the bias row (``w0`` in column 0).  ``row_ptr`` int64 ``[n + 1]``, ``cols`` int32 or int64, ``fields`` int32
    of the same length, ``vals`` float32 or ``None`` (one-hot), ``labels`` float32 ``[n]`` (NaN: predict only;
    ``None`` with ``predict_only``).  ``pred`` float32 ``[n]`` receives ``yhat`` from before each example's own
    update.  ``bad_id`` is set by an entry whose feature is outside ``[0, num_features)`` or whose field is outside
    ``[0, num_fields)`` (skipped).  ``loss``, ``stats``, ``nan_flag``, ``bias_state`` (:func:`fm_state`),
    ``reserve_total``, ``max_ctas`` and ``acc`` (AdaGrad on ``w`` and on both slabs of every pair, DESIGN §2.17) are
    as in :func:`fm_step`.  Every dtype, length and argument refusal comes before the library loads."""
    if loss not in FM_LOSSES:
        raise ValueError(f"loss must be one of {sorted(FM_LOSSES)}, got {loss!r}")
    if not 1 <= int(num_factors) <= FFM_MAX_FACTORS:
        raise ValueError(f"num_factors must lie in [1, {FFM_MAX_FACTORS}], got {num_factors}")
    if not 1 <= int(num_fields) <= FFM_MAX_FIELDS:
        raise ValueError(f"num_fields must lie in [1, {FFM_MAX_FIELDS}], got {num_fields}")
    if int(tab.stride) != ffm_stride(num_fields, num_factors) or int(tab.dim) != int(tab.stride):
        raise ValueError(f"the table's rows must be {ffm_stride(num_fields, num_factors)} floats "
                         f"(4 + num_fields * round_up(num_factors, 4)), got dim {tab.dim}, stride {tab.stride}")
    _check_fm_acc(acc, tab)
    if row_ptr.dtype != torch.int64:
        raise TypeError(f"row_ptr must be {torch.int64}, got {row_ptr.dtype}")
    if cols.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"cols must be int32 or int64, got {cols.dtype}")
    if fields.dtype != torch.int32:
        raise TypeError(f"fields must be {torch.int32}, got {fields.dtype}")
    if fields.numel() != cols.numel():
        raise ValueError("cols and fields must have the same length")
    if vals is not None:
        if vals.dtype != torch.float32:
            raise TypeError(f"vals must be {torch.float32}, got {vals.dtype}")
        if vals.numel() != cols.numel():
            raise ValueError("cols and vals must have the same length")
    n = row_ptr.numel() - 1
    if n < 0:
        raise ValueError("row_ptr must hold n + 1 offsets")
    if labels is None:
        if not predict_only:
            raise ValueError("a training step needs labels (predict_only=True predicts without)")
    else:
        if labels.dtype != torch.float32:
            raise TypeError(f"labels must be {torch.float32}, got {labels.dtype}")
        if labels.numel() != n:
            raise ValueError(f"labels must hold one entry per example: {labels.numel()} != {n}")
    if pred.dtype != torch.float32:
        raise TypeError(f"pred must be {torch.float32}, got {pred.dtype}")
    if pred.numel() != n:
        raise ValueError(f"pred must hold one entry per example: {pred.numel()} != {n}")
    if float(reg_linear) < 0 or float(reg_factors) < 0:
        raise ValueError("reg_linear and reg_factors must be >= 0")
    if int(num_features) < 0:
        raise ValueError(f"num_features must be >= 0, got {num_features}")
    if n >= 2 ** 31 - 1:
        raise ValueError("a micro-batch must hold fewer than 2**31 - 1 examples")
    if bias and not predict_only and bias_state is None:
        raise ValueError("bias=True needs bias_state (see fm_state)")
    _req(row_ptr, "row_ptr"); _req(cols, "cols"); _req(fields, "fields"); _req(pred, "pred")
    if vals is not None:
        _req(vals, "vals")
    if labels is not None:
        _req(labels, "labels")
    a = FfmArgsC()
    a.row_ptr, a.cols, a.fields, a.pred = row_ptr.data_ptr(), cols.data_ptr(), fields.data_ptr(), pred.data_ptr()
    a.vals = vals.data_ptr() if vals is not None else None
    a.labels = labels.data_ptr() if labels is not None else None
    a.n, a.nnz, a.num_features = n, cols.numel(), int(num_features)
    a.num_fields, a.k, a.loss = int(num_fields), int(num_factors), FM_LOSSES[loss]
    a.lr, a.reg_linear, a.reg_factors = float(lr), float(reg_linear), float(reg_factors)
    _fm_common_args(a, tab, bias, bias_state, predict_only, stats, nan_flag, bad_id, reserve_total, max_ctas, acc)
    if n == 0:
        return
    _check(lib().fps_ffm_step(C.byref(a), _id_bytes(cols), sm_count(pred.device.index), _stream()), "ffm_step")
    _bump()


SKETCH_KINDS = {"bloom": 0, "tow": 1, "minhash": 2}


def sketch_update(tab: ShardTableC, kind: str, keys: torch.Tensor, tweets: torch.Tensor,
                  num_hashes: int, array_size: int = 0) -> None:
    """Sketch push fused with its update (red.or / red.add.s32 / red.min.u64).  csrc/fps_sketch.cu."""
    _req(keys, "keys", torch.int32); _req(tweets, "tweets", torch.int64)
    assert keys.numel() == tweets.numel()
    _check(lib().fps_sketch_update(C.byref(tab), SKETCH_KINDS[kind], C.c_void_p(keys.data_ptr()),
                                   C.c_void_p(tweets.data_ptr()), C.c_longlong(keys.numel()),
                                   int(num_hashes), int(array_size), sm_count(keys.device.index),
                                   _stream()), "sketch_update")
    _bump()


def sketch_query(kind: str, local_rows: torch.Tensor, n_words: int, num_hashes: int, query: torch.Tensor,
                 est: torch.Tensor, num_means: int = 1, key_slot: Optional[torch.Tensor] = None,
                 query_slot: int = 0, freq: Optional[torch.Tensor] = None, query_freq: float = 0.0) -> None:
    """Scan the local shard with one warp per key: tug-of-war median-of-means estimate (``kind="tow"``)
    or MinHash Jaccard / co-occurrence count (``kind="minhash"``, ``freq`` = per-key word frequencies).
    ``key_slot`` / ``query_slot`` restrict the scan to one time slot (time-aware jobs).  Rows that are not
    keys score ``-3e38``.  csrc/fps_sketch.cu."""
    _req(local_rows, "local_rows", torch.int32); _req(query, "query", torch.int32)
    _req(est, "est", torch.float32)
    if key_slot is not None:
        _req(key_slot, "key_slot", torch.int32)
    if freq is not None:
        _req(freq, "freq", torch.float32)
    _check(lib().fps_sketch_query(SKETCH_KINDS[kind], C.c_void_p(local_rows.data_ptr()),
                                  C.c_longlong(local_rows.shape[0]), int(local_rows.shape[1]),
                                  int(num_hashes), int(num_means), C.c_void_p(query.data_ptr()),
                                  C.c_void_p(key_slot.data_ptr() if key_slot is not None else None),
                                  int(query_slot), C.c_void_p(freq.data_ptr() if freq is not None else None),
                                  C.c_float(query_freq), C.c_void_p(est.data_ptr()),
                                  sm_count(local_rows.device.index), _stream()), "sketch_query")
    _bump()


def bloom_query(local_rows: torch.Tensor, n_words: int, query: torch.Tensor, m: float, k: float,
                est: torch.Tensor, key_slot: Optional[torch.Tensor] = None, query_slot: int = 0) -> None:
    _req(local_rows, "local_rows", torch.int32); _req(query, "query", torch.int32)
    _req(est, "est", torch.float32)
    if key_slot is not None:
        _req(key_slot, "key_slot", torch.int32)
    _check(lib().fps_bloom_query(C.c_void_p(local_rows.data_ptr()), C.c_longlong(local_rows.shape[0]),
                                 int(local_rows.shape[1]), int(n_words), C.c_void_p(query.data_ptr()),
                                 C.c_float(m), C.c_float(k),
                                 C.c_void_p(key_slot.data_ptr() if key_slot is not None else None),
                                 int(query_slot), C.c_void_p(est.data_ptr()),
                                 sm_count(local_rows.device.index), _stream()), "bloom_query")
    _bump()
