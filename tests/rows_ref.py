"""Host mirror of the row addressing and the dispatch rules of the generic row kernels (ops/csrc/fps_common.cuh
``fps_locate`` / ``fps_row32``, ops/csrc/fps_core.cu ``pick_lpr`` / ``use_wide`` / ``row_grid``).  CPU only.

``locate`` maps ids to ``(owner shard, slot)``: hash ``abs(id) % G`` and ``abs(id) / G``; range ``id / div`` with the
owner clamped to the last shard; LUT ``lut[id] = owner << 40 | slot``.  ``BREAKS`` switch one rule off for the
sensitivity checks: ``"range_no_clamp"`` drops the last-shard clamp, ``"hash_owner_slot_swapped"`` exchanges owner
and slot, ``"lut_ignored"`` addresses a LUT table as if it were hashed."""
import numpy as np

HASH, RANGE, LUT = 0, 1, 2
LUT_SHIFT = 40
LUT_SLOT_MASK = (1 << LUT_SHIFT) - 1
BREAKS = ("range_no_clamp", "hash_owner_slot_swapped", "lut_ignored")
WIDE_SEG_VEC = 256       # float4 per segment of the wide-row kernel
BLOCK = 256
CTAS_PER_SM = 8          # the row kernels' grid cap is num_sms * 8 CTAs


def locate(ids, mode, num_shards, div, lut=None, breaks=None):
    """(owner, slot) int64 arrays of ``ids`` as the device computes them."""
    if breaks is not None and breaks not in BREAKS:
        raise ValueError(f"unknown break {breaks!r}")
    ids = np.asarray(ids, dtype=np.int64)
    if mode == LUT and breaks == "lut_ignored":
        mode = HASH
    if mode == HASH:
        a = np.abs(ids)
        owner, slot = a % num_shards, a // num_shards
        if breaks == "hash_owner_slot_swapped":
            owner, slot = slot, owner
        return owner, slot
    if mode == LUT:
        e = np.asarray(lut, dtype=np.int64)[ids]
        return e >> LUT_SHIFT, e & LUT_SLOT_MASK
    owner = ids // div
    if breaks != "range_no_clamp":
        owner = np.minimum(owner, num_shards - 1)
    return owner, ids - owner * div


def lut_from_partitioner(num_ids, num_shards, partitioner):
    """The LUT a user partitioner defines: owner ``partitioner(id) % G``, slots in id order per owner."""
    owners = np.array([int(partitioner(i)) % num_shards for i in range(num_ids)], dtype=np.int64)
    slots = np.zeros(num_ids, dtype=np.int64)
    for o in range(num_shards):
        sel = np.nonzero(owners == o)[0]
        slots[sel] = np.arange(sel.size)
    return (owners << LUT_SHIFT) | slots


def stride_of(dim):
    return (dim + 3) // 4 * 4


def pick_lpr(nvec):
    """Lanes per row of the narrow row kernels: the power of two >= nvec, at most 32."""
    lpr = 1
    while lpr < nvec and lpr < 32:
        lpr <<= 1
    return lpr


def use_wide(stride, buf_width, touch):
    """Whether ``fps_pull_gather`` / ``fps_push_add`` take the wide-row kernel."""
    return stride // 4 > WIDE_SEG_VEC and buf_width % 4 == 0 and buf_width == stride and not touch


def lane_groups(num_sms, lpr):
    """Lane-groups of the capped grid of the narrow row kernels."""
    return num_sms * CTAS_PER_SM * (BLOCK // lpr)


def place(ids, values, owner, slot, num_shards, rows_per_shard, stride):
    """The shard arrays ``[G, rows_per_shard, stride]`` after ``table[ids] = values`` on zeroed shards, or None
    when some id lands outside every shard."""
    owner, slot = np.asarray(owner), np.asarray(slot)
    if ((owner < 0) | (owner >= num_shards) | (slot < 0) | (slot >= rows_per_shard)).any():
        return None
    out = np.zeros((num_shards, rows_per_shard, stride), dtype=np.float32)
    out[owner, slot, :values.shape[1]] = values
    return out
