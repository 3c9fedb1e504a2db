// Shared device-side definitions for the fps_b200 kernel library (sm_90a).
//
// A "ShardTable" is the device view of one parameter-server table: G shards (one per
// GPU / PS instance), each a dense row-major [rows_per_shard, stride] fp32 block living
// in that GPU's HBM and mapped into every peer's address space (CUDA IPC / VMM).  A
// pull is a load through base[owner(id)], a push is a red.add through the same pointer:
// there are no messages on the hot path (SURVEY §5.8; replaces FPS:411-463 routing).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define FPS_MAX_SHARDS 16

// HASH / RANGE are computed; LUT is a device lookup table id -> (owner << 40 | slot) that realises
// arbitrary user partitioners (FPS:343 paramPartitioner) and interned opaque / string ids.
enum FpsPartition : int { FPS_PART_HASH = 0, FPS_PART_RANGE = 1, FPS_PART_LUT = 2 };
#define FPS_LUT_SLOT_MASK ((1ll << 40) - 1)

struct ShardTable {
  float* base[FPS_MAX_SHARDS];          // peer-mapped base pointer per shard
  unsigned int* touched[FPS_MAX_SHARDS];  // optional per-shard touched bitmap (may be null)
  long long rows_per_shard;             // slot capacity of every shard
  long long div;                        // range partition divisor (ceil(featureCount / G))
  int num_shards;
  int dim;     // logical row length in floats
  int stride;  // physical row stride in floats (multiple of 4, zero padded)
  int mode;    // FpsPartition
  int shard_shift;  // log2(num_shards) if it is a power of two, else -1 (fast hash locate)
  int pad_;
  const long long* lut;  // FPS_PART_LUT: lut[id] = owner << 40 | slot (device memory, local to the reader)
};

// id -> (owner shard, slot).  Hash mode mirrors `abs(id.hashCode) % psParallelism`
// (FPS:191-199) for non-negative ints; range mode mirrors RangePSLogicWithClose.scala:51-62.
__device__ __forceinline__ void fps_locate(const ShardTable& t, long long id, int& owner,
                                           long long& slot) {
  if (t.mode == FPS_PART_HASH) {
    long long a = id < 0 ? -id : id;
    owner = (int)(a % t.num_shards);
    slot = a / t.num_shards;
  } else if (t.mode == FPS_PART_LUT) {
    const long long e = t.lut[id];
    owner = (int)(e >> 40);
    slot = e & FPS_LUT_SLOT_MASK;
  } else {
    owner = (int)(id / t.div);
    if (owner >= t.num_shards) owner = t.num_shards - 1;
    slot = id - (long long)owner * t.div;
  }
}

// 32-bit fast path: ids known to fit in an int (IdT == int); shift/mask when G is a power of two.
__device__ __forceinline__ float* fps_row32(const ShardTable& t, int id) {
  if (t.mode == FPS_PART_HASH) {
    const unsigned a = (unsigned)(id < 0 ? -id : id);
    unsigned owner, slot;
    if (t.shard_shift >= 0) {
      owner = a & ((1u << t.shard_shift) - 1u);
      slot = a >> t.shard_shift;
    } else {
      slot = a / (unsigned)t.num_shards;
      owner = a - slot * (unsigned)t.num_shards;
    }
    return t.base[owner] + (size_t)slot * (size_t)t.stride;
  }
  if (t.mode == FPS_PART_LUT) {
    const long long e = t.lut[id];
    return t.base[(int)(e >> 40)] + (size_t)(e & FPS_LUT_SLOT_MASK) * (size_t)t.stride;
  }
  unsigned owner = (unsigned)id / (unsigned)t.div;
  if (owner >= (unsigned)t.num_shards) owner = t.num_shards - 1;
  const unsigned slot = (unsigned)id - owner * (unsigned)t.div;
  return t.base[owner] + (size_t)slot * (size_t)t.stride;
}

__device__ __forceinline__ float* fps_row(const ShardTable& t, long long id) {
  int owner;
  long long slot;
  fps_locate(t, id, owner, slot);
  return t.base[owner] + slot * (long long)t.stride;
}

__device__ __forceinline__ void fps_touch(const ShardTable& t, long long id) {
  int owner;
  long long slot;
  fps_locate(t, id, owner, slot);
  unsigned int* bm = t.touched[owner];
  if (bm != nullptr) {
    asm volatile("red.relaxed.sys.global.or.b32 [%0], %1;" ::"l"(bm + (slot >> 5)),
                 "r"(1u << (slot & 31))
                 : "memory");
  }
}

template <typename IdT>
__device__ __forceinline__ float* fps_row_t(const ShardTable& t, IdT id) {
  if (sizeof(IdT) == 4) return fps_row32(t, (int)id);
  return fps_row(t, (long long)id);
}
// worker-local slot of a user: user / workerParallelism (32-bit / shift fast paths)
template <typename IdT>
__device__ __forceinline__ size_t fps_user_slot(IdT user, int user_div, int user_shift) {
  if (user_shift >= 0) return (size_t)((unsigned long long)user >> user_shift);
  if (sizeof(IdT) == 4) return (size_t)((unsigned)user / (unsigned)user_div);
  return (size_t)((long long)user / user_div);
}

// ---- 16-byte peer-capable memory ops --------------------------------------------------
// Pull: plain (weak) vector load; peer addresses route over NVLink and bypass local L2.
__device__ __forceinline__ float4 fps_ld_row4(const float* p) {
  float4 v;
  asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
// Push fused with paramUpdate (vectorSum, Vector.scala:72-84): one 16-byte reduction applied by
// the owner's memory system.  SASS: REDG.E.ADD.F32x4.FTZ.RN.STRONG.SYS.
__device__ __forceinline__ void fps_red_add4(float* p, float4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// L2 eviction-priority variants (createpolicy + .L2::cache_hint): used by the L2-blocked MF step to
// keep the current item bucket resident (evict_last) while the once-touched user rows stream through
// (evict_first).
__device__ __forceinline__ unsigned long long fps_policy_evict_first() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ unsigned long long fps_policy_evict_last() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ float4 fps_ld_row4_hint(const float* p, unsigned long long pol) {
  float4 v;
  asm volatile("ld.global.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void fps_red_add4_hint(float* p, float4 v, unsigned long long pol) {
  asm volatile("red.relaxed.sys.global.add.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol)
               : "memory");
}

// ---- Philox4x32-10 counter RNG (K4: init is a pure function of (seed, id, column)) -----
struct Philox4 {
  uint32_t x, y, z, w;
};
__host__ __device__ __forceinline__ uint32_t fps_mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}
__host__ __device__ __forceinline__ Philox4 fps_philox(uint32_t c0, uint32_t c1, uint32_t c2,
                                                       uint32_t c3, uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = fps_mulhi32(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = fps_mulhi32(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  Philox4 o;
  o.x = c0; o.y = c1; o.z = c2; o.w = c3;
  return o;
}
__host__ __device__ __forceinline__ float fps_u01(uint32_t x) {
  return (float)(x >> 8) * (1.0f / 16777216.0f);
}

// K5: in-kernel negative `j` of record `pos`, uniform over [0, a.num_items) from the Philox stream keyed
// (pos, j, a.step, a.seed).  A draw equal to the positive is shifted by 1 + s.z % 7, reduced modulo
// num_items - 1 so that it never lands back on the positive (num_items >= 2).  `a` is the kernel's argument
// block (MfArgs, BprArgs): step, seed and num_items are read where the draw uses them, which keeps every
// kernel's machine code as it was when each spelled the draw out.
template <typename Args, typename IdT>
__device__ __forceinline__ long long fps_k5_negative(const Args& a, long long pos, int j, IdT positive) {
  const Philox4 s = fps_philox((uint32_t)pos, (uint32_t)((unsigned long long)pos >> 32), (uint32_t)j,
                               (uint32_t)a.step, (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  const unsigned long long h = ((unsigned long long)s.x << 32) | s.y;
  long long neg = (long long)(h % (unsigned long long)a.num_items);
  if (neg == (long long)positive)
    neg = (neg + 1 + (long long)((s.z % 7u) % (unsigned long long)(a.num_items - 1))) % a.num_items;
  return neg;
}

// ---- training records ---------------------------------------------------------------------------------------
// A batch is either packed64 records in `users` (format 1: user:26 | item:22 | fp16 rating:16, 8 B per update)
// or users / items / ratings arrays of IdT ids (format 0).  The host packs with the same layout
// (ops/native.py pack_ratings, fps_host.cpp).  Which records are void is the caller's rule.
constexpr int FPS_REC_USER_SHIFT = 38;
constexpr int FPS_REC_ITEM_SHIFT = 16;
constexpr unsigned long long FPS_REC_ITEM_MASK = 0x3FFFFFull;

// Record i with its ids as OutT.  Returned by value, rating first: a decoder writing through reference parameters,
// or this struct with the ids first, changed the code nvcc generates for the pointwise and BPR kernels.
template <typename OutT>
struct FpsRecord {
  float rating;
  OutT user, item;
};
template <typename IdT, typename OutT = IdT>
__device__ __forceinline__ FpsRecord<OutT> fps_record(int format, const void* users, const void* items,
                                                      const float* ratings, long long i) {
  FpsRecord<OutT> r;
  if (format == 1) {
    const unsigned long long rec = reinterpret_cast<const unsigned long long*>(users)[i];
    r.user = (OutT)(rec >> FPS_REC_USER_SHIFT);
    r.item = (OutT)((rec >> FPS_REC_ITEM_SHIFT) & FPS_REC_ITEM_MASK);
    r.rating = __half2float(__ushort_as_half((unsigned short)(rec & 0xFFFFull)));
  } else {
    r.user = (OutT)reinterpret_cast<const IdT*>(users)[i];
    r.item = (OutT)reinterpret_cast<const IdT*>(items)[i];
    r.rating = ratings[i];
  }
  return r;
}
// The item of record i alone.
template <typename IdT>
__device__ __forceinline__ long long fps_record_item(int format, const void* users, const void* items, long long i) {
  if (format == 1)
    return (long long)((reinterpret_cast<const unsigned long long*>(users)[i] >> FPS_REC_ITEM_SHIFT) &
                       FPS_REC_ITEM_MASK);
  return (long long)reinterpret_cast<const IdT*>(items)[i];
}

// Warp-subgroup all-reduce (sum) over LPR consecutive lanes (LPR power of two <= 32).
template <int LPR>
__device__ __forceinline__ float fps_group_sum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
