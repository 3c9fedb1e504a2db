// Worker-side replica <-> master delta exchange (sender-side combining over NVLink).
//
// A worker trains a LOCAL replica of a PS table with the fused kernels (pulls and pushes stay in local
// HBM).  The replica is laid out owner-major -- segment o holds the rows of PS shard o in slot order --
// so segment o IS the per-destination send buffer of the reference's batching senders
// (M/common/CombinationLogic.scala:12-33, CombinationWorkerSender.scala:9-36), and a flush of
// destination o is a contiguous streaming pass over three arrays:
//
//     v = master_o (owner's HBM, NVLink peer)     c = replica segment     b = base segment
//     d = c - b   -> red.add into master_o   (my updates since the last flush: the batched PUSH)
//     f = v - b   -> red.add into c          (what the other workers pushed since: the batched PULL answer)
//     b = v + d                              ("the master as this worker knows it")
//
// Invariant: c - b == local updates not yet pushed; it holds element-wise whatever the training
// kernels do concurrently (they only red.add into c), so the exchange needs no barrier and nothing is
// ever lost (tests: multi-rank conservation over overlapping exchanges).
//
// Two kernels:
//  * fps_flush_policy_kernel -- the device-side CountLogic / TimerLogic (CountLogic.scala:5-29,
//    TimerLogic.scala:6-51): per destination, "messages buffered >= max" and/or "globaltimer deadline
//    passed", combined with AND / OR, evaluated on the GPU from device counters (fed by the bucket
//    histogram of the training step).  Output: the bit mask of destinations to flush now.
//  * fps_replica_exchange_kernel -- a few persistent CTAs (one producer lane + 4 consumer warps) that
//    stream the flagged segments through a shared-memory ring with TMA bulk copies (cp.async.bulk,
//    SASS UBLKCP; the remote leg is a bulk read of the owner's HBM over NVLink) completing on mbarriers.
//    Because the wire latency is carried by the TMA engine and not by resident warps, ~32 CTAs are enough
//    to move a slice per training step and the kernel runs NEXT TO the HBM-bound training kernel (which
//    leaves exactly those CTA slots free) instead of time-slicing the GPU with it.
#include "fps_common.cuh"
#include "fps_tma.cuh"

#define EX_CONSUMERS 128
#define EX_THREADS (32 + EX_CONSUMERS)
#define EX_VEC_PER_THREAD 4
#define EX_CHUNK_VEC (EX_CONSUMERS * EX_VEC_PER_THREAD)   // 512 float4 = 8 KiB per array per stage
#define EX_MAX_STAGES 8

struct FlushPolicy {
  unsigned long long count_max;    // CountLogic: flush when >= count_max messages are buffered (0 = off)
  unsigned long long interval_ns;  // TimerLogic: flush when the oldest buffered message is this old (0 = off)
  unsigned long long add_uniform;  // messages to add to every destination before evaluating (no histogram feed)
  int require_all;                 // 0: any trigger (OR), 1: all enabled triggers (AND)
  int force;                       // 1: flush every destination now
  int num_dest;
  int pad_;
};

struct FlushState {                                 // device memory, one per replica
  unsigned long long pending[FPS_MAX_SHARDS];       // messages buffered per destination since its last flush
  unsigned long long last_ns[FPS_MAX_SHARDS];       // globaltimer at the last flush
  unsigned long long flushes[FPS_MAX_SHARDS];       // flush count per destination (metrics)
  unsigned int mask;                                // OUT: destinations to flush in the next exchange
  unsigned int evals;                               // policy evaluations so far
};

__global__ void fps_flush_policy_kernel(const FlushPolicy p, FlushState* st) {
  const int o = threadIdx.x;
  bool fire = false;
  if (o < p.num_dest) {
    const unsigned long long now = fps_globaltimer_ns();
    // the counters are fed concurrently by the histogram kernel of the next micro-batch: atomics only
    unsigned long long pend = atomicAdd(&st->pending[o], p.add_uniform) + p.add_uniform;
    if (st->last_ns[o] == 0) st->last_ns[o] = now;
    const bool has_count = p.count_max != 0, has_timer = p.interval_ns != 0;
    const bool cnt = has_count && pend >= p.count_max;
    const bool tim = has_timer && pend != 0 && (now - st->last_ns[o]) >= p.interval_ns;
    if (p.force) fire = true;
    else if (p.require_all) fire = (has_count || has_timer) && (!has_count || cnt) && (!has_timer || tim);
    else fire = cnt || tim;
    if (fire) {
      atomicAdd(&st->pending[o], 0ull - pend);   // everything counted so far leaves with this flush
      st->last_ns[o] = now;
      st->flushes[o] += 1;
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, fire);
  if (o == 0) {
    st->mask = m;
    st->evals += 1;
  }
}

extern "C" int fps_flush_policy(const FlushPolicy* p, FlushState* st, cudaStream_t stream) {
  if (p->num_dest < 1 || p->num_dest > FPS_MAX_SHARDS) return -1401;
  fps_flush_policy_kernel<<<1, 32, 0, stream>>>(*p, st);
  return (int)cudaGetLastError();
}

struct ExchArgs {
  ShardTable master;        // peer-mapped master shards (base[o] = shard o)
  float* cache;             // replica  [num_shards][rps][stride]
  float* base;              // base     [num_shards][rps][stride]
  long long rps;            // rows per segment (== master.rows_per_shard)
  long long slot_lo, slot_hi;  // sub-range of every flagged segment
  const FlushState* state;  // mask source (nullptr: use mask_override)
  unsigned int mask_override;
  int n_stages;
  int chunk_rows;           // rows per pipeline stage (chunk_rows * stride/4 <= EX_CHUNK_VEC)
  int sequential;           // 0: interleave destinations chunk by chunk (spreads the NVLink load),
                            // 1: destination after destination (follows the L2-blocked training sweep)
  int slices;               // > 1: every flush of destination o moves ONE of `slices` equal sub-ranges of
  int slice_offset;         //   its segment, rotating: slice = (flushes[o] + o + slice_offset) % slices
  unsigned int skip_mask;   // destinations never exchanged (the worker's own shard is trained in place)
  int pad_;
};

__device__ __forceinline__ int ex_nth_set_bit(unsigned mask, int n) {
  for (int i = 0; i < n; ++i) mask &= mask - 1;
  return __ffs(mask) - 1;
}

// Slots [lo, hi) of destination o in one launch, the same in both exchange kernels: the whole
// [slot_lo, slot_hi), or when sliced one `slice_len` slice of it, slice = (flushes[o] + o + slice_offset) %
// slices (flushes[o] was bumped by the policy kernel).  Slices past slot_hi are empty (lo == hi).
__device__ __forceinline__ void ex_dest_range(const ExchArgs& a, int o, bool sliced, long long slice_len,
                                              long long& lo, long long& hi) {
  lo = a.slot_lo;
  hi = a.slot_hi;
  if (sliced) {
    const long long sl = (long long)((a.state->flushes[o] + (unsigned long long)(o + a.slice_offset)) %
                                     (unsigned long long)a.slices);
    lo = a.slot_lo + sl * slice_len;
    hi = lo + slice_len < a.slot_hi ? lo + slice_len : a.slot_hi;
    if (lo > hi) lo = hi;
  }
}

__global__ void __launch_bounds__(EX_THREADS, 1)
    fps_replica_exchange_kernel(const __grid_constant__ ExchArgs a) {
  extern __shared__ __align__(128) unsigned char ex_smem[];
  const int S = a.n_stages;
  const int stride = a.master.stride;
  const int nvec = stride >> 2;
  const uint32_t row_bytes = (uint32_t)stride * 4u;
  const size_t arr_bytes = (size_t)EX_CHUNK_VEC * 16;          // one array of one stage
  float4* buf = reinterpret_cast<float4*>(ex_smem);             // [S][3][EX_CHUNK_VEC]
  uint64_t* full = reinterpret_cast<uint64_t*>(ex_smem + (size_t)S * 3 * arr_bytes);
  uint64_t* empty = full + S;

  unsigned mask = a.state != nullptr ? a.state->mask : a.mask_override;
  mask &= (a.master.num_shards >= 32) ? 0xffffffffu : ((1u << a.master.num_shards) - 1u);
  mask &= ~a.skip_mask;
  const int n_dest = __popc(mask);
  if (n_dest == 0) return;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool sliced = a.slices > 1 && a.state != nullptr;
  const long long seg_slots = a.slot_hi - a.slot_lo;
  const long long slice_len = sliced ? (seg_slots + a.slices - 1) / a.slices : seg_slots;
  __shared__ long long seg_lo[FPS_MAX_SHARDS], seg_hi[FPS_MAX_SHARDS];
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], EX_CONSUMERS / 32);
    }
    mbar_fence_init();
  }
  if (threadIdx.x < a.master.num_shards) {
    const int o = threadIdx.x;
    long long lo, hi;
    ex_dest_range(a, o, sliced, slice_len, lo, hi);
    seg_lo[o] = lo;
    seg_hi[o] = hi;
  }
  __syncthreads();

  const long long n_slots = slice_len;
  const long long cps = (n_slots + a.chunk_rows - 1) / a.chunk_rows;   // chunks per (sub-)segment
  const long long total = cps * n_dest;

  // chunk g -> (destination o, first slot, rows)
  auto decode = [&](long long g, int& o, long long& slot0, int& rows) {
    int di;
    long long ci;
    if (a.sequential) {
      di = (int)(g / cps);
      ci = g - (long long)di * cps;
    } else {
      ci = g / n_dest;
      di = (int)(g - ci * n_dest);
    }
    o = ex_nth_set_bit(mask, di);
    slot0 = seg_lo[o] + ci * a.chunk_rows;
    const long long left = seg_hi[o] - slot0;
    rows = (int)(left < a.chunk_rows ? left : a.chunk_rows);
    if (rows < 0) rows = 0;
  };

  if (warp == 0) {
    if (lane != 0) return;
    // ============================ PRODUCER: TMA bulk reads ============================
    long long k = 0;
    for (long long g = blockIdx.x; g < total; g += gridDim.x, ++k) {
      const int s = (int)(k % S);
      const uint32_t ph = (uint32_t)((k / S) & 1);
      if (k >= S) mbar_wait(&empty[s], ph ^ 1u);
      int o, rows;
      long long slot0;
      decode(g, o, slot0, rows);
      const uint32_t bytes = (uint32_t)rows * row_bytes;
      const size_t seg_off = ((size_t)o * (size_t)a.rps + (size_t)slot0) * (size_t)stride;
      float4* st = buf + (size_t)s * 3 * EX_CHUNK_VEC;
      mbar_arrive_expect_tx(&full[s], 3u * bytes);     // rows == 0 (tail of a short slice): plain arrive
      if (bytes != 0) {
        tma_bulk_g2s(st, a.master.base[o] + (size_t)slot0 * (size_t)stride, bytes, &full[s]);  // NVLink leg
        tma_bulk_g2s(st + EX_CHUNK_VEC, a.cache + seg_off, bytes, &full[s]);
        tma_bulk_g2s(st + 2 * EX_CHUNK_VEC, a.base + seg_off, bytes, &full[s]);
      }
    }
    return;
  }
  // ============================ CONSUMERS: delta math + one-sided reductions ============================
  const int tid = threadIdx.x - 32;
  long long k = 0;
  for (long long g = blockIdx.x; g < total; g += gridDim.x, ++k) {
    const int s = (int)(k % S);
    const uint32_t ph = (uint32_t)((k / S) & 1);
    int o, rows;
    long long slot0;
    decode(g, o, slot0, rows);
    const int nq = rows * nvec;
    const size_t seg_off = ((size_t)o * (size_t)a.rps + (size_t)slot0) * (size_t)stride;
    float* mrow = a.master.base[o] + (size_t)slot0 * (size_t)stride;
    float* crow = a.cache + seg_off;
    float* brow = a.base + seg_off;
    const float4* st = buf + (size_t)s * 3 * EX_CHUNK_VEC;
    mbar_wait(&full[s], ph);
    float4 v[EX_VEC_PER_THREAD], c[EX_VEC_PER_THREAD], b[EX_VEC_PER_THREAD];
#pragma unroll
    for (int u = 0; u < EX_VEC_PER_THREAD; ++u) {
      const int q = tid + u * EX_CONSUMERS;
      if (q < nq) {
        v[u] = st[q];
        c[u] = st[EX_CHUNK_VEC + q];
        b[u] = st[2 * EX_CHUNK_VEC + q];
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);   // stage can be refilled while the results go out
#pragma unroll
    for (int u = 0; u < EX_VEC_PER_THREAD; ++u) {
      const int q = tid + u * EX_CONSUMERS;
      if (q < nq) {
        const float4 d = make_float4(c[u].x - b[u].x, c[u].y - b[u].y, c[u].z - b[u].z, c[u].w - b[u].w);
        const float4 f = make_float4(v[u].x - b[u].x, v[u].y - b[u].y, v[u].z - b[u].z, v[u].w - b[u].w);
        const bool has_d = d.x != 0.f || d.y != 0.f || d.z != 0.f || d.w != 0.f;
        const bool has_f = f.x != 0.f || f.y != 0.f || f.z != 0.f || f.w != 0.f;
        if (has_d) fps_red_add4(mrow + 4 * q, d);   // batched PUSH: REDG.ADD.F32x4 over NVLink
        if (has_f) fps_red_add4(crow + 4 * q, f);   // batched pull answer folded into the replica
        if (has_d || has_f)
          *reinterpret_cast<float4*>(brow + 4 * q) =
              make_float4(v[u].x + d.x, v[u].y + d.y, v[u].z + d.z, v[u].w + d.w);
      }
    }
  }
}

// Fallback for rows wider than one pipeline stage (> 8 KiB): register-staged loads, same math.
__global__ void __launch_bounds__(256)
    fps_replica_exchange_wide_kernel(const __grid_constant__ ExchArgs a) {
  unsigned mask = (a.state != nullptr ? a.state->mask : a.mask_override) & ~a.skip_mask;
  const int stride = a.master.stride;
  const int nvec = stride >> 2;
  const bool sliced = a.slices > 1 && a.state != nullptr;
  const long long seg_slots = a.slot_hi - a.slot_lo;
  const long long slice_len = sliced ? (seg_slots + a.slices - 1) / a.slices : seg_slots;
  for (int o = 0; o < a.master.num_shards; ++o) {
    if (!((mask >> o) & 1u)) continue;
    long long lo, hi;
    ex_dest_range(a, o, sliced, slice_len, lo, hi);
    const long long per_seg = (hi - lo) * nvec;
    float* m = a.master.base[o] + (size_t)lo * stride;
    const size_t seg_off = ((size_t)o * (size_t)a.rps + (size_t)lo) * (size_t)stride;
    float* cseg = a.cache + seg_off;
    float* bseg = a.base + seg_off;
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < per_seg;
         q += (long long)gridDim.x * blockDim.x) {
      const float4 v = fps_ld_row4(m + 4 * q);
      const float4 c = fps_ld_row4(cseg + 4 * q);
      const float4 b = *reinterpret_cast<const float4*>(bseg + 4 * q);
      const float4 d = make_float4(c.x - b.x, c.y - b.y, c.z - b.z, c.w - b.w);
      const float4 f = make_float4(v.x - b.x, v.y - b.y, v.z - b.z, v.w - b.w);
      const bool has_d = d.x != 0.f || d.y != 0.f || d.z != 0.f || d.w != 0.f;
      const bool has_f = f.x != 0.f || f.y != 0.f || f.z != 0.f || f.w != 0.f;
      if (has_d) fps_red_add4(m + 4 * q, d);
      if (has_f) fps_red_add4(cseg + 4 * q, f);
      if (has_d || has_f)
        *reinterpret_cast<float4*>(bseg + 4 * q) = make_float4(v.x + d.x, v.y + d.y, v.z + d.z, v.w + d.w);
    }
  }
}

// n_ctas: CTAs of the exchange grid (the training kernel leaves that many CTA slots free);
// n_stages <= 0 picks the default ring depth (4), more than EX_MAX_STAGES is clamped to it.  Refuses a shard
// count outside [1, FPS_MAX_SHARDS] (the kernels index per-shard arrays of that size), a stride that is not a
// positive multiple of 4 (16-byte bulk copies and vector reductions) and a slot range outside [0, rps).
// An empty range (slot_hi <= slot_lo) launches nothing.  Returns 0 or an error code.
extern "C" int fps_replica_exchange(const ExchArgs* args, int n_ctas, cudaStream_t stream) {
  ExchArgs a = *args;
  if (a.master.num_shards < 1 || a.master.num_shards > FPS_MAX_SHARDS) return -1403;
  if (a.master.stride < 4 || a.master.stride % 4 != 0) return -1404;
  if (a.slot_lo < 0 || a.slot_hi > a.rps) return -1405;
  if (a.slot_hi <= a.slot_lo) return 0;
  if (n_ctas < 1) n_ctas = 1;
  const int nvec = a.master.stride >> 2;
  if (nvec > EX_CHUNK_VEC) {   // one row does not fit a stage: register-staged fallback
    fps_replica_exchange_wide_kernel<<<n_ctas * 4, 256, 0, stream>>>(a);
    return (int)cudaGetLastError();
  }
  a.chunk_rows = EX_CHUNK_VEC / nvec;
  if (a.n_stages <= 0) a.n_stages = 4;
  if (a.n_stages > EX_MAX_STAGES) a.n_stages = EX_MAX_STAGES;
  const size_t smem = (size_t)a.n_stages * 3 * EX_CHUNK_VEC * 16 + 2 * a.n_stages * sizeof(uint64_t) + 64;
  cudaError_t e = cudaFuncSetAttribute(fps_replica_exchange_kernel,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  fps_replica_exchange_kernel<<<n_ctas, EX_THREADS, smem, stream>>>(a);
  return (int)cudaGetLastError();
}
