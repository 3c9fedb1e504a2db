// Message tier on the device: peer-memory request / response rings, a persistent server kernel and
// a device-side credit counter (pull limiter).
//
// This is the GPU replacement of the reference's iteration feedback edge (FPS:447-480) for the
// stores that need *logic* on the server (per-key locks, non-commutative paramUpdate): the fused
// kernels of fps_core.cu cover additive updates with zero messages, everything else goes through
// these rings.
//
//   worker w  --(request ring  Req[s][w], lives in shard s's HBM, written over NVLink)-->  shard s
//   shard  s  --(response ring Resp[w][s], lives in worker w's HBM, written over NVLink)--> worker w
//
// Rings are single-producer / single-consumer, entries are published with st.release.sys and
// observed with ld.acquire.sys, so FIFO order per (producer, consumer) pair -- the ordering the
// reference's per-id answer queues rely on (SURVEY 3.2) -- holds by construction.
//
// Server ops (the "registered-op table"): PULL answers the row; PUSH applies ADD / ASSIGN / MAX / MIN.
// Lock modes reproduce LockPSLogicA / LockPSLogicB (M/server/LockPSLogicA.scala:13-46,
// LockPSLogicB.scala:15-50): a pull takes the row lock, later pulls queue (B: one entry per worker),
// a push applies the update and either unlocks or hands the fresh value to the queue head.
//
// Credit counter = addPullLimiter (WL:196-250) on the device: at most `limit` unanswered pulls;
// excess pull ids wait in a FIFO spill queue; every consumed answer releases one credit and issues
// exactly one queued pull (contract of T/WorkerLogicTest.scala:34-46, tests/test_gpu_rings.py).
//
// Every spin loop is bounded (FPS_SPIN_LIMIT) and reports through an error word instead of hanging.
#include "fps_common.cuh"

#define FPS_SPIN_LIMIT (1u << 22)
#define RING_MAX_PEERS 16

enum RingOp : int { OP_PULL = 1, OP_PUSH = 2 };
enum UpdateOp : int { UPD_ADD = 0, UPD_ASSIGN = 1, UPD_MAX = 2, UPD_MIN = 3 };
enum LockMode : int { LOCK_NONE = 0, LOCK_A = 1, LOCK_B = 2 };
enum RingErr : int { ERR_NONE = 0, ERR_SPIN = 1, ERR_PUSH_UNKNOWN = 2, ERR_POOL = 3 };

struct RingHdr {               // 128 bytes, producer and consumer words on separate lines
  unsigned long long head;     // next slot to write  (producer)
  unsigned long long pad0[7];
  unsigned long long tail;     // next slot to read   (consumer)
  unsigned long long pad1[7];
};
struct Entry {                 // followed by `stride` floats of payload
  int op;
  int peer;                    // requests: asking worker; responses: answering shard
  long long id;
  unsigned int tag;
  unsigned int pad;
};

struct RingSet {               // one direction of one rank's rings, as seen by one side
  unsigned char* const* base;  // device table of ring base addresses (header + entries), [n_peers * lanes]:
                               //   ring of (peer p, lane l) = base[p * lanes + l]
  int n_peers;
  int lanes;                   // parallel rings per (worker, shard) pair; a key always uses lane
                               //   slot(id) % lanes, so FIFO order per key and pair is preserved
  int capacity;                // entries per ring (power of two)
  int stride;                  // payload floats
  int entry_bytes;             // sizeof(Entry) + 4 * stride, multiple of 16
  int pad_;
};

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ RingHdr* ring_hdr(const RingSet& r, int peer) {
  return reinterpret_cast<RingHdr*>(r.base[peer]);
}
__device__ __forceinline__ Entry* ring_entry(const RingSet& r, int peer, unsigned long long slot) {
  return reinterpret_cast<Entry*>(r.base[peer] + sizeof(RingHdr) +
                                  (size_t)(slot & (unsigned long long)(r.capacity - 1)) * r.entry_bytes);
}
__device__ __forceinline__ float* entry_payload(Entry* e) {
  return reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(e) + sizeof(Entry));
}

// Warp-cooperative enqueue (single producer per ring).  `peer` is the RING INDEX (peer * lanes + lane).
// `tail_cache` (optional, owned by the producer) holds the last consumer tail this producer has seen: the
// remote tail is re-read only when the ring looks full, so a put costs no NVLink round trip in the
// common case.  Publication: every lane's stores are ordered before lane 0's st.release.sys by the
// __syncwarp barrier (release is cumulative), so no separate system fence is needed.
// Returns false on spin-limit.
__device__ bool ring_put(const RingSet& r, int peer, int op, int self, long long id, unsigned tag,
                         const float* payload, int lane, int* err,
                         unsigned long long* tail_cache = nullptr) {
  RingHdr* h = ring_hdr(r, peer);
  unsigned long long head = 0;
  int ok = 1;
  if (lane == 0) {
    head = h->head;  // only this producer writes head: a plain read of our own last value
    unsigned long long tail = tail_cache ? *tail_cache : 0ull;
    if (head - tail >= (unsigned long long)r.capacity) {
      unsigned spins = 0;
      while (head - (tail = ld_acquire_sys(&h->tail)) >= (unsigned long long)r.capacity) {
        if (++spins > FPS_SPIN_LIMIT) { ok = 0; break; }
        __nanosleep(64);
      }
      if (tail_cache) *tail_cache = tail;
    }
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  head = __shfl_sync(0xffffffffu, head, 0);
  if (!ok) { if (lane == 0) atomicExch(err, ERR_SPIN); return false; }
  Entry* e = ring_entry(r, peer, head);
  if (lane == 0) { e->op = op; e->peer = self; e->id = id; e->tag = tag; e->pad = 0; }
  float* dst = entry_payload(e);
  for (int q = lane; q < r.stride; q += 32) dst[q] = payload ? payload[q] : 0.f;
  __syncwarp();
  if (lane == 0) st_release_sys(&h->head, head + 1);
  return true;
}

// ---- lane-per-message helpers (small payloads: one lane moves a whole entry) ----------------------------
#define FPS_BATCH_MAX_STRIDE 32     // floats; wider payloads use the warp-cooperative per-message paths
__device__ __forceinline__ void entry_write(Entry* e, int op, int self, long long id, unsigned tag,
                                            const float* payload, int stride) {
  e->op = op; e->peer = self; e->id = id; e->tag = tag; e->pad = 0;
  if (payload != nullptr) {
    float* dst = entry_payload(e);       // 8-byte aligned (24-byte header inside a 16-byte aligned entry)
    if ((stride & 1) == 0 && (reinterpret_cast<unsigned long long>(payload) & 7ull) == 0) {
      for (int q = 0; q < stride; q += 2)
        *reinterpret_cast<float2*>(dst + q) = *reinterpret_cast<const float2*>(payload + q);
    } else {
      for (int q = 0; q < stride; ++q) dst[q] = payload[q];
    }
  }
}
// producer side of an SPSC ring: make sure `n` more entries fit behind `head` (lane 0 spins, result broadcast)
__device__ __forceinline__ bool ring_reserve_space(RingHdr* h, unsigned long long head, int n, int capacity,
                                                   unsigned long long* tail_cache, int lane, int* err) {
  int ok = 1;
  if (lane == 0 && head + (unsigned long long)n - *tail_cache > (unsigned long long)capacity) {
    unsigned spins = 0;
    unsigned long long tail;
    while (head + (unsigned long long)n - (tail = ld_acquire_sys(&h->tail)) > (unsigned long long)capacity) {
      if (++spins > FPS_SPIN_LIMIT) { ok = 0; break; }
      __nanosleep(64);
    }
    *tail_cache = tail;
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  if (!ok && lane == 0) atomicExch(err, ERR_SPIN);
  return ok != 0;
}

// Multi-producer enqueue for the RESPONSE rings.  A worker's response ring for shard S is written by the
// server warp that serves that worker's requests AND, under the lock logics, by the warps of other workers
// that hand a released key over to a queued waiter -- several producers, all on this GPU.  Slots are
// reserved with a local atomic, filled, and published strictly in reservation order.
__device__ bool ring_put_mp(const RingSet& r, int ring, unsigned long long* reserve,
                            unsigned long long* published, unsigned long long* tail_cache, int op, int self,
                            long long id, unsigned tag, const float* payload, int lane, int* err) {
  RingHdr* h = ring_hdr(r, ring);
  unsigned long long slot = 0;
  int ok = 1;
  if (lane == 0) {
    slot = atomicAdd(reserve + ring, 1ull);
    // the consumer's tail as last seen by any producer of this ring (local memory, monotone): the remote
    // tail is re-read only when the ring looks full
    volatile unsigned long long* tc = tail_cache + ring;
    unsigned long long tail = *tc;
    if (slot - tail >= (unsigned long long)r.capacity) {
      unsigned spins = 0;
      while (slot - (tail = ld_acquire_sys(&h->tail)) >= (unsigned long long)r.capacity) {
        if (++spins > FPS_SPIN_LIMIT) { ok = 0; break; }
        __nanosleep(64);
      }
      atomicMax(tail_cache + ring, tail);
    }
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  slot = __shfl_sync(0xffffffffu, slot, 0);
  if (!ok) { if (lane == 0) atomicExch(err, ERR_SPIN); return false; }
  Entry* e = ring_entry(r, ring, slot);
  if (lane == 0) { e->op = op; e->peer = self; e->id = id; e->tag = tag; e->pad = 0; }
  float* dst = entry_payload(e);
  for (int q = lane; q < r.stride; q += 32) dst[q] = payload ? payload[q] : 0.f;
  __syncwarp();
  if (lane == 0) {
    volatile unsigned long long* pub = published + ring;
    unsigned spins = 0;
    while (*pub != slot) {                                   // wait for the earlier reservations
      if (++spins > FPS_SPIN_LIMIT) { ok = 0; break; }
      if (spins > 8) __nanosleep(64);
    }
    if (ok) {
      st_release_sys(&h->head, slot + 1);                    // release: cumulative over the warp's stores
      __threadfence();
      *pub = slot + 1;
    }
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  if (!ok && lane == 0) atomicExch(err, ERR_SPIN);
  return ok != 0;
}

// ============================================================================================
// persistent server kernel
// ============================================================================================
struct LockNode { int worker; unsigned tag; int next; };
struct ServerArgs {
  RingSet req;        // my request rings (local memory), one per worker
  RingSet resp;       // every worker's response ring for me (peer memory)
  ShardTable tab;     // the table; only rows of shard `self` are touched
  int self;           // this shard's index
  int update_op;      // UpdateOp
  int lock_mode;      // LockMode
  int* lock_state;    // [rows]: 0 unlocked, 1 locked                    (lock modes)
  int* lock_mutex;    // [rows]: spin mutex protecting the waiter list    (lock modes)
  int* wait_head;     // [rows]: head of the waiter list (-1 = empty), tail appended by walking
  LockNode* pool;     // waiter node pool
  int* pool_next;     // bump allocator over the pool (nodes are recycled through free_head)
  int* free_head;
  int pool_size;
  unsigned int* touched;  // [rows/32] bitmap: row ever pulled (lazy-init "exists" semantics)
  volatile int* stop;     // host sets to 1 to drain and exit
  int* err;
  unsigned long long* counters;  // [0] pulls served, [1] pushes applied, [2] answers sent
  unsigned long long* resp_reserve;    // [workers * lanes] slot reservation of every response ring (local)
  unsigned long long* resp_published;  // [workers * lanes] slots published so far (in-order publish)
  unsigned long long* resp_tail_cache; // [workers * lanes] last consumer tail seen (saves NVLink round trips)
};

__device__ __forceinline__ float* local_row(const ServerArgs& a, long long id, long long& slot) {
  int owner;
  fps_locate(a.tab, id, owner, slot);
  return a.tab.base[a.self] + slot * (long long)a.tab.stride;
}

__device__ void apply_update(const ServerArgs& a, float* row, const float* delta, int lane) {
  for (int q = lane; q < a.tab.stride; q += 32) {
    const float d = delta[q];
    if (a.update_op == UPD_ADD) {
      atomicAdd(row + q, d);
    } else if (a.update_op == UPD_ASSIGN) {
      row[q] = d;
    } else {
      int* p = reinterpret_cast<int*>(row + q);
      int old = *p, assumed;
      do {
        assumed = old;
        const float cur = __int_as_float(assumed);
        const float nv = (a.update_op == UPD_MAX) ? fmaxf(cur, d) : fminf(cur, d);
        old = atomicCAS(p, assumed, __float_as_int(nv));
      } while (old != assumed);
    }
  }
  __syncwarp();
}

__device__ bool answer(const ServerArgs& a, int worker, int ring_lane, long long id, unsigned tag,
                       const float* row, int lane) {
  return ring_put_mp(a.resp, worker * a.resp.lanes + ring_lane, a.resp_reserve, a.resp_published,
                     a.resp_tail_cache, OP_PULL, a.self, id, tag, row, lane, a.err);
}

// One warp per request ring; the rings of one shard are spread over as many CTAs as needed (8 warps each),
// so a shard with W workers x L lanes is served by W * L warps in parallel.
#define SERVER_WARPS 8
__global__ void __launch_bounds__(32 * SERVER_WARPS)
    fps_server_loop_kernel(const __grid_constant__ ServerArgs a) {
  const int w = blockIdx.x * SERVER_WARPS + (threadIdx.x >> 5);  // this warp serves request ring w
  const int lane = threadIdx.x & 31;
  if (w >= a.req.n_peers * a.req.lanes) return;
  const int ring_lane = w % a.req.lanes;
  RingHdr* h = ring_hdr(a.req, w);
  unsigned long long tail = h->tail, tail_pub = tail;
  unsigned long long c_pull = 0, c_push = 0, c_ans = 0;   // flushed to the global counters when idle / at exit
  unsigned idle = 0;
  while (true) {
    unsigned long long head = 0;
    if (lane == 0) head = ld_acquire_sys(&h->head);
    head = __shfl_sync(0xffffffffu, head, 0);
    if (tail == head) {
      if (lane == 0) {
        if (tail_pub != tail) { st_release_sys(&h->tail, tail); tail_pub = tail; }
        if (c_pull | c_push | c_ans) {
          atomicAdd(a.counters + 0, c_pull); atomicAdd(a.counters + 1, c_push); atomicAdd(a.counters + 2, c_ans);
          c_pull = c_push = c_ans = 0;
        }
      }
      if (*a.stop) break;
      if (++idle > 64) __nanosleep(256);
      continue;
    }
    idle = 0;
    if (a.lock_mode == LOCK_NONE && a.tab.stride <= FPS_BATCH_MAX_STRIDE) {
      // ---- lane-per-message batch: up to 32 requests of this ring at once ---------------------------------
      const int n = (int)min((unsigned long long)32, head - tail);
      const bool mine = lane < n;
      Entry* e = mine ? ring_entry(a.req, w, tail + lane) : nullptr;
      const int op = mine ? e->op : 0;
      const long long id = mine ? e->id : (long long)(-1 - lane);
      const unsigned tag = mine ? e->tag : 0u;
      const int worker = w / a.req.lanes;
      long long slot = 0;
      float* row = mine ? local_row(a, id, slot) : nullptr;
      // requests for the same key keep their ring order: they are handled in successive rounds
      const unsigned peers = __match_any_sync(0xffffffffu, id);
      const int my_round = __popc(peers & ((1u << lane) - 1u));
      int rounds = my_round;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) rounds = max(rounds, __shfl_xor_sync(0xffffffffu, rounds, o));
      // the answers of this batch go to ONE response ring: reserve their slots together
      const unsigned pull_mask = __ballot_sync(0xffffffffu, mine && op == OP_PULL);
      const int np = __popc(pull_mask);
      const int ring = worker * a.resp.lanes + ring_lane;
      RingHdr* rh = ring_hdr(a.resp, ring);
      unsigned long long base = 0;
      int ok = 1;
      if (np > 0) {
        if (lane == 0) {
          base = atomicAdd(a.resp_reserve + ring, (unsigned long long)np);
          volatile unsigned long long* tc = a.resp_tail_cache + ring;
          unsigned long long rt = *tc;
          if (base + np - rt > (unsigned long long)a.resp.capacity) {
            unsigned spins = 0;
            while (base + np - (rt = ld_acquire_sys(&rh->tail)) > (unsigned long long)a.resp.capacity) {
              if (++spins > FPS_SPIN_LIMIT) { ok = 0; break; }
              __nanosleep(64);
            }
            atomicMax(a.resp_tail_cache + ring, rt);
          }
        }
        ok = __shfl_sync(0xffffffffu, ok, 0);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (!ok) { if (lane == 0) atomicExch(a.err, ERR_SPIN); return; }
      }
      const unsigned long long my_slot = base + (unsigned long long)__popc(pull_mask & ((1u << lane) - 1u));
      for (int rd = 0; rd <= rounds; ++rd) {
        if (mine && my_round == rd) {
          if (a.touched) atomicOr(a.touched + (slot >> 5), 1u << (slot & 31));
          if (op == OP_PULL) {
            entry_write(ring_entry(a.resp, ring, my_slot), OP_PULL, a.self, id, tag, row, a.resp.stride);
          } else {
            const float* d = entry_payload(e);
            for (int q = 0; q < a.tab.stride; ++q) {
              if (a.update_op == UPD_ADD) atomicAdd(row + q, d[q]);
              else if (a.update_op == UPD_ASSIGN) row[q] = d[q];
              else {
                int* p = reinterpret_cast<int*>(row + q);
                int old = *p, assumed;
                do {
                  assumed = old;
                  const float cur = __int_as_float(assumed);
                  const float nv = (a.update_op == UPD_MAX) ? fmaxf(cur, d[q]) : fminf(cur, d[q]);
                  old = atomicCAS(p, assumed, __float_as_int(nv));
                } while (old != assumed);
              }
            }
          }
        }
        __threadfence();     // a later round (same key) must see this round's row
        __syncwarp();
      }
      if (np > 0) {          // publish the batch of answers, in reservation order
        if (lane == 0) {
          volatile unsigned long long* pub = a.resp_published + ring;
          unsigned spins = 0;
          while (*pub != base) {
            if (++spins > FPS_SPIN_LIMIT) { ok = 0; break; }
            if (spins > 8) __nanosleep(64);
          }
          if (ok) {
            st_release_sys(&rh->head, base + np);
            __threadfence();
            *pub = base + np;
          }
        }
        ok = __shfl_sync(0xffffffffu, ok, 0);
        if (!ok) { if (lane == 0) atomicExch(a.err, ERR_SPIN); return; }
      }
      c_pull += np; c_ans += np; c_push += n - np;
      tail += n;
      if (lane == 0 && tail - tail_pub >= (unsigned long long)(a.req.capacity / 4)) {
        st_release_sys(&h->tail, tail);
        tail_pub = tail;
      }
      __syncwarp();
      continue;
    }
    Entry* e = ring_entry(a.req, w, tail);
    const int op = e->op;
    const long long id = e->id;
    const unsigned tag = e->tag;
    const int worker = e->peer;
    long long slot;
    float* row = local_row(a, id, slot);
    if (a.lock_mode == LOCK_NONE) {
      if (op == OP_PULL) {
        if (lane == 0 && a.touched) atomicOr(a.touched + (slot >> 5), 1u << (slot & 31));
        if (!answer(a, worker, ring_lane, id, tag, row, lane)) return;
        ++c_pull; ++c_ans;
      } else {
        apply_update(a, row, entry_payload(e), lane);
        if (lane == 0 && a.touched) atomicOr(a.touched + (slot >> 5), 1u << (slot & 31));
        ++c_push;
      }
    } else {
      // ---- LockPSLogicA / B: all state changes of one row are serialised by a spin mutex ----
      int granted = 0, hand_worker = -1;
      unsigned hand_tag = 0;
      if (lane == 0) {
        unsigned spins = 0;
        while (atomicCAS(a.lock_mutex + slot, 0, 1) != 0)
          if (++spins > FPS_SPIN_LIMIT) { atomicExch(a.err, ERR_SPIN); break; }
        __threadfence();
        if (op == OP_PULL) {
          if (a.touched) atomicOr(a.touched + (slot >> 5), 1u << (slot & 31));
          if (a.lock_state[slot] == 0) {
            a.lock_state[slot] = 1;
            granted = 1;
          } else {
            bool dup = false;
            int last = -1;
            for (int n = a.wait_head[slot]; n >= 0; n = a.pool[n].next) {
              if (a.lock_mode == LOCK_B && a.pool[n].worker == worker) dup = true;
              last = n;
            }
            if (!dup) {
              const int node = atomicAdd(a.pool_next, 1);  // bump allocation (pool sized by the host)
              if (node >= a.pool_size) {
                atomicExch(a.err, ERR_POOL);
              } else {
                a.pool[node].worker = worker;
                a.pool[node].tag = tag;
                a.pool[node].next = -1;
                if (last < 0) a.wait_head[slot] = node; else a.pool[last].next = node;
              }
            }
          }
        } else {
          const bool known = a.touched == nullptr ||
                             ((a.touched[slot >> 5] >> (slot & 31)) & 1u) != 0;
          if (!known) atomicExch(a.err, ERR_PUSH_UNKNOWN);  // "Not existed model ..." (LockPSLogicA:43)
        }
      }
      granted = __shfl_sync(0xffffffffu, granted, 0);
      if (op == OP_PULL) {
        if (lane == 0) { __threadfence(); atomicExch(a.lock_mutex + slot, 0); }
        if (granted) {
          if (!answer(a, worker, ring_lane, id, tag, row, lane)) return;
          ++c_ans;
        }
        ++c_pull;
      } else {
        apply_update(a, row, entry_payload(e), lane);
        if (lane == 0) {
          const int n = a.wait_head[slot];
          if (n < 0) {
            a.lock_state[slot] = 0;                 // queue empty -> unlock
          } else {
            hand_worker = a.pool[n].worker;         // hand over to the head, stay locked
            hand_tag = a.pool[n].tag;
            a.wait_head[slot] = a.pool[n].next;
          }
          __threadfence();
          atomicExch(a.lock_mutex + slot, 0);
        }
        ++c_push;
        hand_worker = __shfl_sync(0xffffffffu, hand_worker, 0);
        hand_tag = __shfl_sync(0xffffffffu, hand_tag, 0);
        if (hand_worker >= 0) {
          if (!answer(a, hand_worker, ring_lane, id, hand_tag, row, lane)) return;
          ++c_ans;
        }
      }
    }
    ++tail;
    // hand the consumed slots back in batches (the producer re-reads our tail only when its ring looks full)
    if (lane == 0 && tail - tail_pub >= (unsigned long long)(a.req.capacity / 4)) {
      st_release_sys(&h->tail, tail);
      tail_pub = tail;
    }
    __syncwarp();
  }
  if (lane == 0) {
    st_release_sys(&h->tail, tail);
    atomicAdd(a.counters + 0, c_pull); atomicAdd(a.counters + 1, c_push); atomicAdd(a.counters + 2, c_ans);
  }
}

extern "C" int fps_server_loop_launch(const ServerArgs* a, cudaStream_t stream) {
  const int rings = a->req.n_peers * a->req.lanes;
  fps_server_loop_kernel<<<(rings + SERVER_WARPS - 1) / SERVER_WARPS, 32 * SERVER_WARPS, 0, stream>>>(*a);
  return (int)cudaGetLastError();
}

// ============================================================================================
// worker side: credit counter + issue / collect kernels (one warp each)
// ============================================================================================
struct ClientState {            // device-resident, one per worker
  int credits;                  // remaining pull credits (pullLimit - in flight)
  int limit;
  unsigned long long issued;    // pulls actually sent  (== the mock's pullCounter in the unit test)
  unsigned long long spill_head, spill_tail;  // FIFO of pull ids waiting for a credit
  unsigned int next_tag;
  int err;
};
struct ClientArgs {
  RingSet req;        // request rings of every shard for me (peer memory), indexed by shard
  RingSet resp;       // my response rings (local memory), indexed by shard
  ShardTable tab;     // only used for id -> owner shard
  ClientState* st;
  long long* spill;   // [spill_cap] ids
  int spill_cap;
  int self;           // worker index
};

// request / response ring index of a key: (owner shard, slot % lanes)
__device__ __forceinline__ int ring_of(const ShardTable& t, int lanes, long long id) {
  int owner; long long slot;
  fps_locate(t, id, owner, slot);
  return owner * lanes + (int)(slot % lanes);
}

__device__ bool issue_pull(const ClientArgs& a, long long id, int lane) {
  unsigned tag = 0;
  if (lane == 0) { tag = a.st->next_tag++; }
  tag = __shfl_sync(0xffffffffu, tag, 0);
  const bool ok = ring_put(a.req, ring_of(a.tab, a.req.lanes, id), OP_PULL, a.self, id, tag, nullptr, lane, &a.st->err);
  if (ok && lane == 0) a.st->issued++;
  return ok;
}

// pulls: limited by the credit counter, excess ids spill FIFO.  pushes: never limited.
__global__ void __launch_bounds__(32)
    fps_client_issue_kernel(const __grid_constant__ ClientArgs a, const long long* __restrict__ ids,
                            const float* __restrict__ deltas, int n, int op) {
  const int lane = threadIdx.x;
  for (int i = 0; i < n; ++i) {
    const long long id = ids[i];
    if (op == OP_PUSH) {
      if (!ring_put(a.req, ring_of(a.tab, a.req.lanes, id), OP_PUSH, a.self, id, 0u,
                    deltas + (size_t)i * a.req.stride, lane, &a.st->err))
        return;
      continue;
    }
    int take = 0;
    if (lane == 0) {
      if (a.st->credits > 0) { a.st->credits--; take = 1; }
      else if (a.st->spill_tail - a.st->spill_head < (unsigned long long)a.spill_cap)
        a.spill[a.st->spill_tail++ % a.spill_cap] = id;
      else a.st->err = ERR_POOL;
    }
    take = __shfl_sync(0xffffffffu, take, 0);
    if (take && !issue_pull(a, id, lane)) return;
  }
}

// Drain up to max_n answers: copy them out, release one credit each and issue ONE spilled pull.
__global__ void __launch_bounds__(32)
    fps_client_collect_kernel(const __grid_constant__ ClientArgs a, long long* __restrict__ out_ids,
                              float* __restrict__ out_vals, int max_n, int* __restrict__ n_out) {
  const int lane = threadIdx.x;
  int got = 0;
  for (int s = 0; s < a.resp.n_peers * a.resp.lanes && got < max_n; ++s) {
    RingHdr* h = ring_hdr(a.resp, s);
    unsigned long long tail = h->tail;
    while (got < max_n) {
      const unsigned long long head = ld_acquire_sys(&h->head);
      if (tail == head) break;
      Entry* e = ring_entry(a.resp, s, tail);
      if (lane == 0) out_ids[got] = e->id;
      const float* src = entry_payload(e);
      for (int q = lane; q < a.resp.stride; q += 32) out_vals[(size_t)got * a.resp.stride + q] = src[q];
      __syncwarp();
      ++tail; ++got;
      long long queued = -1;
      if (lane == 0) {
        st_release_sys(&h->tail, tail);
        a.st->credits++;                                   // pullCounter -= 1
        if (a.st->spill_head != a.st->spill_tail) {        // one queued pull per answer
          queued = a.spill[a.st->spill_head++ % a.spill_cap];
          a.st->credits--;
        }
      }
      queued = __shfl_sync(0xffffffffu, queued, 0);
      if (queued >= 0 && !issue_pull(a, queued, lane)) { if (lane == 0) *n_out = got; return; }
    }
  }
  if (lane == 0) *n_out = got;
}

extern "C" int fps_client_issue(const ClientArgs* a, const long long* ids, const float* deltas, int n,
                                int op, cudaStream_t stream) {
  if (n <= 0) return 0;
  fps_client_issue_kernel<<<1, 32, 0, stream>>>(*a, ids, deltas, n, op);
  return (int)cudaGetLastError();
}
extern "C" int fps_client_collect(const ClientArgs* a, long long* out_ids, float* out_vals, int max_n,
                                  int* n_out, cudaStream_t stream) {
  fps_client_collect_kernel<<<1, 32, 0, stream>>>(*a, out_ids, out_vals, max_n, n_out);
  return (int)cudaGetLastError();
}
// ============================================================================================
// throughput path: batched transactions through the message tier
// ============================================================================================
// A worker hands the kernel a whole micro-batch of keys, pre-sorted by ring (owner shard, lane).  One warp
// per ring is BOTH the single producer of the request ring and the single consumer of the response ring:
//   * pulls are issued in order under the worker's device credit counter (pullLimit, WL:196-250) -- the
//     keys that have not been issued yet ARE the FIFO spill queue of the limiter;
//   * every answer is copied to out_vals[message], releases its credit and (mode PULL_PUSH) immediately
//     triggers push(id, deltas[message]) -- the onPullRecv -> ps.push pattern of every reference worker
//     (e.g. PSOnlineMatrixFactorizationWorker.scala:42-55), which is also what releases a LockPSLogic lock;
//   * mode PUSH_ONLY streams pushes (non-commutative `assign` / max / min updates are applied by the
//     server warps in ring order).
// No launch per drain: the kernel lives until its messages are sent and all its pulls are answered.
// Deadlock freedom: a ring never has more pulls outstanding than its response ring holds, so a server
// warp never blocks on this worker's response ring and therefore always drains the request ring.
enum TxnMode : int { TXN_PULL_PUSH = 0, TXN_PULL_ONLY = 1, TXN_PUSH_ONLY = 2 };
struct TxnArgs {
  RingSet req;            // request rings of every (shard, lane) for me (peer memory)
  RingSet resp;           // my response rings, same indexing (local memory)
  const long long* ids;   // [n] keys sorted by ring index
  const float* deltas;    // [n, stride] (modes with a push)
  const int* seg;         // [rings + 1] segment offsets into ids
  float* out_vals;        // [n, stride] answers, by message (pull modes)
  int* credits;           // worker-wide credit counter: [credits, stalls]
  int* err;
  unsigned long long* counters;  // [0] pulls sent, [1] pushes sent, [2] answers consumed
  int self;
  int mode;
  int per_ring_cap;       // pulls one ring may have outstanding (fair share of the credits; <= ring capacity)
  int pad_;
};

#define TXN_WARPS 8
__global__ void __launch_bounds__(32 * TXN_WARPS)
    fps_client_txn_kernel(const __grid_constant__ TxnArgs a) {
  const int r = blockIdx.x * TXN_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int n_rings = a.req.n_peers * a.req.lanes;
  if (r >= n_rings) return;
  int pos = a.seg[r];
  const int end = a.seg[r + 1];
  if (pos == end) return;
  RingHdr* hq = ring_hdr(a.req, r);
  RingHdr* hr = ring_hdr(a.resp, r);
  unsigned long long qhead = hq->head;            // I am the only producer of this request ring
  unsigned long long qtail_cache = 0;             // the server's tail of it, as last seen
  unsigned long long rtail = hr->tail, rtail_pub = rtail;
  int outstanding = 0;
  // a ring never holds more than its share of the worker's credits: otherwise the first rings to run take
  // them all and most server warps idle (it matters for the lock stores, whose server path is per message)
  const int max_out = a.per_ring_cap > 0 ? min(a.per_ring_cap, a.resp.capacity) : a.resp.capacity;
  const int stride = a.req.stride;
  const bool lane_batches = stride <= FPS_BATCH_MAX_STRIDE;   // one lane moves one message
  unsigned long long n_pull = 0, n_push = 0, n_ans = 0;
  unsigned idle = 0;
  while (pos < end || outstanding > 0) {
    bool progressed = false;
    // ---- consume answers (and, in PULL_PUSH mode, send the pushes they trigger) -------------------------------
    if (outstanding > 0) {
      unsigned long long rhead = 0;
      if (lane == 0) rhead = ld_acquire_sys(&hr->head);
      rhead = __shfl_sync(0xffffffffu, rhead, 0);            // one observation for the whole warp
      while (rtail != rhead) {
        if (lane_batches) {
          const int n = (int)min((unsigned long long)32, rhead - rtail);
          const bool mine = lane < n;
          unsigned msg = 0;
          long long id = 0;
          if (mine) {
            Entry* e = ring_entry(a.resp, r, rtail + lane);
            msg = e->tag; id = e->id;
            const float* src = entry_payload(e);
            float* dst = a.out_vals + (size_t)msg * stride;
            for (int q = 0; q < stride; ++q) dst[q] = src[q];
          }
          if (a.mode == TXN_PULL_PUSH) {
            if (!ring_reserve_space(hq, qhead, n, a.req.capacity, &qtail_cache, lane, a.err)) return;
            if (mine)
              entry_write(ring_entry(a.req, r, qhead + lane), OP_PUSH, a.self, id, msg,
                          a.deltas + (size_t)msg * stride, stride);
            __syncwarp();
            qhead += n;
            if (lane == 0) st_release_sys(&hq->head, qhead);
            n_push += n;
          }
          rtail += n; outstanding -= n; n_ans += n;
          if (lane == 0) atomicAdd(a.credits, n);           // onPullRecv done: release the credits
        } else {
          Entry* e = ring_entry(a.resp, r, rtail);
          const unsigned msg = e->tag;
          const long long id = e->id;
          const float* src = entry_payload(e);
          for (int q = lane; q < stride; q += 32) a.out_vals[(size_t)msg * stride + q] = src[q];
          __syncwarp();
          ++rtail; --outstanding; ++n_ans;
          if (a.mode == TXN_PULL_PUSH) {
            if (!ring_put(a.req, r, OP_PUSH, a.self, id, msg, a.deltas + (size_t)msg * stride, lane, a.err,
                          &qtail_cache))
              return;
            ++n_push;
          }
          if (lane == 0) atomicAdd(a.credits, 1);
        }
        progressed = true;
      }
      if (lane == 0 && rtail != rtail_pub) {               // one release per drained batch of answers
        st_release_sys(&hr->tail, rtail);
        rtail_pub = rtail;
      }
    }
    // ---- issue the next messages ---------------------------------------------------------------------------------
    if (pos < end) {
      int k = min(lane_batches ? 32 : 1, end - pos);
      if (a.mode != TXN_PUSH_ONLY) {
        k = min(k, max_out - outstanding);
        int got = 0;
        if (lane == 0 && k > 0) {                            // one non-blocking attempt on the credit counter
          const int cur = *reinterpret_cast<volatile int*>(a.credits);
          const int take = min(k, cur);
          if (take > 0 && atomicCAS(a.credits, cur, cur - take) == cur) got = take;
        }
        k = __shfl_sync(0xffffffffu, got, 0);
      }
      if (k > 0) {
        const int op = a.mode == TXN_PUSH_ONLY ? OP_PUSH : OP_PULL;
        if (lane_batches) {
          if (!ring_reserve_space(hq, qhead, k, a.req.capacity, &qtail_cache, lane, a.err)) return;
          if (lane < k)
            entry_write(ring_entry(a.req, r, qhead + lane), op, a.self, a.ids[pos + lane], (unsigned)(pos + lane),
                        op == OP_PUSH ? a.deltas + (size_t)(pos + lane) * stride : nullptr, stride);
          __syncwarp();
          qhead += k;
          if (lane == 0) st_release_sys(&hq->head, qhead);
        } else {
          if (!ring_put(a.req, r, op, a.self, a.ids[pos], (unsigned)pos,
                        op == OP_PUSH ? a.deltas + (size_t)pos * stride : nullptr, lane, a.err, &qtail_cache))
            return;
        }
        pos += k;
        if (op == OP_PULL) { outstanding += k; n_pull += k; } else { n_push += k; }
        progressed = true;
      }
    }
    if (progressed) {
      idle = 0;
    } else {
      if (++idle > FPS_SPIN_LIMIT) { if (lane == 0) atomicExch(a.err, ERR_SPIN); return; }
      if (idle > 16) __nanosleep(128);
    }
  }
  if (lane == 0) {
    atomicAdd(a.counters + 0, n_pull);
    atomicAdd(a.counters + 1, n_push);
    atomicAdd(a.counters + 2, n_ans);
  }
}

extern "C" int fps_client_txn(const TxnArgs* a, cudaStream_t stream) {
  const int rings = a->req.n_peers * a->req.lanes;
  fps_client_txn_kernel<<<(rings + TXN_WARPS - 1) / TXN_WARPS, 32 * TXN_WARPS, 0, stream>>>(*a);
  return (int)cudaGetLastError();
}

extern "C" int fps_ring_entry_bytes(int stride) {
  int b = (int)sizeof(Entry) + 4 * stride;
  return (b + 15) / 16 * 16;
}
extern "C" int fps_ring_bytes(int capacity, int stride) {
  return (int)sizeof(RingHdr) + capacity * fps_ring_entry_bytes(stride);
}

// CUDA loads kernels lazily; the first launch of a not-yet-loaded kernel needs a context-wide
// synchronisation and therefore DEADLOCKS while a persistent kernel is resident.  Force-load every
// kernel of this file before the server starts.
extern "C" int fps_rings_preload() {
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncGetAttributes(&fa, fps_server_loop_kernel);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, fps_client_issue_kernel);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, fps_client_collect_kernel);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, fps_client_txn_kernel);
  return (int)e;
}
