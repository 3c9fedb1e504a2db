// K5: device-side negative sampling with a bounded per-user memory of recently seen items.
//
// Behaviour being reproduced (PSOnlineMatrixFactorizationWorker.scala:61-78): every incoming rating
// appends its item to the user's recent-items queue (bounded by `userMemory`, oldest evicted), then up
// to `negativeSampleRate` random items that are NOT in that memory are emitted as rating-0 training
// records ahead of the positive one.  Here the memory is a ring `seen[user_slot, memory]` in the
// worker's HBM and one warp handles one rating: the 32 lanes hold the ring in registers, every
// candidate drawn from the Philox stream (seed, step, position, negative, try) is tested against the
// ring with one ballot, and at most `max_tries` candidates are drawn per negative (the reference
// loops until it finds one; the bound keeps a pathological user from stalling the batch -- a
// negative that could not be found is emitted with user = -1 and skipped by the consumer).
//
// Output: expanded arrays [n_pos * (1 + neg_rate)], record p*(1+neg)+0 = the positive rating and
// +1.. = its negatives, directly consumable by fps_mf_sgd_fused (neg_rate = 0).
#include "fps_common.cuh"

#define NEG_MAX_PER_LANE 8  // memory <= 256

struct NegArgs {
  const void* users;
  const void* items;
  const float* ratings;
  long long n_pos;
  int neg_rate;
  int format;               // 0: arrays, 1: packed64 records in `users`
  long long num_items;
  unsigned long long seed;
  unsigned long long step;
  int* seen;                // [n_local_users, memory], -1 = empty
  int* seen_pos;            // [n_local_users] number of items ever appended (ring cursor)
  int memory;
  int user_div;
  int max_tries;
  int pad_;
  int* out_users;
  int* out_items;
  float* out_ratings;
};

template <typename IdT>
__global__ void __launch_bounds__(256) fps_neg_sample_kernel(const NegArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int per = 1 + a.neg_rate;
  for (long long pos = warp; pos < a.n_pos; pos += n_warps) {
    const FpsRecord<long long> rec = fps_record<IdT, long long>(a.format, a.users, a.items, a.ratings, pos);
    const long long user = rec.user, item = rec.item;
    const float rating = rec.rating;
    const long long slot = user / a.user_div;
    int* ring = a.seen + slot * a.memory;
    // append the positive item (ring cursor is bumped atomically: the same user may occur more
    // than once in a micro-batch, handled by different warps)
    int cur = 0;
    if (lane == 0) {
      cur = atomicAdd(a.seen_pos + slot, 1);
      ring[cur % a.memory] = (int)item;
    }
    __syncwarp();
    int mine[NEG_MAX_PER_LANE];
#pragma unroll
    for (int c = 0; c < NEG_MAX_PER_LANE; ++c) {
      const int q = lane + 32 * c;
      mine[c] = (q < a.memory) ? ring[q] : -1;
    }
    if (lane == 0) {
      a.out_users[pos * per] = (int)user;
      a.out_items[pos * per] = (int)item;
      a.out_ratings[pos * per] = rating;
    }
    for (int j = 1; j < per; ++j) {
      long long chosen = -1;
      for (int t = 0; t < a.max_tries && chosen < 0; t += 2) {
        // one Philox call yields two 64-bit candidates
        Philox4 s = fps_philox((uint32_t)pos, (uint32_t)((unsigned long long)pos >> 32),
                               (uint32_t)(j | (t << 8)), (uint32_t)a.step, (uint32_t)a.seed,
                               (uint32_t)(a.seed >> 32));
        const unsigned long long h0 = ((unsigned long long)s.x << 32) | s.y;
        const unsigned long long h1 = ((unsigned long long)s.z << 32) | s.w;
        const long long c0 = (long long)(h0 % (unsigned long long)a.num_items);
        const long long c1 = (long long)(h1 % (unsigned long long)a.num_items);
        bool hit0 = (c0 == item), hit1 = (c1 == item);
#pragma unroll
        for (int c = 0; c < NEG_MAX_PER_LANE; ++c) {
          hit0 |= (mine[c] == (int)c0);
          hit1 |= (mine[c] == (int)c1);
        }
        const bool any0 = __any_sync(0xffffffffu, hit0);
        const bool any1 = __any_sync(0xffffffffu, hit1);
        if (!any0) chosen = c0;
        else if (!any1 && t + 1 < a.max_tries) chosen = c1;
      }
      if (lane == 0) {
        a.out_users[pos * per + j] = chosen >= 0 ? (int)user : -1;
        a.out_items[pos * per + j] = chosen >= 0 ? (int)chosen : 0;
        a.out_ratings[pos * per + j] = 0.f;
      }
    }
  }
}

extern "C" int fps_neg_sample(const NegArgs* a, int id_bytes, int num_sms, cudaStream_t stream) {
  if (a->n_pos <= 0) return 0;
  if (a->memory < 1 || a->memory > 32 * NEG_MAX_PER_LANE) return -1101;
  long long blocks = (a->n_pos + 7) / 8;
  if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
  if (id_bytes == 8)
    fps_neg_sample_kernel<long long><<<(int)blocks, 256, 0, stream>>>(*a);
  else
    fps_neg_sample_kernel<int><<<(int)blocks, 256, 0, stream>>>(*a);
  return (int)cudaGetLastError();
}
