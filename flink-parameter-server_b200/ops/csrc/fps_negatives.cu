// Negative sampling over a draw domain other than the whole id range.  Output layout as in fps_sampler.cu:
// expanded records [n_pos * (1 + neg_rate)], record p*(1+neg)+0 the positive, +1.. its negatives at rating 0,
// a negative that was not drawn or not found voided with user = -1; fps_mf_sgd_fused (neg_rate = 0) and the
// BPR kernel's explicit negatives consume them as they are.
//
// Two domains, two kernels:
//
// * fps_neg_seen_kernel -- the items this worker has seen so far (PSOnlineMatrixFactorizationWorker.scala:61-88,
//   ops/csrc/fps_host.cpp:216-249).  A device registry holds them in first-occurrence order (`order`, `count`).
//   Record p of a micro-batch draws from D_p = order[0 : count_before + (items first seen in this batch at
//   positions < p)]: its own first-seen item is not in its domain, the next record's domain holds it.  It draws
//   max(0, min(|D_p| - |ring_p|, neg_rate)) negatives, each a Philox index into D_p rejected against the
//   user's recent-items ring (kept exactly as K5 keeps it) and the positive, at most `max_tries` times.
//   One cooperative launch: per-item minimum position (atomicMin), grid sync, first-occurrence flags scanned
//   per CTA, grid sync, append to `order`, grid sync, draw.
// * fps_neg_noise_kernel -- a fixed weighted domain (skip-gram unigram noise): an fp64 inverse CDF built once
//   by fps_noise_cdf, a 53-bit Philox uniform and an upper-bound binary search; the positive is rejected.
//
// Draws are keyed (position, negative, try, step, seed) as in K5: the output depends on the seed, the step and
// the stream, never on the grid.
#include <cooperative_groups.h>
#include <limits.h>
#include "fps_common.cuh"

namespace cg = cooperative_groups;

#define NS_THREADS 256
#define NS_MAX_PER_LANE 8     // ring memory <= 256
#define NS_CDF_CHUNK 256      // words per thread of the CDF's first pass

struct NegDomainArgs {
  const void* users;
  const void* items;
  const float* ratings;
  long long n_pos;
  int neg_rate;
  int format;               // 0: arrays, 1: packed64 records in `users`
  unsigned long long seed;
  unsigned long long step;
  int max_tries;
  // seen-items registry
  int memory;               // 0: no recent-items ring
  int* seen;                // [n_local_users, memory] ring, -1 = empty
  int* seen_pos;            // [n_local_users] items ever appended (ring cursor)
  int user_div;
  int cta_cap;              // entries of cta_new
  long long num_items;      // registry capacity; ids outside [0, num_items) never enter it
  int* order;               // [num_items] ids in first-occurrence order
  int* count;               // [1] ids in `order`
  int* first_pos;           // [num_items] -1: in the registry, INT_MAX: unseen, else min position in this batch
  int* scratch;             // [n_pos] 2 * (first occurrences before it in its CTA) + its own flag
  int* cta_new;             // [cta_cap] first occurrences per CTA
  // weighted domain
  const double* cdf;        // [vocab] inclusive prefix sums of the weights
  long long vocab;
  long long last_nonzero;   // the last word of positive weight
  int* out_users;
  int* out_items;
  float* out_ratings;
};

template <typename IdT>
__device__ __forceinline__ long long ns_item(const NegDomainArgs& a, long long pos) {
  return fps_record_item<IdT>(a.format, a.users, a.items, pos);
}

// Two 64-bit hashes of try t (and t + 1) of negative j of record pos.
__device__ __forceinline__ void ns_hash(const NegDomainArgs& a, long long pos, int j, int t, unsigned long long& h0,
                                        unsigned long long& h1) {
  const Philox4 s = fps_philox((uint32_t)pos, (uint32_t)((unsigned long long)pos >> 32), (uint32_t)(j | (t << 8)),
                               (uint32_t)a.step, (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  h0 = ((unsigned long long)s.x << 32) | s.y;
  h1 = ((unsigned long long)s.z << 32) | s.w;
}

// ---- seen-items registry ------------------------------------------------------------------------------------
template <typename IdT>
__global__ void __launch_bounds__(NS_THREADS) fps_neg_seen_kernel(const NegDomainArgs a, long long per_cta) {
  __shared__ int warp_sum[NS_THREADS / 32];
  __shared__ int carry_s;
  __shared__ int cta_off_s;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long lo = (long long)blockIdx.x * per_cta;
  const long long hi = lo + per_cta < a.n_pos ? lo + per_cta : a.n_pos;
  const int count_before = *a.count;   // read by every CTA before CTA 0 rewrites it (after the second sync)

  // 1. the first position of every item not yet in the registry
  for (long long i = lo + threadIdx.x; i < hi; i += NS_THREADS) {
    const long long item = ns_item<IdT>(a, i);
    if (item >= 0 && item < a.num_items && a.first_pos[item] > (int)i) atomicMin(a.first_pos + item, (int)i);
  }
  grid.sync();

  // 2. flag each record holding its item's first occurrence; exclusive scan of the flags over the CTA's chunk
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (long long t0 = lo; t0 < hi; t0 += NS_THREADS) {
    const long long i = t0 + threadIdx.x;
    bool flag = false;
    if (i < hi) {
      const long long item = ns_item<IdT>(a, i);
      flag = item >= 0 && item < a.num_items && a.first_pos[item] == (int)i;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_sum[wid] = __popc(bal);
    __syncthreads();
    int before = carry_s + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < wid; ++w) before += warp_sum[w];
    if (i < hi) a.scratch[i] = 2 * before + (flag ? 1 : 0);
    __syncthreads();
    if (threadIdx.x == 0) {
      int s = 0;
      for (int w = 0; w < NS_THREADS / 32; ++w) s += warp_sum[w];
      carry_s += s;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) a.cta_new[blockIdx.x] = carry_s;
  grid.sync();

  // 3. the CTA's offset among this batch's new items; append them and mark them registered
  if (wid == 0) {
    int s = 0;
    for (int b = lane; b < (int)blockIdx.x; b += 32) s += a.cta_new[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) cta_off_s = s;
    if (blockIdx.x == 0) {
      int tot = 0;
      for (int b = lane; b < (int)gridDim.x; b += 32) tot += a.cta_new[b];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      if (lane == 0) *a.count = count_before + tot;
    }
  }
  __syncthreads();
  const int base = count_before + cta_off_s;
  for (long long i = lo + threadIdx.x; i < hi; i += NS_THREADS) {
    const int sc = a.scratch[i];
    if (sc & 1) {
      const long long item = ns_item<IdT>(a, i);
      a.order[base + (sc >> 1)] = (int)item;
      a.first_pos[item] = -1;
    }
  }
  grid.sync();

  // 4. one warp per record: append the positive to the user's ring, then draw from D_p
  const int per = 1 + a.neg_rate;
  for (long long pos = lo + wid; pos < hi; pos += NS_THREADS / 32) {
    const FpsRecord<long long> rec = fps_record<IdT, long long>(a.format, a.users, a.items, a.ratings, pos);
    const long long user = rec.user, item = rec.item;
    const float rating = rec.rating;
    const long long dom = (long long)base + (a.scratch[pos] >> 1);
    int mine[NS_MAX_PER_LANE];
    int ring_len = 0;
    if (a.memory > 0) {
      int* ring = a.seen + (user / a.user_div) * a.memory;
      int cur = 0;
      if (lane == 0) {
        cur = atomicAdd(a.seen_pos + user / a.user_div, 1);
        ring[cur % a.memory] = (int)item;
      }
      cur = __shfl_sync(0xffffffffu, cur, 0);
      ring_len = cur + 1 < a.memory ? cur + 1 : a.memory;
      __syncwarp();
#pragma unroll
      for (int c = 0; c < NS_MAX_PER_LANE; ++c) {
        const int q = lane + 32 * c;
        mine[c] = (q < a.memory) ? ring[q] : -1;
      }
    } else {
#pragma unroll
      for (int c = 0; c < NS_MAX_PER_LANE; ++c) mine[c] = -1;
    }
    long long n_draw = dom - ring_len;
    if (n_draw > a.neg_rate) n_draw = a.neg_rate;
    if (lane == 0) {
      a.out_users[pos * per] = (int)user;
      a.out_items[pos * per] = (int)item;
      a.out_ratings[pos * per] = rating;
    }
    for (int j = 1; j < per; ++j) {
      long long chosen = -1;
      for (int t = 0; j <= n_draw && t < a.max_tries && chosen < 0; t += 2) {
        unsigned long long h0, h1;
        ns_hash(a, pos, j, t, h0, h1);
        const long long c0 = a.order[h0 % (unsigned long long)dom];
        const long long c1 = a.order[h1 % (unsigned long long)dom];
        bool hit0 = (c0 == item), hit1 = (c1 == item);
#pragma unroll
        for (int c = 0; c < NS_MAX_PER_LANE; ++c) {
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

extern "C" int fps_neg_sample_seen(const NegDomainArgs* a, int id_bytes, int num_sms, cudaStream_t stream) {
  if (a->n_pos <= 0) return 0;
  if (a->memory < 0 || a->memory > 32 * NS_MAX_PER_LANE || a->n_pos >= INT_MAX || a->num_items >= INT_MAX ||
      a->cta_cap < 1)
    return -1401;
  const void* fn = id_bytes == 8 ? (const void*)fps_neg_seen_kernel<long long> : (const void*)fps_neg_seen_kernel<int>;
  int occ = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, NS_THREADS, 0);
  if (e != cudaSuccess) return (int)e;
  long long grid = (long long)num_sms * occ;   // every CTA must be resident (grid sync)
  const long long need = (a->n_pos + NS_THREADS - 1) / NS_THREADS;
  if (grid > need) grid = need;
  if (grid > a->cta_cap) grid = a->cta_cap;
  if (grid < 1) grid = 1;
  long long per_cta = (a->n_pos + grid - 1) / grid;
  NegDomainArgs args = *a;
  void* params[] = {&args, &per_cta};
  e = cudaLaunchCooperativeKernel(fn, dim3((unsigned)grid), dim3(NS_THREADS), params, 0, stream);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaGetLastError();
}

// ---- fixed weighted domain ----------------------------------------------------------------------------------
// Inverse CDF of w = count ** power (w = 0 where count = 0), in fp64.  Each thread scans NS_CDF_CHUNK words in
// order, one thread then chains the chunk totals, and every word gets its chunk's offset added.  Every prefix
// is a left-to-right sum, so a word of weight 0 has exactly its predecessor's prefix and is never drawn.
__global__ void fps_noise_cdf_local(const double* __restrict__ counts, long long n, double power,
                                    double* __restrict__ cdf, double* __restrict__ totals) {
  const long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long lo = c * NS_CDF_CHUNK;
  if (lo >= n) return;
  const long long hi = lo + NS_CDF_CHUNK < n ? lo + NS_CDF_CHUNK : n;
  double s = 0.0;
  for (long long i = lo; i < hi; ++i) {
    const double x = counts[i];
    s += x > 0.0 ? pow(x, power) : 0.0;
    cdf[i] = s;
  }
  totals[c] = s;
}

__global__ void fps_noise_cdf_chain(double* totals, long long n_chunks) {
  double off = 0.0;
  for (long long c = 0; c < n_chunks; ++c) {
    const double t = totals[c];
    totals[c] = off;
    off = off + t;
  }
}

__global__ void fps_noise_cdf_offset(double* __restrict__ cdf, long long n, const double* __restrict__ offsets) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    cdf[i] = offsets[i / NS_CDF_CHUNK] + cdf[i];
}

extern "C" int fps_noise_cdf(const double* counts, long long n, double power, double* cdf, double* totals,
                             cudaStream_t stream) {
  if (n <= 0) return -1401;
  const long long n_chunks = (n + NS_CDF_CHUNK - 1) / NS_CDF_CHUNK;
  fps_noise_cdf_local<<<(unsigned)((n_chunks + 127) / 128), 128, 0, stream>>>(counts, n, power, cdf, totals);
  fps_noise_cdf_chain<<<1, 1, 0, stream>>>(totals, n_chunks);
  long long blocks = (n + 255) / 256;
  if (blocks > 4096) blocks = 4096;
  fps_noise_cdf_offset<<<(unsigned)blocks, 256, 0, stream>>>(cdf, n, totals);
  return (int)cudaGetLastError();
}

// One thread per output record: j == 0 copies the positive, j >= 1 draws negative j.
template <typename IdT>
__global__ void __launch_bounds__(NS_THREADS) fps_neg_noise_kernel(const NegDomainArgs a) {
  const int per = 1 + a.neg_rate;
  const long long n_out = a.n_pos * per;
  const double total = a.cdf[a.vocab - 1];
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < n_out;
       o += (long long)gridDim.x * blockDim.x) {
    const long long pos = o / per;
    const int j = (int)(o - pos * per);
    const FpsRecord<long long> rec = fps_record<IdT, long long>(a.format, a.users, a.items, a.ratings, pos);
    const long long user = rec.user, item = rec.item;
    const float rating = rec.rating;
    if (j == 0) {
      a.out_users[o] = (int)user;
      a.out_items[o] = (int)item;
      a.out_ratings[o] = rating;
      continue;
    }
    long long chosen = -1;
    for (int t = 0; t < a.max_tries && chosen < 0; t += 2) {
      unsigned long long h[2];
      ns_hash(a, pos, j, t, h[0], h[1]);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        if (chosen >= 0 || t + q >= a.max_tries) continue;
        const double x = (double)(h[q] >> 11) * 0x1.0p-53 * total;
        long long l = 0, r = a.vocab;       // the first word whose prefix exceeds x
        while (l < r) {
          const long long m = (l + r) >> 1;
          if (a.cdf[m] > x) r = m;
          else l = m + 1;
        }
        const long long c = l < a.vocab ? l : a.last_nonzero;   // x rounded up to the total
        if (c != item) chosen = c;
      }
    }
    a.out_users[o] = chosen >= 0 ? (int)user : -1;
    a.out_items[o] = chosen >= 0 ? (int)chosen : 0;
    a.out_ratings[o] = 0.f;
  }
}

extern "C" int fps_neg_sample_noise(const NegDomainArgs* a, int id_bytes, int num_sms, cudaStream_t stream) {
  if (a->n_pos <= 0) return 0;
  if (a->vocab < 1 || a->last_nonzero < 0 || a->last_nonzero >= a->vocab) return -1401;
  const long long n_out = a->n_pos * (1 + a->neg_rate);
  long long blocks = (n_out + NS_THREADS - 1) / NS_THREADS;
  if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
  if (id_bytes == 8)
    fps_neg_noise_kernel<long long><<<(int)blocks, NS_THREADS, 0, stream>>>(*a);
  else
    fps_neg_noise_kernel<int><<<(int)blocks, NS_THREADS, 0, stream>>>(*a);
  return (int)cudaGetLastError();
}
