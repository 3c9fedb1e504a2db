// L2 blocking for the fused MF step: reorder a micro-batch so that ratings whose item rows live in the
// same slice of the item table are processed together.
//
// Why: one update touches a user row and an item row.  The user side is compulsory HBM traffic (10M
// users, every row read once and written once), but the item table (1M x 256 B = 256 MB) is hit ~4x
// per 4M-rating micro-batch and is five times the size of the 50 MB L2 of an H100: processed in arrival
// order most item reads miss and most REDG-dirtied lines are written back before their next use.
// Dealing the ratings into buckets of <= 16 MB of item rows (a third of the L2) turns the item side into
// one streaming pass per bucket.  Asynchronous
// SGD has no ordering contract inside a micro-batch (the reference's workers interleave arbitrarily),
// so the reordering is semantically free.
//
// Two streaming kernels, no host synchronisation: a histogram over the bucket ids, then a scatter in
// which each CTA reserves one contiguous run per bucket (shared-memory ranks + one global atomic per
// (CTA, bucket)).  Cost: read the batch twice, write it once (~100 MB for 4M packed records).
#include <cuda_fp16.h>
#include "fps_common.cuh"

#define BK_MAX 64        // max buckets
#define BK_THREADS 256
#define BK_PER_THREAD 8  // records per thread in the scatter kernel

struct BucketArgs {
  const void* users;   // format 0: ids; format 1: packed64 records (user:26 | item:22 | fp16 rating)
  const void* items;
  const float* ratings;
  long long n;
  int format;
  int id_bytes;        // 4 or 8 (format 0)
  int shift;           // bucket = row >> shift, row = owner(item) * rps + slot(item): the row index of the
  int n_buckets;       //   owner-major table the fused kernel reads (num_shards == 1: row == item)
  unsigned int* scratch;  // [2 * BK_MAX]: totals, cursors (zeroed by the launcher)
  void* out_users;
  void* out_items;
  float* out_ratings;
  long long rps;       // rows per owner segment
  int num_shards;      // owners (hash partition item % num_shards); 1 = plain item >> shift
  int shard_shift;     // log2(num_shards) or -1
  unsigned long long* pending;  // optional [num_shards]: += records per destination (device-side CountLogic feed)
};

__device__ __forceinline__ long long bk_item(const BucketArgs& a, long long i) {
  if (a.format == 1)
    return (long long)((reinterpret_cast<const unsigned long long*>(a.users)[i] >> 16) & 0x3FFFFFull);
  if (a.id_bytes == 8) return reinterpret_cast<const long long*>(a.items)[i];
  return (long long)reinterpret_cast<const int*>(a.items)[i];
}
__device__ __forceinline__ int bk_owner(const BucketArgs& a, long long item) {
  if (a.num_shards <= 1) return 0;
  const unsigned long long u = (unsigned long long)(item < 0 ? -item : item);
  return a.shard_shift >= 0 ? (int)(u & (unsigned long long)(a.num_shards - 1)) : (int)(u % (unsigned)a.num_shards);
}
__device__ __forceinline__ int bk_bucket(const BucketArgs& a, long long item) {
  long long row = item < 0 ? -item : item;
  if (a.num_shards > 1) {
    const unsigned long long u = (unsigned long long)row;
    const unsigned long long slot = a.shard_shift >= 0 ? (u >> a.shard_shift) : (u / (unsigned)a.num_shards);
    row = (long long)bk_owner(a, item) * a.rps + (long long)slot;
  }
  const long long b = row >> a.shift;
  return (int)(b < a.n_buckets ? b : a.n_buckets - 1);
}

__global__ void __launch_bounds__(BK_THREADS) fps_bucket_hist_kernel(const BucketArgs a) {
  __shared__ unsigned int hist[BK_MAX];
  __shared__ unsigned int ohist[FPS_MAX_SHARDS];
  if (threadIdx.x < BK_MAX) hist[threadIdx.x] = 0;
  if (threadIdx.x < FPS_MAX_SHARDS) ohist[threadIdx.x] = 0;
  __syncthreads();
  const bool feed = a.pending != nullptr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < a.n;
       i += (long long)gridDim.x * blockDim.x) {
    const long long item = bk_item(a, i);
    atomicAdd(&hist[bk_bucket(a, item)], 1u);
    if (feed) atomicAdd(&ohist[bk_owner(a, item)], 1u);
  }
  __syncthreads();
  if (threadIdx.x < a.n_buckets && hist[threadIdx.x] != 0)
    atomicAdd(a.scratch + threadIdx.x, hist[threadIdx.x]);
  if (feed && threadIdx.x < a.num_shards && ohist[threadIdx.x] != 0)
    atomicAdd(a.pending + threadIdx.x, (unsigned long long)ohist[threadIdx.x]);
}

__global__ void __launch_bounds__(BK_THREADS) fps_bucket_scatter_kernel(const BucketArgs a) {
  __shared__ unsigned int hist[BK_MAX];
  __shared__ unsigned int base[BK_MAX];
  if (threadIdx.x < BK_MAX) hist[threadIdx.x] = 0;
  __syncthreads();
  const long long chunk0 = (long long)blockIdx.x * (BK_THREADS * BK_PER_THREAD);
  int bucket[BK_PER_THREAD];
  unsigned int rank[BK_PER_THREAD];
#pragma unroll
  for (int u = 0; u < BK_PER_THREAD; ++u) {
    const long long i = chunk0 + u * BK_THREADS + threadIdx.x;
    bucket[u] = -1;
    if (i < a.n) {
      bucket[u] = bk_bucket(a, bk_item(a, i));
      rank[u] = atomicAdd(&hist[bucket[u]], 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x < a.n_buckets) {
    unsigned int start = 0;  // exclusive prefix of the bucket totals
    for (int b = 0; b < threadIdx.x; ++b) start += a.scratch[b];
    const unsigned int mine = hist[threadIdx.x];
    base[threadIdx.x] = start + (mine ? atomicAdd(a.scratch + BK_MAX + threadIdx.x, mine) : 0u);
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < BK_PER_THREAD; ++u) {
    if (bucket[u] < 0) continue;
    const long long i = chunk0 + u * BK_THREADS + threadIdx.x;
    const long long o = (long long)base[bucket[u]] + rank[u];
    if (a.format == 1) {
      reinterpret_cast<unsigned long long*>(a.out_users)[o] =
          reinterpret_cast<const unsigned long long*>(a.users)[i];
    } else {
      if (a.id_bytes == 8) {
        reinterpret_cast<long long*>(a.out_users)[o] = reinterpret_cast<const long long*>(a.users)[i];
        reinterpret_cast<long long*>(a.out_items)[o] = reinterpret_cast<const long long*>(a.items)[i];
      } else {
        reinterpret_cast<int*>(a.out_users)[o] = reinterpret_cast<const int*>(a.users)[i];
        reinterpret_cast<int*>(a.out_items)[o] = reinterpret_cast<const int*>(a.items)[i];
      }
      a.out_ratings[o] = a.ratings[i];
    }
  }
}

extern "C" int fps_bucket_by_item(const BucketArgs* a, int num_sms, cudaStream_t stream) {
  if (a->n <= 0) return 0;
  if (a->n_buckets < 1 || a->n_buckets > BK_MAX || a->n >= (1ll << 32)) return -1301;
  cudaError_t e = cudaMemsetAsync(a->scratch, 0, 2 * BK_MAX * sizeof(unsigned int), stream);
  if (e != cudaSuccess) return (int)e;
  long long hb = (a->n + BK_THREADS - 1) / BK_THREADS;
  if (hb > (long long)num_sms * 8) hb = (long long)num_sms * 8;
  fps_bucket_hist_kernel<<<(int)hb, BK_THREADS, 0, stream>>>(*a);
  const long long per = BK_THREADS * BK_PER_THREAD;
  fps_bucket_scatter_kernel<<<(int)((a->n + per - 1) / per), BK_THREADS, 0, stream>>>(*a);
  return (int)cudaGetLastError();
}
