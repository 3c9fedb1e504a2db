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
// One cooperative kernel, no host synchronisation (fps_bucket_deal_kernel below): a histogram over the bucket
// ids, a grid sync, then a scatter in which each CTA reserves one contiguous run per bucket (shared-memory ranks
// + one global atomic per (CTA, bucket)).  Cost: read the batch from HBM once and from L2 once, write it once.
#include <cooperative_groups.h>
#include "fps_common.cuh"

namespace cg = cooperative_groups;

#define BK_MAX 64        // max buckets
#define BK_THREADS 256

struct BucketArgs {
  const void* users;   // format 0: ids; format 1: packed64 records (user:26 | item:22 | fp16 rating)
  const void* items;
  const float* ratings;
  long long n;
  int format;
  int id_bytes;        // 4 or 8 (format 0)
  int shift;           // bucket = row >> shift, row = owner(item) * rps + slot(item): the row index of the
  int n_buckets;       //   owner-major table the fused kernel reads (num_shards == 1: row == item)
  unsigned int* scratch;  // [2 * BK_MAX]: totals, cursors (zeroed by the kernel)
  void* out_users;
  void* out_items;
  float* out_ratings;
  long long rps;       // rows per owner segment
  int num_shards;      // owners (hash partition item % num_shards); 1 = plain item >> shift
  int shard_shift;     // log2(num_shards) or -1
  unsigned long long* pending;  // optional [num_shards]: += records per destination (device-side CountLogic feed)
};

__device__ __forceinline__ long long bk_item(const BucketArgs& a, long long i) {
  // not fps_record_item: its two instantiations behind a runtime id width cost this kernel 144 instructions
  if (a.format == 1)
    return (long long)((reinterpret_cast<const unsigned long long*>(a.users)[i] >> FPS_REC_ITEM_SHIFT) &
                       FPS_REC_ITEM_MASK);
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

// One cooperative launch per micro-batch.  Each CTA owns a contiguous chunk of the batch:
//   1. CTA 0 zeroes the counters while every CTA counts its chunk's buckets in shared memory;  grid sync;
//   2. the CTA counts go to the global totals (and the per-destination feed);  grid sync;
//   3. each CTA reserves one run per bucket (exclusive prefix of the totals + a cursor atomic) and re-reads its
//      chunk -- an L2 hit: the batch is a few MB -- to write every record at its run's next slot.
// Against a memset + histogram kernel + scatter kernel this reads the batch from HBM once and leaves two
// stream operations (and the launch gaps around them) out of every micro-batch.
__global__ void __launch_bounds__(BK_THREADS) fps_bucket_deal_kernel(const BucketArgs a, long long per_cta) {
  __shared__ unsigned int hist[BK_MAX];
  __shared__ unsigned int base[BK_MAX];
  __shared__ unsigned int ohist[FPS_MAX_SHARDS];
  cg::grid_group grid = cg::this_grid();
  if (threadIdx.x < BK_MAX) hist[threadIdx.x] = 0;
  if (threadIdx.x < FPS_MAX_SHARDS) ohist[threadIdx.x] = 0;
  if (blockIdx.x == 0 && threadIdx.x < 2 * BK_MAX) a.scratch[threadIdx.x] = 0;
  __syncthreads();
  const bool feed = a.pending != nullptr;
  const long long lo = (long long)blockIdx.x * per_cta;
  const long long hi = lo + per_cta < a.n ? lo + per_cta : a.n;
  for (long long i = lo + threadIdx.x; i < hi; i += BK_THREADS) {
    const long long item = bk_item(a, i);
    atomicAdd(&hist[bk_bucket(a, item)], 1u);
    if (feed) atomicAdd(&ohist[bk_owner(a, item)], 1u);
  }
  __syncthreads();
  grid.sync();
  if (threadIdx.x < a.n_buckets && hist[threadIdx.x] != 0)
    atomicAdd(a.scratch + threadIdx.x, hist[threadIdx.x]);
  if (feed && threadIdx.x < a.num_shards && ohist[threadIdx.x] != 0)
    atomicAdd(a.pending + threadIdx.x, (unsigned long long)ohist[threadIdx.x]);
  grid.sync();
  if (threadIdx.x < a.n_buckets) {
    unsigned int start = 0;  // exclusive prefix of the bucket totals
    for (int b = 0; b < threadIdx.x; ++b) start += a.scratch[b];
    const unsigned int mine = hist[threadIdx.x];
    base[threadIdx.x] = start + (mine ? atomicAdd(a.scratch + BK_MAX + threadIdx.x, mine) : 0u);
    hist[threadIdx.x] = 0;   // from here on: the next free slot of this CTA's run
  }
  __syncthreads();
  for (long long i = lo + threadIdx.x; i < hi; i += BK_THREADS) {
    const int b = bk_bucket(a, bk_item(a, i));
    const long long o = (long long)base[b] + atomicAdd(&hist[b], 1u);
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
  int occ = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fps_bucket_deal_kernel, BK_THREADS, 0);
  if (e != cudaSuccess) return (int)e;
  long long grid = (long long)num_sms * (occ < 4 ? occ : 4);   // every CTA must be resident (grid sync)
  const long long need = (a->n + BK_THREADS - 1) / BK_THREADS;
  if (grid > need) grid = need;
  if (grid < 1) grid = 1;
  long long per_cta = (a->n + grid - 1) / grid;
  BucketArgs args = *a;
  void* params[] = {&args, &per_cta};
  e = cudaLaunchCooperativeKernel((const void*)fps_bucket_deal_kernel, dim3((unsigned)grid), dim3(BK_THREADS),
                                  params, 0, stream);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaGetLastError();
}
