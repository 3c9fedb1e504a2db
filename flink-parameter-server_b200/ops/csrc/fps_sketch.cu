// K8-K10: streaming-sketch updates fused with the push (one-sided reductions on the owner's HBM).
//
//   Bloom      : bitmap[key][pos >> 5] |= 1 << (pos & 31)        red.global.or.b32
//                (BloomPSLogic.scala:16-22: set bits)
//   tug-of-war : counter[key][j] += bit_j ? +1 : -1               red.global.add.s32
//                (BitSetBasedPSLogic.scala:14-25)
//   MinHash    : sig[key][j] = min(sig[key][j], hash_j(tweet) << 32 | tweet)   red.global.min.u64
//                (SendHashPSLogic.scala:17-40: keep the tweet with the smaller hash per slot)
//   Bloom query: est[key] = n(A) + n(B) - n(A u B), n(X) = -m/k ln(1 - |X|/m)   (popcount scan)
//                (BloomPredictPSLogic.scala:47-58, Utils.scala:29-43)
//
// Keys are dense slot ids produced by the host-side interning dictionary; rows live in a ShardTable
// whose 4-byte cells are reinterpreted as u32 / s32 / u64.  hash64 is the same seeded mixer as
// models/sketch/hashing.py::hash64, so host and device sketches agree bit for bit.
#include "fps_common.cuh"

__host__ __device__ __forceinline__ unsigned long long fps_hash64(unsigned long long x,
                                                                  unsigned long long seed) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull * (seed + 1ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

enum FpsSketchKind : int { SK_BLOOM = 0, SK_TOW = 1, SK_MINHASH = 2 };

template <int KIND>
__global__ void __launch_bounds__(256)
    fps_sketch_update_kernel(const __grid_constant__ ShardTable t, const int* __restrict__ keys,
                             const long long* __restrict__ tweets, long long n, int num_hashes,
                             int array_size) {
  const long long total = n * (long long)num_hashes;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < total;
       g += (long long)gridDim.x * blockDim.x) {
    const long long rec = g / num_hashes;
    const int j = (int)(g - rec * num_hashes);
    const unsigned long long tw = (unsigned long long)tweets[rec];
    unsigned int* row = reinterpret_cast<unsigned int*>(fps_row32(t, keys[rec]));
    if (KIND == SK_BLOOM) {
      const unsigned int pos = (unsigned int)(fps_hash64(tw, (unsigned long long)j) %
                                              (unsigned long long)array_size);
      asm volatile("red.relaxed.sys.global.or.b32 [%0], %1;" ::"l"(row + (pos >> 5)),
                   "r"(1u << (pos & 31))
                   : "memory");
    } else if (KIND == SK_TOW) {
      const unsigned long long h = fps_hash64(tw, (unsigned long long)(j >> 6));
      const int d = ((h >> (j & 63)) & 1ull) ? 1 : -1;
      asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(row + j), "r"(d) : "memory");
    } else {
      const unsigned long long h = fps_hash64(tw, (unsigned long long)j) >> 32;
      const unsigned long long packed = (h << 32) | (tw & 0xFFFFFFFFull);
      asm volatile("red.relaxed.sys.global.min.u64 [%0], %1;" ::"l"(
                       reinterpret_cast<unsigned long long*>(row) + j),
                   "l"(packed)
                   : "memory");
    }
  }
}

extern "C" int fps_sketch_update(const ShardTable* t, int kind, const int* keys,
                                 const long long* tweets, long long n, int num_hashes,
                                 int array_size, int num_sms, cudaStream_t stream) {
  if (n <= 0) return 0;
  long long total = n * (long long)num_hashes;
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)num_sms * 16) blocks = (long long)num_sms * 16;
  const int g = (int)blocks;
  if (kind == SK_BLOOM)
    fps_sketch_update_kernel<SK_BLOOM><<<g, 256, 0, stream>>>(*t, keys, tweets, n, num_hashes, array_size);
  else if (kind == SK_TOW)
    fps_sketch_update_kernel<SK_TOW><<<g, 256, 0, stream>>>(*t, keys, tweets, n, num_hashes, array_size);
  else if (kind == SK_MINHASH)
    fps_sketch_update_kernel<SK_MINHASH><<<g, 256, 0, stream>>>(*t, keys, tweets, n, num_hashes, array_size);
  else
    return -1007;
  return (int)cudaGetLastError();
}

// one warp per local key: popcount(B) and popcount(B | Q)
__global__ void __launch_bounds__(256)
    fps_bloom_query_kernel(const unsigned int* __restrict__ local_rows, long long n_rows, int stride_words,
                           int n_words, const unsigned int* __restrict__ query, float m, float k,
                           const int* __restrict__ key_slot, int query_slot, float* __restrict__ est) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += n_warps) {
    if (key_slot != nullptr && key_slot[r] != query_slot) {   // time-aware: same-slot keys only
      if (lane == 0) est[r] = -3.0e38f;
      continue;
    }
    const unsigned int* row = local_rows + r * (long long)stride_words;
    int cb = 0, cu = 0, cq = 0;
    for (int w = lane; w < n_words; w += 32) {
      const unsigned int b = row[w], q = query[w];
      cb += __popc(b); cu += __popc(b | q); cq += __popc(q);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      cb += __shfl_xor_sync(0xffffffffu, cb, o);
      cu += __shfl_xor_sync(0xffffffffu, cu, o);
      cq += __shfl_xor_sync(0xffffffffu, cq, o);
    }
    if (lane == 0) {
      // bloomEq in fp64, as the reference computes it.  In float, c/m is rounded before 1 - c/m when m is not a
      // power of two, and at small c that error dominates the log (1% at m = 1000003).  Three logs on one lane
      // per row, after a popcount pass over the whole row.
      const double md = m, kd = k;
      const double nA = -md / kd * log(1.0 - (double)cq / md);
      const double nB = -md / kd * log(1.0 - (double)cb / md);
      const double nU = -md / kd * log(1.0 - (double)cu / md);
      const double e = nA + nB - nU;
      // empty rows are not keys; a saturated filter makes some n(X) infinite and e NaN or -inf: not a key either
      est[r] = (cb == 0 || !isfinite(e)) ? -3.0e38f : (float)e;
    }
  }
}

extern "C" int fps_bloom_query(const unsigned int* local_rows, long long n_rows, int stride_words,
                               int n_words, const unsigned int* query, float m, float k,
                               const int* key_slot, int query_slot, float* est,
                               int num_sms, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  long long blocks = (n_rows * 32 + 255) / 256;
  if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
  fps_bloom_query_kernel<<<(int)blocks, 256, 0, stream>>>(local_rows, n_rows, stride_words, n_words,
                                                          query, m, k, key_slot, query_slot, est);
  return (int)cudaGetLastError();
}

// ----------------------------------------------------------------------------------------
// K9 query: tug-of-war co-occurrence estimate = MEDIAN over `num_means` groups of the MEAN slice
// dot-product of the int32 counters (SketchPredictPSLogic.scala:23-40).  One warp per local key;
// lane g keeps the mean of group g, the median is found by rank counting over shuffles.
// K10 query: MinHash Jaccard estimate = fraction of signature slots holding the same tweet id
// (MinHashPredictPSLogic.scala:33-36), optionally converted to a co-occurrence count with the word
// frequencies, Math.round(J * (f_q + f_w) / (J + 1)) in double  (MinHashPredict.scala:60-141 Aggregate).
// Time-aware variants (TimeAwareToWPredictPSLogic.scala, TimeAwareBloomPredictPSLogic.scala:19-27): keys
// are (word, timeSlot); `key_slot[r] != query_slot` rows are excluded from the scan.
// ----------------------------------------------------------------------------------------
#define SK_NEG_INF (-3.0e38f)

__global__ void __launch_bounds__(256)
    fps_tow_query_kernel(const int* __restrict__ rows, long long n_rows, int stride_words, int n_hashes,
                         int num_means, const int* __restrict__ query, const int* __restrict__ key_slot,
                         int query_slot, float* __restrict__ est) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int size = max(1, (n_hashes + num_means - 1) / num_means);
  const int m = (n_hashes + size - 1) / size;   // groups actually formed (<= 32)
  for (long long r = warp; r < n_rows; r += n_warps) {
    if (key_slot != nullptr && key_slot[r] != query_slot) {
      if (lane == 0) est[r] = SK_NEG_INF;
      continue;
    }
    const int* row = rows + r * (long long)stride_words;
    double mine = 0.0;
    for (int g = 0; g < m; ++g) {
      const int lo = g * size, hi = min(n_hashes, lo + size);
      long long acc = 0;
      for (int j = lo + lane; j < hi; j += 32) acc += (long long)row[j] * (long long)query[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == g) mine = (double)acc / (double)(hi - lo);
    }
    const bool valid = lane < m;
    int rank = 0;                                   // position in DESCENDING order, ties by lane
    for (int k = 0; k < m; ++k) {
      const double vk = __shfl_sync(0xffffffffu, mine, k);
      if (valid && (vk > mine || (vk == mine && k < lane))) ++rank;
    }
    double c = 0.0;
    if (valid && rank == m / 2) c += mine;
    if (valid && (m & 1) == 0 && rank == m / 2 - 1) c += mine;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) est[r] = (float)((m & 1) == 0 ? 0.5 * c : c);
  }
}

__global__ void __launch_bounds__(256)
    fps_minhash_query_kernel(const unsigned long long* __restrict__ rows, long long n_rows,
                             int stride_u64, int n_hashes, const unsigned long long* __restrict__ query,
                             const int* __restrict__ key_slot, int query_slot,
                             const float* __restrict__ freq, float query_freq, float* __restrict__ est) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += n_warps) {
    if (key_slot != nullptr && key_slot[r] != query_slot) {
      if (lane == 0) est[r] = SK_NEG_INF;
      continue;
    }
    const unsigned long long* row = rows + r * (long long)stride_u64;
    int eq = 0, filled = 0, qfilled = 0;
    for (int j = lane; j < n_hashes; j += 32) {
      const unsigned long long a = row[j], b = query[j];
      filled += a != ~0ull;
      qfilled += b != ~0ull;
      eq += (a != ~0ull) && (b != ~0ull) && ((unsigned int)a == (unsigned int)b);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      eq += __shfl_xor_sync(0xffffffffu, eq, o);
      filled += __shfl_xor_sync(0xffffffffu, filled, o);
      qfilled += __shfl_xor_sync(0xffffffffu, qfilled, o);
    }
    if (lane == 0) {
      const bool both = filled != 0 && qfilled != 0;
      float s;
      if (filled == 0) {
        s = SK_NEG_INF;                                        // not a key of this shard
      } else if (freq != nullptr) {
        // Math.round((J * (f_q + f_r)) / (J + 1)) on doubles, in the reference's order: halves round up
        const double J = both ? (double)eq / (double)n_hashes : 0.0;
        const double x = J * ((double)query_freq + (double)freq[r]) / (J + 1.0);
        const double f = floor(x);
        s = (float)(x - f >= 0.5 ? f + 1.0 : f);
      } else {
        s = both ? (float)eq / (float)n_hashes : 0.f;
      }
      est[r] = s;
    }
  }
}

extern "C" int fps_sketch_query(int kind, const void* rows, long long n_rows, int stride_words, int n_hashes,
                                int num_means, const void* query, const int* key_slot, int query_slot,
                                const float* freq, float query_freq, float* est, int num_sms,
                                cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  long long blocks = (n_rows * 32 + 255) / 256;
  if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
  if (kind == SK_TOW) {
    if (num_means < 1) num_means = 1;
    const int size = (n_hashes + num_means - 1) / num_means;
    if ((n_hashes + size - 1) / size > 32) return -1008;   // more than 32 groups: not supported on the device
    fps_tow_query_kernel<<<(int)blocks, 256, 0, stream>>>((const int*)rows, n_rows, stride_words, n_hashes,
                                                          num_means, (const int*)query, key_slot, query_slot, est);
  } else if (kind == SK_MINHASH) {
    fps_minhash_query_kernel<<<(int)blocks, 256, 0, stream>>>(
        (const unsigned long long*)rows, n_rows, stride_words / 2, n_hashes, (const unsigned long long*)query,
        key_slot, query_slot, freq, query_freq, est);
  } else {
    return -1007;
  }
  return (int)cudaGetLastError();
}
