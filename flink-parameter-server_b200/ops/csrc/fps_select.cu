// Row-wise selection kernels for the top-K paths (K6 "radix select for top-K", K12 "device K-way merge"):
//
//   fps_row_kth   : K-th largest value of every row            (theta of the two-pass tensor-core top-K,
//                   and the tightened theta of an overflowing candidate buffer)
//   fps_row_topk  : sorted top-K (score, item) of every row's candidate list / concatenated partial
//                   lists (CollectTopKFromEachWorker.scala:41-56 without the host round trip)
//
// Both take optional per-row arguments for the seen-item filter of the generators: fps_row_kth a
// per-row k (the (K + E_q)-th tile maximum is the bound when E_q items of row q are excluded), and
// fps_row_topk an exclusion list per row in CSR form (offsets [n_rows+1], items sorted and
// de-duplicated within each row).  An excluded candidate is found by binary search and never enters
// the radix select or the sort; the plain instantiation of fps_row_topk is the code without the lookup.
//
// One CTA per row.  Selection is an MSD radix select over order-preserving 32-bit keys (4 passes of 8
// bits, per-warp shared-memory histograms), so the cost is O(n) per row regardless of K -- torch.topk
// on the same shapes was the largest term of the top-K pipeline (profiles/topk_mma.md).  The final
// <= 2K survivors are ordered by a shared-memory bitonic sort on (score, -item) composite keys, which
// also makes the order among equal scores deterministic (smaller item id first).
#include "fps_common.cuh"

#define SEL_THREADS 256
#define SEL_WARPS (SEL_THREADS / 32)
#define SEL_STAGE_MAX 40960   // rows up to this many floats are staged in shared memory (160 KB)

__device__ __forceinline__ uint32_t sel_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float sel_unkey(uint32_t k) {
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
  return __uint_as_float(u);
}

// Key of the k-th largest (k is 1-based, 1 <= k <= n) of key_at(0..n).  Block-wide; all threads return it.
template <class KeyAt>
__device__ uint32_t sel_block_kth_key(KeyAt key_at, int n, int k, uint32_t* hist /*[SEL_WARPS*256]*/,
                                      uint32_t* bcast /*[2]*/) {
  uint32_t prefix = 0, mask = 0;
  uint32_t krem = (uint32_t)k;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < SEL_WARPS * 256; i += SEL_THREADS) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += SEL_THREADS) {
      const uint32_t key = key_at(i);
      if ((key & mask) == prefix) atomicAdd(&hist[warp * 256 + ((key >> shift) & 0xFFu)], 1u);
    }
    __syncthreads();
    {
      uint32_t s = 0;
#pragma unroll
      for (int w = 0; w < SEL_WARPS; ++w) s += hist[w * 256 + threadIdx.x];
      hist[threadIdx.x] = s;  // thread t is the only reader / writer of column t
    }
    __syncthreads();
    if (warp == 0) {  // descending scan: lane l owns bins 255-8l .. 248-8l
      uint32_t c[8], tot = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = hist[255 - (lane * 8 + j)];
        tot += c[j];
      }
      uint32_t incl = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const uint32_t excl = incl - tot;
      if (excl < krem && krem <= incl) {
        uint32_t run = excl;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (run + c[j] >= krem) {
            bcast[0] = (uint32_t)(255 - (lane * 8 + j));
            bcast[1] = krem - run;
            break;
          }
          run += c[j];
        }
      }
    }
    __syncthreads();
    prefix |= bcast[0] << shift;
    mask |= 0xFFu << shift;
    krem = bcast[1];
    __syncthreads();
  }
  return prefix;
}

__device__ __forceinline__ uint32_t sel_block_kth_key(const float* src, int n, int k, uint32_t* hist,
                                                      uint32_t* bcast) {
  return sel_block_kth_key([src](int i) { return sel_key(src[i]); }, n, k, hist, bcast);
}

// Is `item` in the sorted list ex[0..n)?  (lower_bound)
__device__ __forceinline__ bool sel_excluded(const int* __restrict__ ex, int n, int item) {
  const int* end = ex + n;
  while (n > 0) {
    const int half = n >> 1;
    if (__ldg(ex + half) < item) {
      ex += half + 1;
      n -= half + 1;
    } else {
      n = half;
    }
  }
  return ex < end && __ldg(ex) == item;
}

// Key 0 sorts below every float key (only the NaN bit pattern 0xFFFFFFFF maps to it): an excluded
// candidate gets it, so it can only be "selected" when a row has fewer than K admissible candidates,
// and the gather passes below skip it.
#define SEL_KEY_EXCLUDED 0u

__global__ void __launch_bounds__(SEL_THREADS)
    fps_row_kth_kernel(const float* __restrict__ x, long long ld, int n_cols,
                       const int* __restrict__ counts, int K, const int* __restrict__ k_per_row, int staged,
                       float* __restrict__ out) {
  extern __shared__ float sel_row[];
  __shared__ uint32_t hist[SEL_WARPS * 256];
  __shared__ uint32_t bcast[2];
  const long long row = blockIdx.x;
  int n = n_cols;
  if (counts != nullptr) n = min(counts[row], n_cols);
  if (k_per_row != nullptr) K = k_per_row[row];
  if (n < K || K < 1) {  // fewer than K values: no bound (uniform branch)
    if (threadIdx.x == 0) out[row] = -3.0e38f;
    return;
  }
  const float* src = x + row * ld;
  if (staged) {
    for (int i = threadIdx.x; i < n; i += SEL_THREADS) sel_row[i] = src[i];
    __syncthreads();
    src = sel_row;
  }
  const uint32_t key = sel_block_kth_key(src, n, K, hist, bcast);
  if (threadIdx.x == 0) out[row] = sel_unkey(key);
}

template <bool EXCL>
__global__ void __launch_bounds__(SEL_THREADS)
    fps_row_topk_kernel(const float* __restrict__ cs, const int* __restrict__ ci, long long ld, int cap,
                        const int* __restrict__ counts, int K, int S, int staged,
                        const int* __restrict__ ex_off, const int* __restrict__ ex_items, int ex_total,
                        float* __restrict__ out_s, int* __restrict__ out_i) {
  extern __shared__ __align__(16) unsigned char sel_dyn[];
  unsigned long long* sortbuf = reinterpret_cast<unsigned long long*>(sel_dyn);  // [S]
  float* stage = reinterpret_cast<float*>(sortbuf + S);                           // [cap] if staged
  __shared__ uint32_t hist[SEL_WARPS * 256];
  __shared__ uint32_t bcast[2];
  __shared__ int n_gt, n_eq;
  const long long row = blockIdx.x;
  int n = cap;
  if (counts != nullptr) n = min(counts[row], cap);
  const float* src = cs + row * ld;
  const int* items = ci + row * ld;
  const int* ex = nullptr;
  int n_ex = 0;
  if (EXCL) {
    // clamped into [0, ex_total]: a malformed CSR gives a wrong filter, never an out-of-bounds read
    const int e0 = min(max(ex_off[row], 0), ex_total);
    ex = ex_items + e0;
    n_ex = min(max(ex_off[row + 1], e0), ex_total) - e0;
  }
  for (int i = threadIdx.x; i < S; i += SEL_THREADS) sortbuf[i] = 0ull;
  if (threadIdx.x == 0) { n_gt = 0; n_eq = 0; }
  if (staged) {
    // an excluded candidate is staged as the float whose key is SEL_KEY_EXCLUDED: one search per candidate
    for (int i = threadIdx.x; i < n; i += SEL_THREADS)
      stage[i] = (EXCL && sel_excluded(ex, n_ex, items[i])) ? __uint_as_float(0xFFFFFFFFu) : src[i];
    src = stage;
  }
  __syncthreads();
  // unstaged rows (cap > SEL_STAGE_MAX - 2S) search on every read instead
  auto key_at = [=](int i) -> uint32_t {
    if (EXCL && !staged && sel_excluded(ex, n_ex, items[i])) return SEL_KEY_EXCLUDED;
    return sel_key(src[i]);
  };
  uint32_t kth = 0;
  if (n > K) kth = sel_block_kth_key(key_at, n, K, hist, bcast);
  for (int i = threadIdx.x; i < n; i += SEL_THREADS) {
    const uint32_t key = key_at(i);
    if (key > kth) {  // at most K-1 of these when n > K, at most n <= K <= S otherwise
      const int slot = atomicAdd(&n_gt, 1);
      if (slot < S) sortbuf[slot] = ((unsigned long long)key << 32) | (0xFFFFFFFFu - (uint32_t)items[i]);
    }
  }
  __syncthreads();
  const int base = min(n_gt, S);
  // EXCL: kth == SEL_KEY_EXCLUDED means fewer than K admissible candidates, all taken by the pass above
  if (!EXCL || kth != SEL_KEY_EXCLUDED) {
    for (int i = threadIdx.x; i < n; i += SEL_THREADS) {
      const uint32_t key = key_at(i);
      if (key == kth) {  // ties with the K-th score: as many as the sort buffer holds
        const int slot = base + atomicAdd(&n_eq, 1);
        if (slot < S) sortbuf[slot] = ((unsigned long long)key << 32) | (0xFFFFFFFFu - (uint32_t)items[i]);
      }
    }
  }
  __syncthreads();
  for (int k = 2; k <= S; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < S; t += SEL_THREADS) {
        const int p = t ^ j;
        if (p > t) {
          const unsigned long long a = sortbuf[t], b = sortbuf[p];
          const bool desc = (t & k) == 0;
          if ((a < b) == desc) { sortbuf[t] = b; sortbuf[p] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < K; i += SEL_THREADS) {
    const unsigned long long e = sortbuf[i];
    out_s[row * K + i] = e ? sel_unkey((uint32_t)(e >> 32)) : -3.0e38f;
    out_i[row * K + i] = e ? (int)(0xFFFFFFFFu - (uint32_t)e) : -1;
  }
}

// k_per_row (optional, int32 [n_rows]) replaces K row by row.
extern "C" int fps_row_kth(const float* x, long long ld, int n_rows, int n_cols, const int* counts,
                           int K, const int* k_per_row, float* out, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  if (K < 1 && k_per_row == nullptr) return -1201;
  const int staged = n_cols <= SEL_STAGE_MAX ? 1 : 0;
  const size_t smem = staged ? (size_t)n_cols * sizeof(float) : 0;
  if (smem > 32 * 1024) {  // static (histograms) + dynamic must stay under 48 KB without the opt-in
    cudaError_t e = cudaFuncSetAttribute(fps_row_kth_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  fps_row_kth_kernel<<<n_rows, SEL_THREADS, smem, stream>>>(x, ld, n_cols, counts, K, k_per_row, staged, out);
  return (int)cudaGetLastError();
}

// ex_off / ex_items (optional, both or neither): per-row exclusion lists, CSR over ex_items[0..ex_total) with
// each row's items sorted ascending (duplicates are harmless).  K <= 2048 bounds the output, not K plus the excluded count.
extern "C" int fps_row_topk(const float* cs, const int* ci, long long ld, int n_rows, int cap,
                            const int* counts, int K, const int* ex_off, const int* ex_items, int ex_total,
                            float* out_s, int* out_i, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  if (K < 1 || K > 2048) return -1202;
  if ((ex_off == nullptr) != (ex_items == nullptr)) return -1203;
  int S = 64;
  while (S < 2 * K) S <<= 1;
  const int staged = cap <= SEL_STAGE_MAX - 2 * S ? 1 : 0;
  const size_t smem = (size_t)S * 8 + (staged ? (size_t)cap * sizeof(float) : 0);
  auto kern = ex_off != nullptr ? fps_row_topk_kernel<true> : fps_row_topk_kernel<false>;
  if (smem > 32 * 1024) {  // static (histograms) + dynamic must stay under 48 KB without the opt-in
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  kern<<<n_rows, SEL_THREADS, smem, stream>>>(cs, ci, ld, cap, counts, K, S, staged, ex_off, ex_items, ex_total,
                                              out_s, out_i);
  return (int)cudaGetLastError();
}
