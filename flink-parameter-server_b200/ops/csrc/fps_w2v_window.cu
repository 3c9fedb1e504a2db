// word2vec skip-gram and CBOW from a token stream (DESIGN §2.13, §2.14): frequent-word subsampling and compaction,
// then one fused SGNS kernel that trains each kept center over its whole dynamic window.
//
// Draws, all Philox4x32-10 with counter (c0, c1, c2, c3) and key (seed lo, seed hi), i = the token's position in
// the call:
//   keep      (i, 0, 0, step):                 u = ((x << 32 | y) >> 11) * 2^-53, kept iff u < keep_p[w] (fp64)
//   radius    (i, 1, 0, step):                 r = 1 + ((x << 32 | y) mod window)
//   negative  (i, 2 | slot << 8, j | t << 8, step): tries t (x, y) and t + 1 (z, w) of negative j of the center's
//             context number `slot`; uniform h mod vocab, or the 53-bit uniform through the fp64 noise CDF as in
//             fps_neg_noise_kernel.  A draw equal to the context word is rejected; all max_tries rejected = void.
//
// fps_w2v_subsample_kernel (one cooperative launch): token -1 and ids outside [0, vocab) are boundaries (the latter
// also counted as dropped), kept words and every boundary form the compacted sequence `seq` (-1 = boundary), with
// each entry's call position in `pos` and its length in *n_comp.  Per-CTA counts, grid sync, CTA offsets, then a
// ballot scan per CTA writes the entries in order.
//
// fps_w2v_kernel<CBOW>: one lane-group per compacted entry (grid-stride loop bounded by *n_comp, so the grid is
// sized without a host sync).  For a kept center c at entry e with radius r, its contexts are the entries
// e-r .. e+r (not e), stopping at a boundary or the end of the call, visited in increasing position.  A list of
// targets is (word, label 1), then `negative` noise words (label 0) rejected against the word, pulled in blocks of
// TB rows; per target with input w: d = w . v_t, g = lr (label - sigmoid(d)), e += g v_t, W_out[t] += g w (pushed
// at once).
//   skip-gram: u = W_in[c] as pulled, D = 0; per context q (slot k): w = u + D, e = 0, the targets of word q,
//     D += e after them; W_in[c] += D, pushed once
//   CBOW, for a center with cw >= 1 contexts: h = (sum of W_in[ctx] as pulled, in increasing position) / cw, the
//     context rows pulled TB at a time before any push; w = h, e = 0, the targets of word c keyed as slot 0;
//     W_in[ctx] += e for every context, once per occurrence: word2vec.c's mean in, unscaled error out.  A center
//     with no context trains and counts nothing.
// A W_out row repeated inside one block of targets is read as it was before the block; one repeated in a later
// block or context of the same center is read with the earlier pushes applied (the same lanes pushed and pull the
// same float4s, in program order).  Rows shared between centers, W_in rows too under CBOW, are updated
// Hogwild-style.
#include <cooperative_groups.h>
#include <limits.h>
#include "fps_common.cuh"
#include "fps_launch.cuh"

namespace cg = cooperative_groups;

#define W2V_THREADS 256

struct W2vArgs {
  const void* tokens;        // [n_tokens] int32 or int64 ids, -1 = sentence boundary
  long long n_tokens;
  long long vocab;
  const double* keep_p;      // [vocab] keep probabilities; nullptr keeps every word
  unsigned long long seed;
  unsigned long long step;
  int* seq;                  // [n_tokens] compacted sequence, -1 = boundary
  int* pos;                  // [n_tokens] call position of each compacted entry
  int* n_comp;               // [1] compacted length
  int* cta_cnt;              // [cta_cap] entries per CTA
  int cta_cap;
  int stride;                // row stride in floats of both tables
  long long* token_stats;    // [4] += tokens, kept, contexts, dropped
  ShardTable w_in;
  ShardTable w_out;
  int window;
  int negative;
  int max_tries;
  float lr;
  const double* cdf;         // [vocab] noise CDF (fps_noise_cdf); nullptr = uniform negatives
  long long last_nonzero;    // the last word of positive noise weight
  float* stats;              // [2] += sum -log sigmoid(+-d), targets trained
  int* nan_flag;
  int reserve_total;         // CTA slots left free for the replica exchange
  int cbow;                  // 0 = skip-gram, 1 = CBOW
};

__device__ __forceinline__ unsigned long long w2v_hash(const W2vArgs& a, long long i, uint32_t c1, uint32_t c2) {
  const Philox4 s = fps_philox((uint32_t)i, c1, c2, (uint32_t)a.step, (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  return ((unsigned long long)s.x << 32) | s.y;
}

// The compacted entry of token i: -2 = subsampled away (no entry), -1 = boundary, else the kept word.
template <typename IdT>
__device__ __forceinline__ int w2v_entry(const W2vArgs& a, long long i, bool& dropped) {
  const long long t = (long long)reinterpret_cast<const IdT*>(a.tokens)[i];
  dropped = false;
  if (t < 0 || t >= a.vocab) {
    dropped = t != -1;
    return -1;
  }
  if (a.keep_p != nullptr) {
    const double u = (double)(w2v_hash(a, i, 0u, 0u) >> 11) * 0x1.0p-53;
    if (!(u < a.keep_p[t])) return -2;
  }
  return (int)t;
}

template <typename IdT>
__global__ void __launch_bounds__(W2V_THREADS) fps_w2v_subsample_kernel(const W2vArgs a, long long per_cta) {
  __shared__ int red_s[3][W2V_THREADS / 32];
  __shared__ int carry_s;
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long lo = (long long)blockIdx.x * per_cta;
  const long long hi = lo + per_cta < a.n_tokens ? lo + per_cta : a.n_tokens;

  // 1. entries, kept words and dropped ids of the CTA's chunk
  int cnt = 0, kept = 0, drop = 0;
  for (long long i = lo + threadIdx.x; i < hi; i += W2V_THREADS) {
    bool d;
    const int c = w2v_entry<IdT>(a, i, d);
    cnt += c != -2;
    kept += c >= 0;
    drop += d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    kept += __shfl_xor_sync(0xffffffffu, kept, o);
    drop += __shfl_xor_sync(0xffffffffu, drop, o);
  }
  if (lane == 0) {
    red_s[0][wid] = cnt;
    red_s[1][wid] = kept;
    red_s[2][wid] = drop;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int s0 = 0, s1 = 0, s2 = 0;
    for (int w = 0; w < W2V_THREADS / 32; ++w) {
      s0 += red_s[0][w];
      s1 += red_s[1][w];
      s2 += red_s[2][w];
    }
    a.cta_cnt[blockIdx.x] = s0;
    if (a.token_stats != nullptr) {
      if (blockIdx.x == 0) atomicAdd((unsigned long long*)a.token_stats + 0, (unsigned long long)a.n_tokens);
      if (s1) atomicAdd((unsigned long long*)a.token_stats + 1, (unsigned long long)s1);
      if (s2) atomicAdd((unsigned long long*)a.token_stats + 3, (unsigned long long)s2);
    }
  }
  grid.sync();

  // 2. the CTA's offset; CTA 0 publishes the compacted length
  if (wid == 0) {
    int s = 0;
    for (int b = lane; b < (int)blockIdx.x; b += 32) s += a.cta_cnt[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) carry_s = s;
    if (blockIdx.x == 0) {
      int tot = 0;
      for (int b = lane; b < (int)gridDim.x; b += 32) tot += a.cta_cnt[b];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      if (lane == 0) *a.n_comp = tot;
    }
  }
  __syncthreads();

  // 3. ballot scan of the chunk: write the entries in order
  for (long long t0 = lo; t0 < hi; t0 += W2V_THREADS) {
    const long long i = t0 + threadIdx.x;
    int c = -2;
    if (i < hi) {
      bool d;
      c = w2v_entry<IdT>(a, i, d);
    }
    const bool flag = c != -2;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) red_s[0][wid] = __popc(bal);
    __syncthreads();
    int before = carry_s + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < wid; ++w) before += red_s[0][w];
    if (flag) {
      a.seq[before] = c;
      a.pos[before] = (int)i;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int s = 0;
      for (int w = 0; w < W2V_THREADS / 32; ++w) s += red_s[0][w];
      carry_s += s;
    }
    __syncthreads();
  }
}

extern "C" int fps_w2v_subsample(const W2vArgs* a, int id_bytes, int num_sms, cudaStream_t stream) {
  if (a->n_tokens <= 0) return 0;
  if (a->n_tokens >= INT_MAX || a->vocab < 1 || a->vocab > INT_MAX || a->cta_cap < 1) return -1501;
  const void* fn = id_bytes == 8 ? (const void*)fps_w2v_subsample_kernel<long long>
                                 : (const void*)fps_w2v_subsample_kernel<int>;
  int occ = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, W2V_THREADS, 0);
  if (e != cudaSuccess) return (int)e;
  long long grid = (long long)num_sms * occ;   // every CTA must be resident (grid sync)
  const long long need = (a->n_tokens + W2V_THREADS - 1) / W2V_THREADS;
  if (grid > need) grid = need;
  if (grid > a->cta_cap) grid = a->cta_cap;
  if (grid < 1) grid = 1;
  long long per_cta = (a->n_tokens + grid - 1) / grid;
  W2vArgs args = *a;
  void* params[] = {&args, &per_cta};
  e = cudaLaunchCooperativeKernel(fn, dim3((unsigned)grid), dim3(W2V_THREADS), params, 0, stream);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaGetLastError();
}

// Noise word j of context `slot` of the center at call position i; -1 when every try drew the context word.
__device__ __forceinline__ int w2v_negative(const W2vArgs& a, long long i, int slot, int j, int ctx) {
  const double total = a.cdf != nullptr ? a.cdf[a.vocab - 1] : 0.0;
  for (int t = 0; t < a.max_tries; t += 2) {
    const Philox4 s = fps_philox((uint32_t)i, 2u | ((uint32_t)slot << 8), (uint32_t)(j | (t << 8)), (uint32_t)a.step,
                                 (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
    const unsigned long long h[2] = {((unsigned long long)s.x << 32) | s.y, ((unsigned long long)s.z << 32) | s.w};
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (t + q >= a.max_tries) break;
      long long c;
      if (a.cdf != nullptr) {
        const double x = (double)(h[q] >> 11) * 0x1.0p-53 * total;
        long long l = 0, r = a.vocab;   // the first word whose prefix exceeds x
        while (l < r) {
          const long long m = (l + r) >> 1;
          if (a.cdf[m] > x) r = m;
          else l = m + 1;
        }
        c = l < a.vocab ? l : a.last_nonzero;
      } else {
        c = (long long)(h[q] % (unsigned long long)a.vocab);
      }
      if (c != ctx) return (int)c;
    }
  }
  return -1;
}

__device__ __forceinline__ float4 w2v_add4(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float w2v_dot4(float4 w, float4 v) { return w.x * v.x + w.y * v.y + w.z * v.z + w.w * v.w; }

template <bool CBOW, int LPR, int VPL, int MINB, int TB>
__global__ void __launch_bounds__(W2V_THREADS, MINB) fps_w2v_kernel(const __grid_constant__ W2vArgs a) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int nvec = a.stride >> 2;
  const int T = 1 + a.negative;
  const long long n = *a.n_comp;
  float loss_acc = 0.f, tgt_acc = 0.f;
  unsigned long long ctx_acc = 0;
  bool bad = false;

  // the trip count is the same for every lane of a warp (n_groups is a multiple of 32 / LPR)
  const long long n_round = ((n + n_groups - 1) / n_groups) * n_groups;
  for (long long e = group; e < n_round; e += n_groups) {
    const int center = e < n ? a.seq[e] : -1;
    const bool ok = center >= 0;
    long long i = 0, L = e, R = e;
    if (ok) {
      i = a.pos[e];
      const long long r = 1 + (long long)(w2v_hash(a, i, 1u, 0u) % (unsigned long long)a.window);
      for (long long q = e - 1; q >= e - r && q >= 0 && a.seq[q] >= 0; --q) L = q;
      for (long long q = e + 1; q <= e + r && q < n && a.seq[q] >= 0; ++q) R = q;
    }
    const int n_left = (int)(e - L), n_ctx = (int)(R - L);
    float* up = fps_row32(a.w_in, ok ? center : 0);
    float4 u[VPL], D[VPL];    // skip-gram: u and D
    float4 h[VPL], ev[VPL];   // CBOW: h; both: e of the current targets
    if constexpr (!CBOW) {
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        u[c] = (ok && q < nvec) ? fps_ld_row4(up + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);   // the PULL of u
        D[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else {
      const bool has_ctx = n_ctx > 0;   // tested before the pulls, for the code nvcc makes (NOTES, Pitfalls)
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        h[c] = make_float4(0.f, 0.f, 0.f, 0.f);
        ev[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      // the PULL of the context rows, TB in flight at a time, summed in increasing position
      for (int k0 = 0; k0 < n_ctx; k0 += TB) {
        float4 x[TB][VPL];
#pragma unroll
        for (int b = 0; b < TB; ++b) {
          const int k = k0 + b;
          const int ctx = k < n_ctx ? a.seq[k < n_left ? L + k : e + 1 + (k - n_left)] : -1;
          const float* xp = fps_row32(a.w_in, ctx >= 0 ? ctx : 0);
#pragma unroll
          for (int c = 0; c < VPL; ++c) {
            const int q = lane + c * LPR;
            x[b][c] = (ctx >= 0 && q < nvec) ? fps_ld_row4(xp + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int b = 0; b < TB; ++b) {
          if (k0 + b >= n_ctx) break;
#pragma unroll
          for (int c = 0; c < VPL; ++c) h[c] = w2v_add4(h[c], x[b][c]);
        }
      }
      if (has_ctx) {
        const float cw = (float)n_ctx;
#pragma unroll
        for (int c = 0; c < VPL; ++c) h[c] = make_float4(h[c].x / cw, h[c].y / cw, h[c].z / cw, h[c].w / cw);
      }
    }
    // one list of targets per context (skip-gram) or one per center, keyed as context slot 0 (CBOW)
    for (int k = 0; CBOW ? k == 0 : __any_sync(0xffffffffu, k < n_ctx); ++k) {
      const bool live = k < n_ctx;
      int word = CBOW ? center : -1;   // the label-1 target, which the noise words must differ from
      if (!CBOW && live) word = a.seq[k < n_left ? L + k : e + 1 + (k - n_left)];
      if constexpr (!CBOW) {
#pragma unroll
        for (int c = 0; c < VPL; ++c) ev[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      // with negative <= LPR, lane l of the group draws negative l, so the draws (a binary search of the CDF each)
      // run side by side instead of one after another
      const bool par = a.negative <= LPR;
      int mine = -1;
      if (par && live && lane < a.negative) mine = w2v_negative(a, i, k, lane, word);
      for (int t0 = 0; t0 < T; t0 += TB) {
        int tid[TB];
        float4 v[TB][VPL];
#pragma unroll
        for (int b = 0; b < TB; ++b) {   // the block's ids, then all of its pulls
          const int t = t0 + b;
          const int src = (int)(threadIdx.x & 31 & ~(LPR - 1)) + (t >= 1 && t - 1 < LPR ? t - 1 : 0);
          const int drawn = __shfl_sync(0xffffffffu, mine, src);
          int id = -1;
          if (live && t < T) id = t == 0 ? word : par ? drawn : w2v_negative(a, i, k, t - 1, word);
          tid[b] = id;
          const float* vp = fps_row32(a.w_out, id >= 0 ? id : 0);
#pragma unroll
          for (int c = 0; c < VPL; ++c) {
            const int q = lane + c * LPR;
            v[b][c] = (id >= 0 && q < nvec) ? fps_ld_row4(vp + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int b = 0; b < TB; ++b) {
          if (t0 + b >= T) break;           // uniform: T is the same for every group
          float part = 0.f;
#pragma unroll
          for (int c = 0; c < VPL; ++c) part += w2v_dot4(CBOW ? h[c] : w2v_add4(u[c], D[c]), v[b][c]);
          const float d = fps_group_sum<LPR>(part);
          if (tid[b] < 0) continue;
          if (!(fabsf(d) <= 3.0e38f)) bad = true;   // NaN/Inf guard
          const float label = (t0 + b == 0) ? 1.f : 0.f;
          const float g = a.lr * (label - 1.f / (1.f + __expf(-d)));
          if (lane == 0) {
            const float x = (t0 + b == 0) ? -d : d;   // -log sigmoid(+-d) = softplus(-+d)
            loss_acc += fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x)));
            tgt_acc += 1.f;
          }
          float* vp = fps_row32(a.w_out, tid[b]);
#pragma unroll
          for (int c = 0; c < VPL; ++c) {
            const int q = lane + c * LPR;
            if (q < nvec) {
              ev[c].x += g * v[b][c].x; ev[c].y += g * v[b][c].y;
              ev[c].z += g * v[b][c].z; ev[c].w += g * v[b][c].w;
              // CBOW reads h[c] in place: a copy of it changes the code nvcc makes at VPL = 1
              float4 s;
              if constexpr (!CBOW) s = w2v_add4(u[c], D[c]);
              const float4& w = CBOW ? h[c] : s;
              fps_red_add4(vp + 4 * q, make_float4(g * w.x, g * w.y, g * w.z, g * w.w));   // the PUSH of g w
            }
          }
        }
      }
      if constexpr (!CBOW) {
        if (live) {
#pragma unroll
          for (int c = 0; c < VPL; ++c) {
            D[c].x += ev[c].x; D[c].y += ev[c].y; D[c].z += ev[c].z; D[c].w += ev[c].w;
          }
          if (lane == 0) ++ctx_acc;
        }
      }
    }
    if constexpr (!CBOW) {
      if (ok) {
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const int q = lane + c * LPR;
          if (q < nvec) fps_red_add4(up + 4 * q, D[c]);   // the one PUSH of the center row
        }
      }
    } else {
      // the PUSH of e to every context row, once per occurrence
      for (int k = 0; k < n_ctx; ++k) {
        float* xp = fps_row32(a.w_in, a.seq[k < n_left ? L + k : e + 1 + (k - n_left)]);
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const int q = lane + c * LPR;
          if (q < nvec) fps_red_add4(xp + 4 * q, ev[c]);
        }
      }
      if (lane == 0) ctx_acc += (unsigned long long)n_ctx;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);
    tgt_acc += __shfl_xor_sync(0xffffffffu, tgt_acc, o);
    ctx_acc += __shfl_xor_sync(0xffffffffu, ctx_acc, o);
  }
  if ((threadIdx.x & 31) == 0 && tgt_acc > 0.f) {
    if (a.stats != nullptr) {
      atomicAdd(a.stats + 0, loss_acc);
      atomicAdd(a.stats + 1, tgt_acc);
    }
    if (a.token_stats != nullptr) atomicAdd((unsigned long long*)a.token_stats + 2, ctx_acc);
  }
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
}

// One CTA per SM slot the occupancy allows, less `reserve_total` for the replica exchange; the grid-stride loop
// covers however many entries the subsample kernel wrote, so the grid needs no host-side count.
template <int LPR, int VPL, int MINB, int TB>
static int launch_w2v(const W2vArgs& a, int num_sms, cudaStream_t stream) {
  void (*kern)(const W2vArgs) = a.cbow ? fps_w2v_kernel<true, LPR, VPL, MINB, TB>
                                       : fps_w2v_kernel<false, LPR, VPL, MINB, TB>;
  const long long blocks = fps_row_grid(kern, W2V_THREADS, W2V_THREADS / LPR, num_sms, a.reserve_total, 0, 1,
                                        a.n_tokens, 1);   // n_comp <= n_tokens
  kern<<<(int)blocks, W2V_THREADS, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// Lane geometry of dispatch_bpr: LPR lanes per row, VPL float4 per lane; MINB keeps each free of spills (ptxas -v).
// TB target rows, and under CBOW TB context rows, are pulled at once: 8 (every target of a context while
// negative <= 7), 6 for rows over 384 floats, where 8 rows of 4 float4 per lane do not fit in 255 registers (6 =
// word2vec's default negative = 5).
extern "C" int fps_w2v_window_fused(const W2vArgs* args, int num_sms, cudaStream_t stream) {
  const W2vArgs& a = *args;
  if (a.n_tokens <= 0) return 0;
  if ((a.stride & 3) != 0 || a.window < 1 || a.window >= (1 << 23) || a.negative < 0 || a.negative > 255 ||
      a.max_tries < 1 || a.max_tries >= (1 << 23) || a.vocab < 1 || a.vocab > INT_MAX || (a.cbow & ~1) != 0)
    return -1501;
  const int nvec = a.stride >> 2;
  if (nvec <= 1) return launch_w2v<1, 1, 2, 8>(a, num_sms, stream);
  if (nvec <= 2) return launch_w2v<2, 1, 2, 8>(a, num_sms, stream);
  if (nvec <= 4) return launch_w2v<4, 1, 2, 8>(a, num_sms, stream);
  if (nvec <= 8) return launch_w2v<8, 1, 2, 8>(a, num_sms, stream);
  if (nvec <= 16) return launch_w2v<16, 1, 2, 8>(a, num_sms, stream);
  if (nvec <= 32) return launch_w2v<32, 1, 2, 8>(a, num_sms, stream);
  if (nvec <= 64) return launch_w2v<32, 2, 1, 8>(a, num_sms, stream);
  if (nvec <= 96) return launch_w2v<32, 3, 1, 8>(a, num_sms, stream);
  if (nvec <= 128) return launch_w2v<32, 4, 1, 6>(a, num_sms, stream);
  return -1000;   // rows wider than 512 floats
}
