// Windowed single-GPU MF step: apply a run of staged micro-batches in one item-major pass, so that every
// item row crosses HBM once per window instead of once per micro-batch.
//
// Why: on one GPU the fused per-launch kernel (fps_core.cu) already streams at ~86 % of a copy_, and half of
// what it moves is item rows: the 1M x 256 B item table is five times the L2, so each micro-batch pulls most of
// the table from HBM and writes it back.  When the micro-batches of a window are conflict-free -- no user twice
// in the window, no item twice in a micro-batch -- their result splits into independent per-item chains: for
// each item, apply its ratings in micro-batch order to a copy of the item row held in registers.  Every user
// row is read and written by exactly one update, so the arithmetic is the per-launch kernel's, in the same
// order (the per-launch group sum's tree, fps_mf_dot4 / fps_mf_grad, adds as add.rn.ftz like red.global.add.f32):
// the tables come out bitwise equal; only when each row is loaded and stored changes.
//
// One cooperative launch per drain (fps_mf_window_kernel), looping until every staged micro-batch is applied:
//   1. build: clear the user bitmap; scatter micro-batch start, start+1, ... (one per grid sync) into the
//      item-major slot table T[j - start][item] = {user slot, rating} with atomicExch, test-and-setting each
//      user's bit.  An occupied T entry or an already-set bit is a conflict: the window ends before that
//      micro-batch.
//   2. chain: one lane-group per item reads its entries, pulls the item row once and the chain's user rows
//      together, applies the updates in order, stores each row once and resets every T entry it saw.
//   3. singleton: a micro-batch that conflicts with itself (an item or a user twice in it) is applied alone
//      with the per-launch update (pull both rows, red.global.add both deltas): racy as it is today.
#include <cooperative_groups.h>
#include "fps_common.cuh"
#include "fps_mf_args.cuh"

namespace cg = cooperative_groups;

#define WIN_MAX 8            // micro-batches per window (T rows)
#define WIN_THREADS 256
#define WIN_EMPTY 0xFFFFFFFFFFFFFFFFull

struct WinArgs {
  const unsigned char* stage;   // staged records, slot j at stage + j * slot_bytes
  long long slot_bytes;
  long long n[WIN_MAX];         // records per slot
  int fmt[WIN_MAX];             // 0: int32 users[n] | int32 items[n] | fp32 ratings[n];  1: packed64[n]
  int n_slots;
  int err_mode;
  float lr;
  int stride;                   // row stride in floats (user and item tables)
  float* user_table;            // [n_local, stride], slot = user (one worker)
  float* item_table;            // [rows, stride]
  long long rows;               // item rows = T row length
  unsigned long long* slots;    // T [n_slots, rows]; WIN_EMPTY everywhere between drains
  unsigned int* user_bits;      // [bm_words]
  long long bm_words;
  unsigned int* ctl;            // [2 * WIN_MAX] conflict flag per scatter attempt (zeroed by the kernel)
  float* stats;                 // [2] += window totals
  float* slot_stats;            // [n_slots, 2] per-micro-batch (sum sq err, updates) (zeroed by the kernel)
  int* nan_flag;
  unsigned long long* phase_ns; // optional [4] += (build ns, apply ns, windows, -): CTA 0's %globaltimer after
                                // each phase's grid sync; [3] is scratch.  Null in production.
};

__device__ __forceinline__ bool win_record(const WinArgs& a, int j, long long i, int& user, int& item,
                                           float& rating) {
  const unsigned char* base = a.stage + (long long)j * a.slot_bytes;
  if (a.fmt[j] == 1) {
    const FpsRecord<int> rec = fps_record<int>(1, base, nullptr, nullptr, i);
    user = rec.user;
    item = rec.item;
    rating = rec.rating;
    return true;
  }
  const long long n = a.n[j];   // arrays: users | items | ratings, n of each
  const FpsRecord<int> rec =
      fps_record<int>(0, base, reinterpret_cast<const int*>(base) + n, reinterpret_cast<const float*>(base) + 2 * n, i);
  user = rec.user;
  item = rec.item;
  rating = rec.rating;
  return user >= 0;   // record voided upstream
}

__device__ __forceinline__ float win_add(float x, float y) {
  float z;
  asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(z) : "f"(x), "f"(y));
  return z;
}
__device__ __forceinline__ float4 win_add4(float4 x, float g, float4 y) {   // x + g * y, rounded like the REDG
  return make_float4(win_add(x.x, g * y.x), win_add(x.y, g * y.y), win_add(x.z, g * y.z), win_add(x.w, g * y.w));
}

__device__ __forceinline__ unsigned long long win_clock() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// phase_ns[k] += time since the previous mark (kept in phase_ns[3], so no register lives across a phase)
__device__ __forceinline__ void win_phase(const WinArgs& a, int k) {
  const unsigned long long t = win_clock();
  a.phase_ns[k] += t - a.phase_ns[3];
  a.phase_ns[3] = t;
  if (k == 1) a.phase_ns[2] += 1ull;
}

// Per-slot (sum sq err, updates) sums: slot r lives in lane r % G of every G-lane group, at index r / G.
// Flushed as warp sums -> CTA sums in shared memory -> one atomic per (CTA, slot) into slot_stats[slot0 + r].
template <int G, int NS>
__device__ __forceinline__ void win_flush_stats(const WinArgs& a, float (&sq)[NS], float (&cnt)[NS], int nr,
                                                int slot0, float* sh) {
  const int lane = threadIdx.x & (G - 1);
  __syncthreads();
  if (threadIdx.x < 2 * WIN_MAX) sh[threadIdx.x] = 0.f;
  __syncthreads();
#pragma unroll
  for (int r = 0; r < WIN_MAX; ++r) {
    if (r < nr) {
      const bool mine = lane == r % G;
      float s = mine ? sq[r / G] : 0.f, c = mine ? cnt[r / G] : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
      }
      if ((threadIdx.x & 31) == 0 && c > 0.f) {
        atomicAdd(sh + 2 * r, s);
        atomicAdd(sh + 2 * r + 1, c);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NS; ++i) sq[i] = cnt[i] = 0.f;
  __syncthreads();
  if (threadIdx.x < 2 * nr && sh[threadIdx.x] != 0.f)
    atomicAdd(a.slot_stats + 2 * slot0 + threadIdx.x, sh[threadIdx.x]);
}

// A row's float4s on a G-lane group, VPL per lane: lane l holds float4s l, l + G, ..., l + (VPL - 1) G.
template <int G, int VPL>
__device__ __forceinline__ void win_load(float4 (&x)[VPL], const float* row, int lane, int nvec, bool on) {
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int c = lane + k * G;
    x[k] = (on && c < nvec) ? *reinterpret_cast<const float4*>(row + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
template <int G, int VPL>
__device__ __forceinline__ void win_store(float* row, const float4 (&x)[VPL], int lane, int nvec) {
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    const int c = lane + k * G;
    if (c < nvec) *reinterpret_cast<float4*>(row + 4 * c) = x[k];
  }
}
// u.v over the group, with the bits of fps_group_sum<G * VPL> over one float4 per lane: its first log2(VPL)
// levels pair float4 c with c + G * VPL / 2, c + G * VPL / 4, ...; those pairs are in this lane, added here in
// the same tree order, and the remaining levels are the shuffles over the G lanes.
template <int G, int VPL>
__device__ __forceinline__ float win_dot(const float4 (&u)[VPL], const float4 (&v)[VPL]) {
  float d[VPL];
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    d[k] = 0.f;
    d[k] += fps_mf_dot4(u[k], v[k]);
  }
#pragma unroll
  for (int h = VPL / 2; h > 0; h >>= 1)
#pragma unroll
    for (int k = 0; k < h; ++k) d[k] += d[k + h];
  return fps_group_sum<G>(d[0]);
}

// Rows of up to LPR float4 (LPR: the dispatch_mf lane count for them, one float4 per lane there) held by
// G = LPR / VPL lanes, VPL float4 per lane: fewer lanes per row leave more of the register file to rows in
// flight.  P = user rows prefetched together per lane-group, MINB = CTAs per SM the registers are held to.
template <int LPR, int VPL, int P, int MINB>
__global__ void __launch_bounds__(WIN_THREADS, MINB) fps_mf_window_kernel(const __grid_constant__ WinArgs a) {
  static_assert(VPL >= 1 && VPL <= LPR && LPR % VPL == 0, "VPL must divide LPR");
  constexpr int G = LPR / VPL;   // lanes per row
  __shared__ float sh[2 * WIN_MAX];
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & (G - 1);
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;   // 32-bit: the grid is one wave of resident CTAs
  const int gthreads = gridDim.x * blockDim.x;
  const int group = gtid / G;
  const int n_groups = gthreads / G;
  const int stride = a.stride;
  const int nvec = stride >> 2;
  constexpr int NS = G < WIN_MAX ? WIN_MAX / G : 1;
  constexpr int NE = NS;   // T entries per lane in the chain
  float sq[NS], cnt[NS];   // see win_flush_stats
#pragma unroll
  for (int i = 0; i < NS; ++i) sq[i] = cnt[i] = 0.f;
  bool bad = false;
  const bool timer = a.phase_ns != nullptr && blockIdx.x == 0 && threadIdx.x == 0;

  if (blockIdx.x == 0) {
    if (threadIdx.x < 2 * WIN_MAX) a.ctl[threadIdx.x] = 0u;
    if (threadIdx.x < 2 * a.n_slots) a.slot_stats[threadIdx.x] = 0.f;
  }
  if (timer) a.phase_ns[3] = win_clock();
  int start = 0, attempt = 0;
  while (start < a.n_slots) {
    // ---- 1. build -------------------------------------------------------------------------------------
    for (long long w = gtid; w < a.bm_words; w += gthreads) a.user_bits[w] = 0u;
    grid.sync();
    int end = start;
    bool clashed = false;
    while (end < a.n_slots) {
      const int j = end;
      unsigned long long* t = a.slots + (long long)(j - start) * a.rows;
      bool clash = false;
      for (long long i = gtid; i < a.n[j]; i += gthreads) {
        int user, item;
        float rating;
        if (!win_record(a, j, i, user, item, rating)) continue;
        const unsigned long long e = ((unsigned long long)__float_as_uint(rating) << 32) | (unsigned int)user;
        clash |= atomicExch(t + item, e) != WIN_EMPTY;
        const unsigned int bit = 1u << (user & 31);
        clash |= (atomicOr(a.user_bits + (user >> 5), bit) & bit) != 0u;
      }
      if (clash) *reinterpret_cast<volatile unsigned int*>(a.ctl + attempt) = 1u;
      grid.sync();
      clashed = *reinterpret_cast<volatile unsigned int*>(a.ctl + attempt) != 0u;
      ++attempt;
      if (clashed) break;
      ++end;
    }
    if (timer) win_phase(a, 0);
    const int nrow = end - start;                  // micro-batches in the window
    const int written = nrow + (clashed ? 1 : 0);  // T rows holding entries (the clashing one partially)
    if (nrow > 0) {
      // ---- 2. chain -------------------------------------------------------------------------------------
      // T entries: lane l of the group loads rows r = l, l + G, ... of its item (every T entry the window
      // wrote, the clashing micro-batch's partial row included), one item ahead of the chain, and resets
      // them itself; the chain gets them by shuffles.
      unsigned long long nxt[NE];
#pragma unroll
      for (int m = 0; m < NE; ++m) {
        const int r = lane + m * G;
        nxt[m] = (group < a.rows && r < written) ? a.slots[(long long)r * a.rows + group] : WIN_EMPTY;
      }
      for (long long base = 0; base < a.rows; base += n_groups) {   // warp-uniform trip count
        const long long item = base + group;
        const bool in = item < a.rows;
        float* vp = a.item_table + (in ? item : 0) * (long long)stride;
        float4 v[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        bool any = false;
        bool loaded = false;
        unsigned long long mine[NE];
#pragma unroll
        for (int m = 0; m < NE; ++m) {
          const int r = lane + m * G;
          mine[m] = nxt[m];
          const long long it2 = item + n_groups;
          nxt[m] = (it2 < a.rows && r < written) ? a.slots[(long long)r * a.rows + it2] : WIN_EMPTY;
          if (mine[m] != WIN_EMPTY) a.slots[(long long)r * a.rows + item] = WIN_EMPTY;
        }
        const int src0 = (threadIdx.x & 31) & ~(G - 1);   // the group's first lane in the warp
#pragma unroll
        for (int c0 = 0; c0 < WIN_MAX; c0 += P) {
          if (c0 < nrow) {
            unsigned long long ent[P];
#pragma unroll
            for (int q = 0; q < P; ++q) {
              const int r = c0 + q;
              ent[q] = __shfl_sync(0xffffffffu, mine[(r / G) % NE], src0 + r % G);
              if (r >= nrow) ent[q] = WIN_EMPTY;   // the clashing micro-batch is not applied
            }
            {
              bool chunk_any = false;
#pragma unroll
              for (int q = 0; q < P; ++q) chunk_any |= ent[q] != WIN_EMPTY;
              if (chunk_any && !loaded) win_load<G, VPL>(v, vp, lane, nvec, true);
              loaded |= chunk_any;
              any |= chunk_any;
              float4 u[P][VPL];
#pragma unroll
              for (int q = 0; q < P; ++q)
                win_load<G, VPL>(u[q], a.user_table + (long long)(unsigned int)ent[q] * stride, lane, nvec,
                                 ent[q] != WIN_EMPTY);
#pragma unroll
              for (int q = 0; q < P; ++q) {
                const int r = c0 + q;
                if (r < nrow) {                    // grid-uniform: the group sum sees the whole warp
                  const float d = win_dot<G, VPL>(u[q], v);
                  const bool ok = ent[q] != WIN_EMPTY;
                  const float rating = __uint_as_float((unsigned int)(ent[q] >> 32));
                  const float resid = rating - d;
                  const float g = fps_mf_grad(a.err_mode, a.lr, rating, d, resid);
                  if (ok) {
                    if (!(fabsf(g) <= 3.0e38f)) bad = true;  // NaN/Inf guard, as the per-launch kernel
                    if (lane == r % G) {
                      sq[r / G] += resid * resid;
                      cnt[r / G] += 1.f;
                    }
                    float4 nu[VPL];
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                      nu[k] = win_add4(u[q][k], g, v[k]);
                      v[k] = win_add4(v[k], g, u[q][k]);
                    }
                    win_store<G, VPL>(a.user_table + (long long)(unsigned int)ent[q] * stride, nu, lane, nvec);
                  }
                }
              }
            }
          }
        }
        if (any) win_store<G, VPL>(vp, v, lane, nvec);
      }
      win_flush_stats<G, NS>(a, sq, cnt, nrow, start, sh);
    } else {
      // ---- 3. singleton: micro-batch `start` has an item or a user twice ----------------------------------
      const int j = start;
      unsigned long long* t = a.slots;
      for (long long base = 0; base < a.n[j]; base += n_groups) {
        const long long i = base + group;
        int user = 0, item = 0;
        float rating = 0.f;
        const bool ok = i < a.n[j] && win_record(a, j, i, user, item, rating);
        float* up = a.user_table + (long long)user * stride;
        float* vp = a.item_table + (long long)item * stride;
        float4 u[VPL], v[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          const int c = lane + k * G;
          u[k] = v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok && c < nvec) {
            v[k] = fps_ld_row4(vp + 4 * c);
            u[k] = *reinterpret_cast<const float4*>(up + 4 * c);
          }
        }
        const float d = win_dot<G, VPL>(u, v);
        const float resid = rating - d;
        const float g = fps_mf_grad(a.err_mode, a.lr, rating, d, resid);
        if (ok) {
          if (!(fabsf(g) <= 3.0e38f)) bad = true;
          if (lane == 0) {
            sq[0] += resid * resid;
            cnt[0] += 1.f;
            t[item] = WIN_EMPTY;
          }
#pragma unroll
          for (int k = 0; k < VPL; ++k) {
            const int c = lane + k * G;
            if (c < nvec) {
              fps_red_add4(up + 4 * c, make_float4(g * v[k].x, g * v[k].y, g * v[k].z, g * v[k].w));
              fps_red_add4(vp + 4 * c, make_float4(g * u[k].x, g * u[k].y, g * u[k].z, g * u[k].w));
            }
          }
        }
      }
      win_flush_stats<G, NS>(a, sq, cnt, 1, start, sh);
      end = start + 1;
    }
    grid.sync();
    if (timer) win_phase(a, 1);
    start = end;
  }
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
  if (blockIdx.x == 0 && threadIdx.x == 0 && a.stats != nullptr) {
    float s = 0.f, c = 0.f;
    for (int j = 0; j < a.n_slots; ++j) {
      s += a.slot_stats[2 * j];
      c += a.slot_stats[2 * j + 1];
    }
    a.stats[0] += s;
    a.stats[1] += c;
  }
}

template <int LPR, int VPL, int P, int MINB>
static int launch_window(const WinArgs& a, int num_sms, cudaStream_t stream) {
  constexpr int V = VPL < LPR ? VPL : LPR;   // narrow rows keep at least one float4 per lane
  int occ = 0;
  cudaError_t e =
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fps_mf_window_kernel<LPR, V, P, MINB>, WIN_THREADS, 0);
  if (e != cudaSuccess) return (int)e;
  if (occ < 1) return -1402;
  const long long grid = (long long)num_sms * occ;   // every CTA resident (grid sync)
  WinArgs args = a;
  void* params[] = {&args};
  e = cudaLaunchCooperativeKernel((const void*)fps_mf_window_kernel<LPR, V, P, MINB>, dim3((unsigned)grid),
                                  dim3(WIN_THREADS), params, 0, stream);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaGetLastError();
}

static int g_win_variant = 0;  // tuning knob: (float4 per lane, user rows prefetched, CTAs/SM), see dispatch_window
extern "C" void fps_set_mf_window_variant(int v) { g_win_variant = v; }

// Defaults by row width (nvec float4): 9..16 float4 (k = 64) as 4 float4 on each of 4 lanes, 2 user rows
// prefetched, 2 CTAs/SM (121 registers, 128 lane-groups per SM); the other widths keep one float4 per lane, 4
// user rows prefetched, 3 CTAs/SM (2 for LPR <= 2).  NOTES.md "Step window" has the sweep behind the choice.
template <int LPR>
static int dispatch_window(const WinArgs& a, int num_sms, cudaStream_t s) {
  constexpr int MINB_V1 = LPR <= 2 ? 2 : 3;   // LPR <= 2: more per-slot sums per lane
  switch (g_win_variant) {
    case 1: return launch_window<LPR, 1, 8, 1>(a, num_sms, s);   // all 8 user rows of a chain at once, 2 CTAs/SM
    case 2: return launch_window<LPR, 1, 4, MINB_V1>(a, num_sms, s);   // one float4 per lane everywhere
    default:
      if constexpr (LPR == 16) return launch_window<16, 4, 2, 2>(a, num_sms, s);
      else return launch_window<LPR, 1, 4, MINB_V1>(a, num_sms, s);
  }
}

// Rows of up to 32 float4 (k <= 128), bucketed by the lane count dispatch_mf picks for them.
extern "C" int fps_mf_window_drain(const WinArgs* a, int num_sms, cudaStream_t stream) {
  if (a->n_slots <= 0) return 0;
  if (a->n_slots > WIN_MAX) return -1401;
  const int nvec = a->stride >> 2;
  if (nvec <= 1) return dispatch_window<1>(*a, num_sms, stream);
  if (nvec <= 2) return dispatch_window<2>(*a, num_sms, stream);
  if (nvec <= 4) return dispatch_window<4>(*a, num_sms, stream);
  if (nvec <= 8) return dispatch_window<8>(*a, num_sms, stream);
  if (nvec <= 16) return dispatch_window<16>(*a, num_sms, stream);
  if (nvec <= 32) return dispatch_window<32>(*a, num_sms, stream);
  return -1400;
}
