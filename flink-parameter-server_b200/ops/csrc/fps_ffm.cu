// Field-aware factorization machine step on a CSR micro-batch (DESIGN §2.16), fused with the pulls and pushes.
//
// Table: num_features + 1 rows of stride = 4 + F kp floats, kp = round_up(k, 4).  Row i =
// [w_i | 0 0 0 | V_i,0 (kp) | .. | V_i,F-1 (kp)], slab f starting at column 4 + f kp (16-byte aligned); columns
// [k, kp) of every slab are padding.  Row num_features is the bias row, w0 in column 0.  An example is a CSR run of
// entries (i, f, x); an entry with i outside [0, num_features) or f outside [0, F) is skipped and raises *bad_id.
// Over the kept entries, every pair a < b in CSR order:
//   yhat = w0 + sum_a x_a w_a + sum_{a<b} x_a x_b <V[i_a, f_b], V[i_b, f_a]>
//   logistic: g = sigmoid(yhat) - y, loss = softplus(yhat) - y yhat;   squared: g = yhat - y, loss = (yhat - y)^2
// and, from the rows as the example pulled them, with c = g x_a x_b:
//   dw_a = -lr (g x_a + reg_linear w_a),   dV[i_a,f_b] = -lr (c V[i_b,f_a] + reg_factors V[i_a,f_b]),
//   dV[i_b,f_a] = -lr (c V[i_a,f_b] + reg_factors V[i_b,f_a]),   padding: 0
// pushed with red.add.  w0 follows the factorization machine's rule (fps_fm_bias.cuh).  One launch per step.
//
// Geometry: one warp per example.  The kept entries are staged per warp in shared memory, CH at a time (row
// pointer, field, x); the triangle of pairs is tiled over chunk pairs (A <= B).  Within a tile the pairs go to
// lane-groups of Q lanes, Q = kp / 4 rounded up to a power of two, lane l holding float4 l of the pair's two slabs, TB pairs in flight per lane.
// Pass 1 sums the pair terms and the linear term (one warp sum gives yhat); pass 2 re-pulls both slabs of each pair
// (L2 hits) and pushes the two deltas, and pushes each entry's dw as its chunk is staged.
//
// AdaGrad (DESIGN §2.17): with acc.base[0] set, acc is a second table of the same geometry holding H = G - 1 per
// element, and the step launches fps_ffm_kernel with ADA set.  Pass 1 and w0 are shared with SGD; pass 2 stages each
// entry's H row beside its row, and every slab chunk and every w is pulled with its H, stepped by
// -lr * gam / sqrtf(1 + H + gam^2) (gam: the bracket above) and pushed with H += gam^2.  The two pass 2 tile loops
// stay apart, as in fps_fm.cu.
#include <limits.h>
#include "fps_common.cuh"
#include "fps_fm_bias.cuh"
#include "fps_launch.cuh"

#define FFM_THREADS 256
#define FFM_WARPS (FFM_THREADS / 32)
#define FFM_CH 64          // entries per staged chunk
#define FFM_MAX_K 64
#define FFM_MAX_FIELDS 256

struct FfmArgs {
  const long long* row_ptr;  // [n + 1]
  const void* cols;          // [nnz] int32 or int64 feature ids
  const int* fields;         // [nnz] field of every entry
  const float* vals;         // [nnz] values, or nullptr: one-hot (every x = 1)
  const float* labels;       // [n] float32; NaN = predict only
  float* pred;               // [n] out: yhat before the example's own update
  float* stats;              // [2] += loss, labelled examples (may be null)
  int* nan_flag;             // set by a non-finite delta (may be null)
  int* bad_id;               // set by an entry whose id or field is out of range (may be null)
  long long n;
  long long nnz;
  long long num_features;    // the bias row's id
  int num_fields;            // F
  int k;                     // factors per slab; slabs are round_up(k, 4) floats apart
  int loss;                  // FmLoss
  float lr;
  float reg_linear;
  float reg_factors;
  int predict_only;          // 1: no push, no stats, no bias step
  int bias;                  // 1: w0 is read and stepped
  double* bias_acc;          // [4]: sum g, labelled (reset by the last CTA), last w0 delta, sum of w0 deltas
  unsigned int* bias_done;   // [1] CTAs finished in this launch (reset by the last CTA)
  ShardTable tab;
  int reserve_total;         // CTA slots left free for the replica exchange
  int max_ctas;              // > 0: at most this many CTAs (tests force one-CTA grids)
  ShardTable acc;            // AdaGrad accumulators, tab's geometry; base[0] == nullptr: plain SGD
};

struct __align__(16) FfmEntry {
  float* row;
  int field;
  float x;
};

// Stage the kept entries of raw entries [j0, min(j0 + FFM_CH, e)) in CSR order into ent; returns how many.  With
// PASS 1 each kept entry adds x w to lin; with PASS 2 it pushes dw (g and the row as re-pulled here).  With ADA the
// entry's H row goes to hent, and PASS 2 takes the AdaGrad step on w.
template <typename IdT, bool ONEHOT, int PASS, bool ADA = false>
__device__ __forceinline__ int ffm_stage(const FfmArgs& a, FfmEntry* ent, long long j0, long long e, float g,
                                         float& lin, bool& bad, bool& bad_id, float** hent = nullptr) {
  const IdT* __restrict__ cols = reinterpret_cast<const IdT*>(a.cols);
  const int lane = threadIdx.x & 31;
  int m = 0;
  __syncwarp();
#pragma unroll
  for (int h = 0; h < FFM_CH / 32; ++h) {
    const long long j = j0 + h * 32 + lane;
    bool keep = false;
    float* row = nullptr;
    float* hrow = nullptr;
    int f = 0;
    float x = 0.f;
    if (j < e) {
      const long long id = (long long)cols[j];
      f = a.fields[j];
      keep = id >= 0 && id < a.num_features && f >= 0 && f < a.num_fields;
      if (keep) {
        row = fps_row_t<IdT>(a.tab, (IdT)id);
        if constexpr (ADA) hrow = fps_row_t<IdT>(a.acc, (IdT)id);
        x = ONEHOT ? 1.f : a.vals[j];
      } else {
        bad_id = true;
      }
    }
    const unsigned mask = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      FfmEntry t;
      t.row = row;
      t.field = f;
      t.x = x;
      ent[m + __popc(mask & ((1u << lane) - 1u))] = t;
      if constexpr (ADA) hent[m + __popc(mask & ((1u << lane) - 1u))] = hrow;
      if (PASS == 1) {
        lin += x * fps_ld_row4(row).x;
      } else if (ADA && PASS == 2) {
        float gg;
        const float d = fps_adagrad1(g * x + a.reg_linear * fps_ld_row4(row).x, fps_ld_row4(hrow).x, a.lr, gg);
        if (!(fabsf(d) + gg <= 3.0e38f)) bad = true;
        fps_red_add1(row, d);
        fps_red_add1(hrow, gg);
      } else if (PASS == 2) {
        const float d = -a.lr * (g * x + a.reg_linear * fps_ld_row4(row).x);
        if (!(fabsf(d) <= 3.0e38f)) bad = true;
        fps_red_add1(row, d);
      }
    }
    m += __popc(mask);
  }
  __syncwarp();
  return m;
}

// Pair p of a tile: (ia, ib) into the A and B chunks.  Same chunk: the triangle ia < ib, p = ib (ib - 1) / 2 + ia;
// two chunks: the rectangle, p = ia mB + ib.
__device__ __forceinline__ void ffm_pair(int p, bool same, int mB, int& ia, int& ib) {
  if (same) {
    int b = (int)((1.f + sqrtf(8.f * (float)p + 1.f)) * 0.5f);
    if (b * (b - 1) / 2 > p) --b;
    if ((b + 1) * b / 2 <= p) ++b;
    ib = b;
    ia = p - b * (b - 1) / 2;
  } else {
    ia = p / mB;
    ib = p - ia * mB;
  }
}

template <typename IdT, int Q, int MINB, int TB, bool ONEHOT, bool ADA>
__global__ void __launch_bounds__(FFM_THREADS, MINB) fps_ffm_kernel(const __grid_constant__ FfmArgs a) {
  constexpr int P = 32 / Q;        // pairs per warp per step
  __shared__ FfmEntry s_ent[FFM_WARPS][2][FFM_CH];
  __shared__ float* s_hrow[ADA ? FFM_WARPS : 1][2][FFM_CH];   // each staged entry's H row (AdaGrad)
  const int lane = threadIdx.x & 31;
  const int li = lane & (Q - 1);   // my float4 of the slab
  const int gi = lane / Q;         // my lane-group
  FfmEntry* entA = s_ent[threadIdx.x >> 5][0];
  FfmEntry* entB = s_ent[threadIdx.x >> 5][1];
  const int kp = 4 * ((a.k + 3) / 4);
  // columns of my float4 inside the slab that hold factors: [k, kp) is padding and receives exact zeros; a lane
  // whose float4 lies past the slab (kp / 4 < Q) neither pulls nor pushes
  const int c0 = 4 * li;
  const bool on = c0 < kp;
  const bool m0 = c0 < a.k, m1 = c0 + 1 < a.k, m2 = c0 + 2 < a.k, m3 = c0 + 3 < a.k;
  const float w0 = a.bias ? fps_ld_row4(fps_row(a.tab, a.num_features)).x : 0.f;

  const long long warp = (blockIdx.x * (long long)FFM_THREADS + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * FFM_THREADS) >> 5;
  float loss_acc = 0.f, lab_acc = 0.f;
  double g_acc = 0.0;
  bool bad = false, bad_id = false;

  // one example per warp: the trip count is warp-uniform
  for (long long ex = warp; ex < a.n; ex += n_warps) {
    long long e = a.row_ptr[ex + 1];
    long long b = a.row_ptr[ex];
    if (e > a.nnz) e = a.nnz;
    if (b < 0) b = 0;
    if (b > e) b = e;
    const int nc = (int)((e - b + FFM_CH - 1) / FFM_CH);
    // ---- pass 1: linear term and pair terms --------------------------------------------------------------
    float acc = 0.f, lin = 0.f;
    for (int A = 0; A < nc; ++A) {
      const int mA = ffm_stage<IdT, ONEHOT, 1>(a, entA, b + (long long)A * FFM_CH, e, 0.f, lin, bad, bad_id);
      for (int B = A; B < nc; ++B) {
        float unused = 0.f;
        const int mB = B == A ? mA : ffm_stage<IdT, ONEHOT, 0>(a, entB, b + (long long)B * FFM_CH, e, 0.f, unused,
                                                               bad, bad_id);
        const FfmEntry* eb = B == A ? entA : entB;
        const int np = B == A ? mA * (mA - 1) / 2 : mA * mB;
        for (int p0 = 0; p0 < np; p0 += P * TB) {
          float4 ra[TB], rb[TB];
          float xx[TB];
#pragma unroll
          for (int t = 0; t < TB; ++t) {
            const int p = p0 + t * P + gi;
            xx[t] = 0.f;
            ra[t] = make_float4(0.f, 0.f, 0.f, 0.f);
            rb[t] = ra[t];
            if (p < np && on) {
              int ia, ib;
              ffm_pair(p, B == A, mB, ia, ib);
              const FfmEntry ea = entA[ia], ebb = eb[ib];
              xx[t] = ea.x * ebb.x;
              ra[t] = fps_ld_row4(ea.row + 4 + ebb.field * kp + c0);   // V[i_a, f_b]
              rb[t] = fps_ld_row4(ebb.row + 4 + ea.field * kp + c0);   // V[i_b, f_a]
            }
          }
#pragma unroll
          for (int t = 0; t < TB; ++t)
            acc += xx[t] * (ra[t].x * rb[t].x + ra[t].y * rb[t].y + ra[t].z * rb[t].z + ra[t].w * rb[t].w);
        }
      }
    }
    const float yhat = w0 + fps_group_sum<32>(lin + acc);
    if (lane == 0) a.pred[ex] = yhat;
    if (a.predict_only) continue;
    const float y = a.labels[ex];
    if (y != y) continue;
    float g;
    if (a.loss == FM_LOGISTIC) {
      g = 1.f / (1.f + expf(-yhat)) - y;
      if (lane == 0) loss_acc += fmaxf(yhat, 0.f) + log1pf(expf(-fabsf(yhat))) - y * yhat;
    } else {
      g = yhat - y;
      if (lane == 0) loss_acc += g * g;
    }
    if (lane == 0) {
      lab_acc += 1.f;
      g_acc += (double)g;
    }
    // ---- pass 2: re-pull both slabs of every pair (AdaGrad: with their H), push the deltas; dw as staged ----
    if constexpr (ADA) {
      float** hA = s_hrow[threadIdx.x >> 5][0];
      float** hB = s_hrow[threadIdx.x >> 5][1];
      for (int A = 0; A < nc; ++A) {
        float unused = 0.f;
        const int mA = ffm_stage<IdT, ONEHOT, 2, true>(a, entA, b + (long long)A * FFM_CH, e, g, unused, bad, bad_id,
                                                        hA);
        for (int B = A; B < nc; ++B) {
          const int mB = B == A ? mA : ffm_stage<IdT, ONEHOT, 0, true>(a, entB, b + (long long)B * FFM_CH, e, 0.f,
                                                                       unused, bad, bad_id, hB);
          const FfmEntry* eb = B == A ? entA : entB;
          float* const* hb_ = B == A ? hA : hB;
          const int np = B == A ? mA * (mA - 1) / 2 : mA * mB;
          for (int p0 = 0; p0 < np; p0 += P * TB) {
            float4 ra[TB], rb[TB], ha[TB], hb[TB];
            float* pa[TB];
            float* pb[TB];
            float* qa[TB];
            float* qb[TB];
            float cc[TB];
#pragma unroll
            for (int t = 0; t < TB; ++t) {
              const int p = p0 + t * P + gi;
              pa[t] = nullptr;
              pb[t] = nullptr;
              qa[t] = nullptr;
              qb[t] = nullptr;
              cc[t] = 0.f;
              ra[t] = make_float4(0.f, 0.f, 0.f, 0.f);
              rb[t] = ra[t];
              ha[t] = ra[t];
              hb[t] = ra[t];
              if (p < np && on) {
                int ia, ib;
                ffm_pair(p, B == A, mB, ia, ib);
                const FfmEntry ea = entA[ia], ebb = eb[ib];
                cc[t] = g * (ea.x * ebb.x);
                const int oa = 4 + ebb.field * kp + c0, ob = 4 + ea.field * kp + c0;
                pa[t] = ea.row + oa;
                pb[t] = ebb.row + ob;
                qa[t] = hA[ia] + oa;
                qb[t] = hb_[ib] + ob;
                ra[t] = fps_ld_row4(pa[t]);
                rb[t] = fps_ld_row4(pb[t]);
                ha[t] = fps_ld_row4(qa[t]);
                hb[t] = fps_ld_row4(qb[t]);
              }
            }
#pragma unroll
            for (int t = 0; t < TB; ++t) {
              if (pa[t] == nullptr) continue;
              const float c = cc[t], rv = a.reg_factors;
              float4 ga, gb, gga, ggb;
              ga.x = m0 ? c * rb[t].x + rv * ra[t].x : 0.f;
              ga.y = m1 ? c * rb[t].y + rv * ra[t].y : 0.f;
              ga.z = m2 ? c * rb[t].z + rv * ra[t].z : 0.f;
              ga.w = m3 ? c * rb[t].w + rv * ra[t].w : 0.f;
              gb.x = m0 ? c * ra[t].x + rv * rb[t].x : 0.f;
              gb.y = m1 ? c * ra[t].y + rv * rb[t].y : 0.f;
              gb.z = m2 ? c * ra[t].z + rv * rb[t].z : 0.f;
              gb.w = m3 ? c * ra[t].w + rv * rb[t].w : 0.f;
              const float4 da = fps_adagrad4(ga, ha[t], a.lr, gga);
              const float4 db = fps_adagrad4(gb, hb[t], a.lr, ggb);
              if (!(fabsf(da.x) + fabsf(da.y) + fabsf(da.z) + fabsf(da.w) + fabsf(db.x) + fabsf(db.y) + fabsf(db.z) +
                        fabsf(db.w) + gga.x + gga.y + gga.z + gga.w + ggb.x + ggb.y + ggb.z + ggb.w <= 3.0e38f))
                bad = true;
              fps_red_add4(pa[t], da);
              fps_red_add4(pb[t], db);
              fps_red_add4(qa[t], gga);
              fps_red_add4(qb[t], ggb);
            }
          }
        }
      }
    } else {
      for (int A = 0; A < nc; ++A) {
        float unused = 0.f;
        const int mA = ffm_stage<IdT, ONEHOT, 2>(a, entA, b + (long long)A * FFM_CH, e, g, unused, bad, bad_id);
        for (int B = A; B < nc; ++B) {
          const int mB = B == A ? mA : ffm_stage<IdT, ONEHOT, 0>(a, entB, b + (long long)B * FFM_CH, e, 0.f, unused,
                                                                 bad, bad_id);
          const FfmEntry* eb = B == A ? entA : entB;
          const int np = B == A ? mA * (mA - 1) / 2 : mA * mB;
          for (int p0 = 0; p0 < np; p0 += P * TB) {
            float4 ra[TB], rb[TB];
            float* pa[TB];
            float* pb[TB];
            float cc[TB];
#pragma unroll
            for (int t = 0; t < TB; ++t) {
              const int p = p0 + t * P + gi;
              pa[t] = nullptr;
              pb[t] = nullptr;
              cc[t] = 0.f;
              ra[t] = make_float4(0.f, 0.f, 0.f, 0.f);
              rb[t] = ra[t];
              if (p < np && on) {
                int ia, ib;
                ffm_pair(p, B == A, mB, ia, ib);
                const FfmEntry ea = entA[ia], ebb = eb[ib];
                cc[t] = g * (ea.x * ebb.x);
                pa[t] = ea.row + 4 + ebb.field * kp + c0;
                pb[t] = ebb.row + 4 + ea.field * kp + c0;
                ra[t] = fps_ld_row4(pa[t]);
                rb[t] = fps_ld_row4(pb[t]);
              }
            }
#pragma unroll
            for (int t = 0; t < TB; ++t) {
              if (pa[t] == nullptr) continue;
              const float c = cc[t], rv = a.reg_factors, lr = a.lr;
              float4 da, db;
              da.x = m0 ? -lr * (c * rb[t].x + rv * ra[t].x) : 0.f;
              da.y = m1 ? -lr * (c * rb[t].y + rv * ra[t].y) : 0.f;
              da.z = m2 ? -lr * (c * rb[t].z + rv * ra[t].z) : 0.f;
              da.w = m3 ? -lr * (c * rb[t].w + rv * ra[t].w) : 0.f;
              db.x = m0 ? -lr * (c * ra[t].x + rv * rb[t].x) : 0.f;
              db.y = m1 ? -lr * (c * ra[t].y + rv * rb[t].y) : 0.f;
              db.z = m2 ? -lr * (c * ra[t].z + rv * rb[t].z) : 0.f;
              db.w = m3 ? -lr * (c * ra[t].w + rv * rb[t].w) : 0.f;
              if (!(fabsf(da.x) + fabsf(da.y) + fabsf(da.z) + fabsf(da.w) + fabsf(db.x) + fabsf(db.y) + fabsf(db.z) +
                        fabsf(db.w) <= 3.0e38f))
                bad = true;
              fps_red_add4(pa[t], da);
              fps_red_add4(pb[t], db);
            }
          }
        }
      }
    }
  }
  fps_fm_bias_tail(a, bad, bad_id, loss_acc, lab_acc, g_acc);
}

template <typename IdT, int Q, int MINB, int TB, bool ADA>
static int launch_ffm(const FfmArgs& a, int num_sms, cudaStream_t stream) {
  void (*kern)(const FfmArgs) = a.vals == nullptr ? fps_ffm_kernel<IdT, Q, MINB, TB, true, ADA>
                                                  : fps_ffm_kernel<IdT, Q, MINB, TB, false, ADA>;
  long long blocks = fps_row_grid(kern, FFM_THREADS, FFM_WARPS, num_sms, a.reserve_total, 0, 1, a.n, 1);
  if (a.max_ctas > 0 && blocks > a.max_ctas) blocks = a.max_ctas;
  kern<<<(int)blocks, FFM_THREADS, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// Q = kp / 4 rounded up to a power of two lanes per pair; MINB keeps every instantiation free of spills (ptxas -v, DESIGN §3).
// AdaGrad holds two more float4 and two more pointers per pair in flight, so it runs TB = ADA_TB pairs per lane.
#define FFM_ADA_TB 2
template <typename IdT, bool ADA>
static int ffm_dispatch(const FfmArgs& a, int num_sms, cudaStream_t s) {
  constexpr int TB = ADA ? FFM_ADA_TB : 4;
  const int q = (a.k + 3) / 4;
  if (q <= 1) return launch_ffm<IdT, 1, 2, TB, ADA>(a, num_sms, s);
  if (q <= 2) return launch_ffm<IdT, 2, 2, TB, ADA>(a, num_sms, s);
  if (q <= 4) return launch_ffm<IdT, 4, 2, TB, ADA>(a, num_sms, s);
  if (q <= 8) return launch_ffm<IdT, 8, 2, TB, ADA>(a, num_sms, s);
  return launch_ffm<IdT, 16, 2, TB, ADA>(a, num_sms, s);
}

extern "C" int fps_ffm_step(const FfmArgs* args, int id_bytes, int num_sms, cudaStream_t stream) {
  const FfmArgs& a = *args;
  if (a.k < 1 || a.k > FFM_MAX_K || a.num_fields < 1 || a.num_fields > FFM_MAX_FIELDS) return -1702;
  if (a.tab.stride != 4 + a.num_fields * 4 * ((a.k + 3) / 4) || a.tab.dim != a.tab.stride) return -1701;
  if (a.loss != FM_LOGISTIC && a.loss != FM_SQUARED) return -1703;
  if (a.n < 0 || a.n >= INT_MAX || a.nnz < 0 || a.num_features < 0) return -1704;
  if (a.bias && !a.predict_only && (a.bias_acc == nullptr || a.bias_done == nullptr)) return -1705;
  const bool ada = a.acc.base[0] != nullptr;
  if (ada && !fps_same_geometry(a.acc, a.tab)) return -1706;
  if (a.n == 0) return 0;
  // predictions come from the AdaGrad kernel too (its pass 1 sums in the same blocks as its training step); with
  // predict_only it never reaches H
  if (id_bytes == 4) return ada ? ffm_dispatch<int, true>(a, num_sms, stream) : ffm_dispatch<int, false>(a, num_sms, stream);
  if (id_bytes == 8)
    return ada ? ffm_dispatch<long long, true>(a, num_sms, stream) : ffm_dispatch<long long, false>(a, num_sms, stream);
  return -1001;
}
