// Factorization machine step on a CSR micro-batch (DESIGN §2.15), fused with the pulls and pushes.
//
// Table: num_features + 1 rows of dim = 1 + k floats, stride = round_up(dim, 4).  Row i = [w_i | v_i,1..k | 0 pad];
// row num_features is the bias row, w0 in column 0.  For an example with entries (i_j, x_j):
//   s_f = sum_j x_j v_{i_j,f},   yhat = w0 + sum_j x_j w_{i_j} + 1/2 sum_f (s_f^2 - sum_j x_j^2 v_{i_j,f}^2)
//   logistic: g = sigmoid(yhat) - y, loss = softplus(yhat) - y yhat;   squared: g = yhat - y, loss = (yhat - y)^2
// and per entry (i, x) of a labelled example, with the row as the example pulled it:
//   dw_i = -lr (g x + reg_linear w_i),   dv_i,f = -lr (g x (s_f - x v_i,f) + reg_factors v_i,f),   pad: 0
// pushed with red.add.v4.f32.  A NaN label only predicts.  w0 is stepped once per launch by the mean of g over
// the labelled examples: every example reads w0 as it was before the launch, and the last CTA to finish (a
// launch counter that resets itself, behind __threadfence) pushes -lr * sum g / n_labelled to the bias row.  One
// launch per step, nothing on the host.
//
// Geometry: one lane-group of LPR lanes per example, lane l holding float4 chunks l, l + LPR, .. (VPL of them).
// Pass 1 pulls TB rows at a time and keeps s_f and the lane's share of x^2 v^2 in registers; yhat is one group
// sum.  Pass 2 re-pulls each row (an L2 hit: pass 1 has just read it) and pushes its delta.  Entries whose id is
// outside [0, num_features) are skipped and raise *bad_id; the end of every example is clamped to nnz.
//
// AdaGrad (DESIGN §2.17, libffm's element-wise rule): with acc.base[0] set, acc is a second table of the same
// geometry holding H = G - 1 per element (a zero heap is the starting state), and the step launches fps_fm_kernel
// with ADA set.  Everything up to g is shared; only pass 2 differs: for every element the SGD rule would step by
// -lr * gam (gam = the bracket above), fm_push_adagrad pulls H with the row chunk and pushes
//   dtheta = -lr * gam / sqrtf(1 + H + gam^2)   and   dH = gam^2
// with two red.add.v4.f32 (padding: gam = 0, so both stay exactly zero).  w0 keeps the SGD rule.  The two pass 2
// bodies stay apart: one body with the H loads under if constexpr changes the SGD instantiations' code.
#include <limits.h>
#include "fps_common.cuh"
#include "fps_fm_bias.cuh"
#include "fps_launch.cuh"

#define FM_THREADS 256
#define FM_BIT(c, i) ((fbits >> (4 * (c) + (i))) & 1u)

struct FmArgs {
  const long long* row_ptr;  // [n + 1]
  const void* cols;          // [nnz] int32 or int64 feature ids
  const float* vals;         // [nnz] values, or nullptr: one-hot (every x = 1)
  const float* labels;       // [n] float32; NaN = predict only
  float* pred;               // [n] out: yhat before the example's own update
  float* stats;              // [2] += loss, labelled examples (may be null)
  int* nan_flag;             // set by a non-finite delta (may be null)
  int* bad_id;               // set by an entry whose id is outside [0, num_features) (may be null)
  long long n;
  long long nnz;
  long long num_features;    // the bias row's id
  int dim;                   // 1 + k
  int loss;                  // FmLoss
  float lr;
  float reg_linear;
  float reg_factors;
  int predict_only;          // 1: no push, no stats, no bias step
  int bias;                  // 1: w0 is read and stepped
  int pad_;
  double* bias_acc;          // [4]: sum g, labelled (reset by the last CTA), last w0 delta, sum of w0 deltas
  unsigned int* bias_done;   // [1] CTAs finished in this launch (reset by the last CTA)
  ShardTable tab;
  int reserve_total;         // CTA slots left free for the replica exchange
  int max_ctas;              // > 0: at most this many CTAs (tests force one-CTA grids)
  ShardTable acc;            // AdaGrad accumulators, tab's geometry; base[0] == nullptr: plain SGD
};

// AdaGrad pass 2 of one example (entries [b, e), gradient g, s = sum x v): re-pull each row chunk with its H chunk,
// push dtheta and gam^2.  fbits as in fps_fm_kernel.
template <typename IdT, int LPR, int VPL, int TB, bool ONEHOT>
__device__ __forceinline__ void fm_push_adagrad(const FmArgs& a, long long b, long long e, float g,
                                                const float4 (&s)[VPL], unsigned fbits, bool& bad) {
  const IdT* __restrict__ cols = reinterpret_cast<const IdT*>(a.cols);
  const int lane = threadIdx.x & (LPR - 1);
  const int nvec = a.tab.stride >> 2;
  const bool has_w = lane == 0;
  for (long long j0 = b; j0 < e; j0 += TB) {
    float x[TB];
    float* rp[TB];
    float* hp[TB];
    float4 r[TB][VPL], h[TB][VPL];
#pragma unroll
    for (int t = 0; t < TB; ++t) {
      const long long j = j0 + t;
      rp[t] = nullptr;
      hp[t] = nullptr;
      x[t] = 0.f;
      if (j < e) {
        const long long id = (long long)cols[j];
        if (id >= 0 && id < a.num_features) {
          rp[t] = fps_row_t<IdT>(a.tab, (IdT)id);
          hp[t] = fps_row_t<IdT>(a.acc, (IdT)id);
          x[t] = ONEHOT ? 1.f : a.vals[j];
        }
      }
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        const bool ld = rp[t] != nullptr && q < nvec;
        r[t][c] = ld ? fps_ld_row4(rp[t] + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
        h[t][c] = ld ? fps_ld_row4(hp[t] + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int t = 0; t < TB; ++t) {
      if (rp[t] == nullptr) continue;
      const float gx = g * x[t];
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        if (q >= nvec) continue;
        const float4 v = r[t][c];
        float4 gm;   // gam, the SGD step's bracket
        gm.x = FM_BIT(c, 0) ? gx * (s[c].x - x[t] * v.x) + a.reg_factors * v.x : 0.f;
        gm.y = FM_BIT(c, 1) ? gx * (s[c].y - x[t] * v.y) + a.reg_factors * v.y : 0.f;
        gm.z = FM_BIT(c, 2) ? gx * (s[c].z - x[t] * v.z) + a.reg_factors * v.z : 0.f;
        gm.w = FM_BIT(c, 3) ? gx * (s[c].w - x[t] * v.w) + a.reg_factors * v.w : 0.f;
        if (c == 0 && has_w) gm.x = gx + a.reg_linear * v.x;
        float4 gg;
        const float4 d = fps_adagrad4(gm, h[t][c], a.lr, gg);
        if (!(fabsf(d.x) + fabsf(d.y) + fabsf(d.z) + fabsf(d.w) + gg.x + gg.y + gg.z + gg.w <= 3.0e38f)) bad = true;
        fps_red_add4(rp[t] + 4 * q, d);
        fps_red_add4(hp[t] + 4 * q, gg);
      }
    }
  }
}

template <typename IdT, int LPR, int VPL, int MINB, int TB, bool ONEHOT, bool ADA>
__global__ void __launch_bounds__(FM_THREADS, MINB) fps_fm_kernel(const __grid_constant__ FmArgs a) {
  constexpr int GPW = 32 / LPR;   // examples per warp per round
  const IdT* __restrict__ cols = reinterpret_cast<const IdT*>(a.cols);
  const int lane = threadIdx.x & (LPR - 1);
  const int nvec = a.tab.stride >> 2;
  const int dim = a.dim;
  // factor columns of my chunks: bit 4c + i is set iff column 4 (lane + c LPR) + i lies in [1, dim)
  unsigned fbits = 0u;
#pragma unroll
  for (int c = 0; c < VPL; ++c)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int col = 4 * (lane + c * LPR) + i;
      if (col >= 1 && col < dim) fbits |= 1u << (4 * c + i);
    }
  const bool has_w = lane == 0;   // chunk 0, column 0 of every row is w
  const float w0 = a.bias ? fps_ld_row4(fps_row(a.tab, a.num_features)).x : 0.f;

  const long long warp = (blockIdx.x * (long long)FM_THREADS + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * FM_THREADS) >> 5;
  const int grp = (threadIdx.x & 31) / LPR;
  float loss_acc = 0.f, lab_acc = 0.f;
  double g_acc = 0.0;
  bool bad = false, bad_id = false;

  // warp-uniform trip count: every lane reaches the group sums of every round
  for (long long base = warp * GPW; base < a.n; base += n_warps * GPW) {
    const long long ex = base + grp;
    const bool live = ex < a.n;
    long long b = 0, e = 0;
    if (live) {
      e = a.row_ptr[ex + 1];
      b = a.row_ptr[ex];
      if (e > a.nnz) e = a.nnz;
      if (b < 0) b = 0;
      if (b > e) b = e;
    }
    // ---- pass 1: linear term, s, sum x^2 v^2 ------------------------------------------------------------
    float4 s[VPL];
#pragma unroll
    for (int c = 0; c < VPL; ++c) s[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    float lin = 0.f, sq = 0.f;
    for (long long j0 = b; j0 < e; j0 += TB) {
      float x[TB];
      float4 r[TB][VPL];
#pragma unroll
      for (int t = 0; t < TB; ++t) {
        const long long j = j0 + t;
        x[t] = 0.f;
        const float* row = nullptr;
        if (j < e) {
          const long long id = (long long)cols[j];
          if (id >= 0 && id < a.num_features) {
            row = fps_row_t<IdT>(a.tab, (IdT)id);
            x[t] = ONEHOT ? 1.f : a.vals[j];
          } else {
            bad_id = true;
          }
        }
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const int q = lane + c * LPR;
          r[t][c] = (row != nullptr && q < nvec) ? fps_ld_row4(row + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int t = 0; t < TB; ++t) {
        if (has_w) lin += x[t] * r[t][0].x;
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const float4 v = make_float4(FM_BIT(c, 0) ? x[t] * r[t][c].x : 0.f, FM_BIT(c, 1) ? x[t] * r[t][c].y : 0.f,
                                       FM_BIT(c, 2) ? x[t] * r[t][c].z : 0.f, FM_BIT(c, 3) ? x[t] * r[t][c].w : 0.f);
          s[c].x += v.x; s[c].y += v.y; s[c].z += v.z; s[c].w += v.w;
          sq += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
        }
      }
    }
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < VPL; ++c) ss += s[c].x * s[c].x + s[c].y * s[c].y + s[c].z * s[c].z + s[c].w * s[c].w;
    const float yhat = w0 + fps_group_sum<LPR>(lin + 0.5f * (ss - sq));
    if (!live) continue;
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
    // ---- pass 2: re-pull (with H under AdaGrad), delta, push ----------------------------------------------
    if constexpr (ADA) {
      fm_push_adagrad<IdT, LPR, VPL, TB, ONEHOT>(a, b, e, g, s, fbits, bad);
    } else {
      for (long long j0 = b; j0 < e; j0 += TB) {
        float x[TB];
        float* rp[TB];
        float4 r[TB][VPL];
#pragma unroll
        for (int t = 0; t < TB; ++t) {
          const long long j = j0 + t;
          rp[t] = nullptr;
          x[t] = 0.f;
          if (j < e) {
            const long long id = (long long)cols[j];
            if (id >= 0 && id < a.num_features) {
              rp[t] = fps_row_t<IdT>(a.tab, (IdT)id);
              x[t] = ONEHOT ? 1.f : a.vals[j];
            }
          }
#pragma unroll
          for (int c = 0; c < VPL; ++c) {
            const int q = lane + c * LPR;
            r[t][c] = (rp[t] != nullptr && q < nvec) ? fps_ld_row4(rp[t] + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int t = 0; t < TB; ++t) {
          if (rp[t] == nullptr) continue;
          const float gx = g * x[t];
#pragma unroll
          for (int c = 0; c < VPL; ++c) {
            const int q = lane + c * LPR;
            if (q >= nvec) continue;
            const float4 v = r[t][c];
            float4 d;
            d.x = FM_BIT(c, 0) ? -a.lr * (gx * (s[c].x - x[t] * v.x) + a.reg_factors * v.x) : 0.f;
            d.y = FM_BIT(c, 1) ? -a.lr * (gx * (s[c].y - x[t] * v.y) + a.reg_factors * v.y) : 0.f;
            d.z = FM_BIT(c, 2) ? -a.lr * (gx * (s[c].z - x[t] * v.z) + a.reg_factors * v.z) : 0.f;
            d.w = FM_BIT(c, 3) ? -a.lr * (gx * (s[c].w - x[t] * v.w) + a.reg_factors * v.w) : 0.f;
            if (c == 0 && has_w) d.x = -a.lr * (gx + a.reg_linear * v.x);
            if (!(fabsf(d.x) + fabsf(d.y) + fabsf(d.z) + fabsf(d.w) <= 3.0e38f)) bad = true;
            fps_red_add4(rp[t] + 4 * q, d);   // the PUSH fused with paramUpdate (+)
          }
        }
      }
    }
  }
  fps_fm_bias_tail(a, bad, bad_id, loss_acc, lab_acc, g_acc);   // per-warp sums; the last CTA steps w0
}

template <typename IdT, int LPR, int VPL, int MINB, int TB, bool ADA>
static int launch_fm(const FmArgs& a, int num_sms, cudaStream_t stream) {
  void (*kern)(const FmArgs) = a.vals == nullptr ? fps_fm_kernel<IdT, LPR, VPL, MINB, TB, true, ADA>
                                                 : fps_fm_kernel<IdT, LPR, VPL, MINB, TB, false, ADA>;
  long long blocks = fps_row_grid(kern, FM_THREADS, FM_THREADS / LPR, num_sms, a.reserve_total, 0, 1, a.n, 1);
  if (a.max_ctas > 0 && blocks > a.max_ctas) blocks = a.max_ctas;
  kern<<<(int)blocks, FM_THREADS, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// Lane geometry of w2v_dispatch: LPR = nvec up to 32 float4, then 32 lanes with VPL = 2, 3 or 4; MINB keeps every
// instantiation free of spills (ptxas -v, DESIGN §3).  Under AdaGrad the H chunks double r[TB][VPL], so the narrow
// rungs pull 4 rows at a time instead of 8.
template <typename IdT, bool ADA>
static int fm_dispatch(const FmArgs& a, int num_sms, cudaStream_t s) {
  constexpr int TB = ADA ? 4 : 8;
  const int nvec = a.tab.stride >> 2;
  if (nvec <= 1) return launch_fm<IdT, 1, 1, 2, TB, ADA>(a, num_sms, s);
  if (nvec <= 2) return launch_fm<IdT, 2, 1, 2, TB, ADA>(a, num_sms, s);
  if (nvec <= 4) return launch_fm<IdT, 4, 1, 2, TB, ADA>(a, num_sms, s);
  if (nvec <= 8) return launch_fm<IdT, 8, 1, 2, TB, ADA>(a, num_sms, s);
  if (nvec <= 16) return launch_fm<IdT, 16, 1, 2, TB, ADA>(a, num_sms, s);
  if (nvec <= 32) return launch_fm<IdT, 32, 1, 2, TB, ADA>(a, num_sms, s);
  if (nvec <= 64) return launch_fm<IdT, 32, 2, 1, 4, ADA>(a, num_sms, s);
  if (nvec <= 96) return launch_fm<IdT, 32, 3, 1, 4, ADA>(a, num_sms, s);
  if (nvec <= 128) return launch_fm<IdT, 32, 4, 1, 4, ADA>(a, num_sms, s);
  return -1000;   // rows wider than 512 floats
}

extern "C" int fps_fm_step(const FmArgs* args, int id_bytes, int num_sms, cudaStream_t stream) {
  const FmArgs& a = *args;
  if (a.tab.stride <= 0 || (a.tab.stride & 3) != 0) return -1601;
  if (a.dim < 1 || a.dim > a.tab.stride) return -1602;
  if (a.loss != FM_LOGISTIC && a.loss != FM_SQUARED) return -1603;
  if (a.n < 0 || a.n >= INT_MAX || a.nnz < 0 || a.num_features < 0) return -1604;
  if (a.bias && !a.predict_only && (a.bias_acc == nullptr || a.bias_done == nullptr)) return -1605;
  const bool ada = a.acc.base[0] != nullptr;
  if (ada && !fps_same_geometry(a.acc, a.tab)) return -1606;
  if (a.n == 0) return 0;
  // predictions come from the AdaGrad kernel too (its pass 1 sums in the same blocks as its training step); with
  // predict_only it never reaches H
  if (id_bytes == 4)
    return ada ? fm_dispatch<int, true>(a, num_sms, stream) : fm_dispatch<int, false>(a, num_sms, stream);
  if (id_bytes == 8)
    return ada ? fm_dispatch<long long, true>(a, num_sms, stream) : fm_dispatch<long long, false>(a, num_sms, stream);
  return -1001;
}
