// WARP (Weighted Approximate-Rank Pairwise, Weston, Bengio and Usunier 2011) matrix-factorisation step for
// sm_90a: pull + sample-until-violation + one hinge update per positive, in one kernel, next to the BPR step of
// fps_mf_bpr.cu (same argument block, same row addressing, same candidate stream).
//
// For every positive record (a, i) with rating > 0, u = anchor row and v_i pulled once, and T = n_neg:
//   candidates t = 0 .. T-1: negatives[pos, t], or BPR's sampled negative t (K5 Philox key (pos, t+1, step, seed));
//                            -1 or the positive itself is void: skipped and not counted
//   x_t = u . (v_i - v_j)    for the live candidates in order, n = live candidates examined so far
//   the first t* with x_t < margin is the violator; then, with N = rank_items,
//     L = ln(max(1, floor((N - 1) / n))),  g = lr * L
//     u   += g * (v_i - v_j) - lr*reg*u      (REDG.ADD.F32x4)
//     v_i += g * u           - lr*reg*v_i    (push)
//     v_j += -g * u          - lr*reg*v_j    (push)
//   no violator among the T candidates: nothing is written.
//   stats[0] += L * (margin - x_t*), [1] += #updated, [2] += #live candidates examined, [3] += #positives
// Every delta is computed from the values as pulled.
//
// Candidates are examined in blocks of C: a block forms C ids, issues all C row pulls, then computes the C dot
// products and takes the first violator in draw order.  Because the violator is the first in draw order and
// each x_t is the same expression whatever the block it sits in, the result is bitwise independent of C.
// The trial loop runs until every lane-group of the warp is done (__any_sync): fps_group_sum shuffles with a
// full-warp mask, so a finished group keeps taking part with its loads and pushes predicated off.
#include "fps_common.cuh"
#include "fps_mf_args.cuh"

template <typename IdT, int LPR, int VPL, int MINB, int FMT, int C>
__global__ void __launch_bounds__(256, MINB) fps_mf_warp_kernel(const __grid_constant__ BprArgs a) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int stride = a.stride;
  const int nvec = stride >> 2;
  const float decay = a.lr * a.reg;
  const int T = a.n_neg;
  const IdT* __restrict__ negs = reinterpret_cast<const IdT*>(a.negatives);
  float loss_acc = 0.f, upd_acc = 0.f, trial_acc = 0.f, pos_acc = 0.f;
  bool bad = false;

  // the trip count is the same for every lane of a warp (n_groups is a multiple of 32 / LPR)
  const long long n_round = ((a.n_pos + n_groups - 1) / n_groups) * n_groups;
  for (long long pos = group; pos < n_round; pos += n_groups) {
    bool ok = pos < a.n_pos;
    IdT anchor = 0, item = 0;
    if (ok) {
      const FpsRecord<IdT> rec = fps_record<IdT>(FMT, a.users, a.items, a.ratings, pos);
      anchor = rec.user;
      item = rec.item;
      const float rating = rec.rating;
      ok = rating > 0.f && anchor >= 0 && item >= 0;
    }
    float* up = bpr_row<IdT>(a.anchor_table, a.anchor_div, a.anchor_shift, a.anchor_sharded,
                             a.anchor_tab, anchor, stride);
    float* vip = bpr_row<IdT>(a.cand_table, a.cand_div, a.cand_shift, a.cand_sharded, a.cand_tab,
                              item, stride);
    float4 u[VPL], vi[VPL], vs[VPL];
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int q = lane + c * LPR;
      if (ok && q < nvec) {
        u[c] = a.anchor_sharded ? fps_ld_row4(up + 4 * q) : *reinterpret_cast<const float4*>(up + 4 * q);
        vi[c] = fps_ld_row4(vip + 4 * q);   // the PULLs
      } else {
        u[c] = make_float4(0.f, 0.f, 0.f, 0.f);
        vi[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      vs[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (ok && lane == 0) pos_acc += 1.f;
    bool active = ok;          // this group is still looking for a violator
    bool hit = false;
    long long jstar = -1;      // the violator's id
    float xstar = 0.f;
    int n = 0;                 // live candidates examined
    for (int t0 = 0; __any_sync(0xffffffffu, active); t0 += C) {
      long long cand[C];
      float4 vj[C][VPL];
#pragma unroll
      for (int b = 0; b < C; ++b) {   // form the block's ids and issue all of its pulls
        const int t = t0 + b;
        long long neg = -1;
        if (active && t < T) {
          if (negs != nullptr) {
            neg = (long long)negs[pos * T + t];
          } else if (a.num_items > 1) {   // BPR's negative t: K5, record pos, negative number t + 1
            neg = fps_k5_negative(a, pos, t + 1, item);
          }
          if (neg == (long long)item) neg = -1;
        }
        cand[b] = neg;
        const bool live = neg >= 0;
        const float* vjp = bpr_row<IdT>(a.cand_table, a.cand_div, a.cand_shift, a.cand_sharded, a.cand_tab,
                                        (IdT)(live ? neg : 0), stride);
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const int q = lane + c * LPR;
          vj[b][c] = (live && q < nvec) ? fps_ld_row4(vjp + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int b = 0; b < C; ++b) {   // the C values of x, then the first violator in draw order
        float d = 0.f;
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          d += u[c].x * (vi[c].x - vj[b][c].x) + u[c].y * (vi[c].y - vj[b][c].y) +
               u[c].z * (vi[c].z - vj[b][c].z) + u[c].w * (vi[c].w - vj[b][c].w);
        }
        const float x = fps_group_sum<LPR>(d);
        if (active && cand[b] >= 0) {
          if (!(fabsf(x) <= 3.0e38f)) bad = true;   // NaN/Inf guard
          ++n;
          if (x < a.margin) {
            active = false;
            hit = true;
            jstar = cand[b];
            xstar = x;
#pragma unroll
            for (int c = 0; c < VPL; ++c) vs[c] = vj[b][c];
          }
        }
      }
      if (t0 + C >= T) active = false;
    }
    if (ok && lane == 0) trial_acc += (float)n;
    if (hit) {
      long long r = (a.rank_items - 1) / n;
      const float L = logf((float)(r > 1 ? r : 1));
      const float g = a.lr * L;
      if (lane == 0) {
        loss_acc += L * (a.margin - xstar);
        upd_acc += 1.f;
      }
      float* pi = (a.cand_sharded && a.use_push_tab) ? fps_row_t<IdT>(a.push_tab, item) : vip;
      float* pj = (a.cand_sharded && a.use_push_tab)
                      ? fps_row_t<IdT>(a.push_tab, (IdT)jstar)
                      : bpr_row<IdT>(a.cand_table, a.cand_div, a.cand_shift, a.cand_sharded, a.cand_tab,
                                     (IdT)jstar, stride);
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        if (q < nvec) {
          const float4 diff = make_float4(vi[c].x - vs[c].x, vi[c].y - vs[c].y, vi[c].z - vs[c].z,
                                          vi[c].w - vs[c].w);
          fps_red_add4(up + 4 * q, bpr_axpy(g, diff, -decay, u[c]));    // anchor update
          fps_red_add4(pi + 4 * q, bpr_axpy(g, u[c], -decay, vi[c]));   // the PUSH of v_i
          fps_red_add4(pj + 4 * q, bpr_axpy(-g, u[c], -decay, vs[c]));  // the PUSH of v_j
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);
    upd_acc += __shfl_xor_sync(0xffffffffu, upd_acc, o);
    trial_acc += __shfl_xor_sync(0xffffffffu, trial_acc, o);
    pos_acc += __shfl_xor_sync(0xffffffffu, pos_acc, o);
  }
  if ((threadIdx.x & 31) == 0 && a.stats != nullptr && pos_acc > 0.f) {
    atomicAdd(a.stats + 0, loss_acc);
    atomicAdd(a.stats + 1, upd_acc);
    atomicAdd(a.stats + 2, trial_acc);
    atomicAdd(a.stats + 3, pos_acc);
  }
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
}

// Static pull limiter: a lane-group has up to 2 + C rows in flight (u, v_i and a block of C candidates), so the
// grid is capped at max_inflight_rows / ((2 + C) * lane-groups per CTA).  `reserve_total` CTA slots stay free
// for the replica exchange that runs next to the step (as in launch_bpr).
template <typename IdT, int LPR, int VPL, int MINB, int FMT, int C>
static int launch_warp(const BprArgs& a, int max_inflight_rows, int num_sms, cudaStream_t stream) {
  const int threads = 256;
  void (*kern)(const BprArgs) = fps_mf_warp_kernel<IdT, LPR, VPL, MINB, FMT, C>;
  const long long blocks = fps_row_grid(kern, threads, threads / LPR, num_sms, a.reserve_total, max_inflight_rows,
                                        2 + C, a.n_pos, 1);
  kern<<<(int)blocks, threads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// One lane geometry: the trial block C (0 = this geometry's default, DC), each C with the MINB that keeps it
// free of spills (ptxas -v, DESIGN §2.12).  8-byte ids hold C more registers of candidate ids: their C = 2 and
// C = 4 kernels take one CTA per SM less.
template <typename IdT, int LPR, int VPL, int FMT, int DC, int M1, int M2, int M4, int M8>
static int launch_warp_c(const BprArgs& a, int trial_block, int max_inflight, int num_sms, cudaStream_t s) {
  constexpr int W8 = sizeof(IdT) == 8 ? 1 : 0;
  constexpr int M2w = M2 - W8 > 0 ? M2 - W8 : 1, M4w = M4 - W8 > 0 ? M4 - W8 : 1;
  switch (trial_block == 0 ? DC : trial_block) {
    case 1: return launch_warp<IdT, LPR, VPL, M1, FMT, 1>(a, max_inflight, num_sms, s);
    case 2: return launch_warp<IdT, LPR, VPL, M2w, FMT, 2>(a, max_inflight, num_sms, s);
    case 4: return launch_warp<IdT, LPR, VPL, M4w, FMT, 4>(a, max_inflight, num_sms, s);
    case 8: return launch_warp<IdT, LPR, VPL, M8, FMT, 8>(a, max_inflight, num_sms, s);
    default: return -1002;   // unsupported trial block
  }
}

// Lane geometry of dispatch_bpr (fps_mf_bpr.cu): LPR lanes per row, VPL float4 per lane.  Default trial block 1:
// at k = 64 on one H100 it was the fastest when the first candidate violates and within 1 % of the fastest (C = 2)
// when none does; larger blocks cost occupancy and pull rows a finished group never uses (DESIGN §2.12).
template <typename IdT, int FMT>
static int dispatch_warp(const BprArgs& a, int trial_block, int max_inflight, int num_sms, cudaStream_t s) {
  const int nvec = a.stride >> 2;
  if (nvec <= 1) return launch_warp_c<IdT, 1, 1, FMT, 1, 4, 4, 3, 2>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 2) return launch_warp_c<IdT, 2, 1, FMT, 1, 4, 4, 3, 2>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 4) return launch_warp_c<IdT, 4, 1, FMT, 1, 4, 4, 3, 2>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 8) return launch_warp_c<IdT, 8, 1, FMT, 1, 4, 4, 3, 2>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 16) return launch_warp_c<IdT, 16, 1, FMT, 1, 4, 4, 3, 2>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 32) return launch_warp_c<IdT, 32, 1, FMT, 1, 4, 4, 3, 2>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 64) return launch_warp_c<IdT, 32, 2, FMT, 1, 3, 3, 2, 1>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 96) return launch_warp_c<IdT, 32, 3, FMT, 1, 2, 2, 1, 1>(a, trial_block, max_inflight, num_sms, s);
  if (nvec <= 128) return launch_warp_c<IdT, 32, 4, FMT, 1, 2, 2, 1, 1>(a, trial_block, max_inflight, num_sms, s);
  return -1000;  // rows wider than 512 floats
}

extern "C" int fps_mf_warp_fused(const BprArgs* args, int id_bytes, int trial_block, int max_inflight_rows,
                                 int num_sms, cudaStream_t stream) {
  if (args->n_pos <= 0 || args->n_neg <= 0) return 0;
  if ((args->stride & 3) != 0) return -1000;
  return fps_with_id_form(args->format, id_bytes, [&](auto form) {
    using F = decltype(form);
    return dispatch_warp<typename F::Id, F::fmt>(*args, trial_block, max_inflight_rows, num_sms, stream);
  });
}
