// Pairwise (BPR, Rendle et al. 2009) matrix-factorisation step for sm_90a: pull + SGD + push of one
// (anchor, positive, negative) triple in one kernel, next to the pointwise step of fps_core.cu.
//
// For every positive record (a, i) with rating > 0 and each of its n negatives j:
//   x   = u . (v_i - v_j)                       (u = anchor row, v = candidate rows, all as pulled)
//   g   = lr * sigmoid(-x)
//   u   += g * (v_i - v_j) - lr*reg*u           (REDG.ADD.F32x4)
//   v_i += g * u           - lr*reg*v_i         (push)
//   v_j += -g * u          - lr*reg*v_j         (push)
//   stats[0] += softplus(-x), stats[1] += 1, stats[2] += (x > 0)
// One lane-group handles one positive: u and v_i are pulled once, the n negatives are pulled in turn,
// and the summed u / v_i deltas of the n triples are pushed once.  Every delta is computed from the
// values as pulled (the contract of the fused pointwise kernel), so a batch whose anchors and
// candidates are all distinct gives the same result in any schedule.
//
// Negatives come from an int tensor [n_pos, n] (-1 voids a triple) or are drawn in the kernel from
// the K5 Philox stream of fps_mf_sgd_fused_kernel (key (pos, j, step, seed), uniform over
// [0, num_items), the positive rejected by a shift of 1 + s.z % 7).  The shift is reduced modulo
// num_items - 1 so that it never lands back on the positive, as in every kernel that draws K5.
//
// Rows: the anchor rows and the candidate rows are each read either from a worker-local table
// (slot = id / div) or through a ShardTable (local shard, NVLink peer shard, or a replica); the
// candidate deltas may go to a separate push table (replica staging).  The pointwise learner keeps
// users on the PS and items local, the MF model the other way round; both use this one kernel.
//
// Row-wise AdaGrad (the ADA instantiations, DESIGN §2.10): the same deltas with lr = 1, each row
// stepped by lr / (sqrt(G + |delta|^2 / k) + eps) with G its accumulator as pulled, and G += |delta|^2 / k.
// One kernel body serves both rules: the AdaGrad-only work sits under `if constexpr (ADA)`, and the push of
// the anchor and the positive is written once per rule.
#include "fps_common.cuh"
#include "fps_mf_args.cuh"

// BprArgs, bpr_row and bpr_axpy: fps_mf_args.cuh (shared with the WARP step of fps_mf_warp.cu)

// ADA: row-wise AdaGrad.  Candidate rows are then always read through cand_tab (the host refuses a
// worker-local candidate table), and every lane of a warp computes the squared-norm sums, live or not,
// because fps_group_sum shuffles over the whole warp.
template <typename IdT, int LPR, int VPL, int MINB, int FMT, bool ADA>
__global__ void __launch_bounds__(256, MINB) fps_mf_bpr_kernel(const __grid_constant__ BprArgs a) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int stride = a.stride;
  const int nvec = stride >> 2;
  const float decay = ADA ? a.reg : a.lr * a.reg;   // AdaGrad takes the deltas at learning rate 1
  const float inv_k = 1.f / (float)a.cand_tab.dim;
  const IdT* __restrict__ negs = reinterpret_cast<const IdT*>(a.negatives);
  float loss_acc = 0.f, cnt_acc = 0.f, ok_acc = 0.f;
  bool bad = false;

  // the trip count is the same for every lane of a warp (n_groups is a multiple of 32 / LPR), so the
  // full-warp shuffles of fps_group_sum below always see the whole warp
  const long long n_round = ((a.n_pos + n_groups - 1) / n_groups) * n_groups;
  for (long long pos = group; pos < n_round; pos += n_groups) {
    bool ok = pos < a.n_pos;
    IdT anchor = 0, item = 0;
    if (ok) {
      const FpsRecord<IdT> rec = fps_record<IdT>(FMT, a.users, a.items, a.ratings, pos);
      anchor = rec.user;
      item = rec.item;
      const float rating = rec.rating;
      // rating <= 0 (a pointwise stream's explicit negatives) and voided records are not positives
      ok = rating > 0.f && anchor >= 0 && item >= 0;
    }
    float* up = bpr_row<IdT>(a.anchor_table, a.anchor_div, a.anchor_shift, a.anchor_sharded,
                             a.anchor_tab, anchor, stride);
    float* vip = ADA ? fps_row_t<IdT>(a.cand_tab, item)
                     : bpr_row<IdT>(a.cand_table, a.cand_div, a.cand_shift, a.cand_sharded, a.cand_tab, item, stride);
    float* gup = nullptr;
    float* gip = nullptr;
    if constexpr (ADA) {
      gup = a.anchor_sharded ? fps_row_t<IdT>(a.anchor_acc_tab, anchor)
                             : a.anchor_acc + fps_user_slot<IdT>(anchor, a.anchor_div, a.anchor_shift);
      gip = fps_row_t<IdT>(a.cand_acc, item);
    }
    float4 u[VPL], vi[VPL], du[VPL];
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
      du[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float G_u = 0.f, G_i = 0.f;
    if constexpr (ADA) {   // the accumulators, pulled with the rows
      G_u = ok ? fps_ld_f32(gup) : 0.f;
      G_i = ok ? fps_ld_f32(gip) : 0.f;
    }
    float g_sum = 0.f;
    int n_live = 0;
    for (int j = 0; j < a.n_neg; ++j) {
      long long neg = -1;
      if (ok) {
        if (negs != nullptr) {
          neg = (long long)negs[pos * a.n_neg + j];
        } else if (a.num_items > 1) {   // K5 stream of the pointwise kernel: record pos, negative number j + 1
          neg = fps_k5_negative(a, pos, j + 1, item);
        }
        if (neg == (long long)item) neg = -1;   // an explicit negative equal to the positive is void
      }
      const bool live = neg >= 0;
      const IdT jid = (IdT)(live ? neg : 0);
      float* vjp = ADA ? fps_row_t<IdT>(a.cand_tab, jid)
                       : bpr_row<IdT>(a.cand_table, a.cand_div, a.cand_shift, a.cand_sharded, a.cand_tab, jid, stride);
      float* gjp = ADA ? fps_row_t<IdT>(a.cand_acc, jid) : nullptr;
      float4 vj[VPL];
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        vj[c] = (live && q < nvec) ? fps_ld_row4(vjp + 4 * q) : make_float4(0.f, 0.f, 0.f, 0.f);
        d += u[c].x * (vi[c].x - vj[c].x) + u[c].y * (vi[c].y - vj[c].y) +
             u[c].z * (vi[c].z - vj[c].z) + u[c].w * (vi[c].w - vj[c].w);
      }
      float G_j = 0.f;
      if constexpr (ADA) {
        // G_j is read by lane 0, which issued this row's earlier G += s, and shuffled to the group: a negative
        // repeated in the list then reads G_j + s_j of its earlier triple on every lane (DESIGN §2.10).  A plain
        // load on the other lanes is not ordered after lane 0's reduction.
        G_j = (live && lane == 0) ? fps_ld_f32(gjp) : 0.f;
        G_j = __shfl_sync(0xffffffffu, G_j, 0, LPR);
      }
      const float x = fps_group_sum<LPR>(d);
      float g, s_j = 0.f;
      if constexpr (ADA) {
        g = 1.f / (1.f + __expf(x));   // sigmoid(-x)
        float n2 = 0.f;
#pragma unroll
        for (int c = 0; c < VPL; ++c) {   // delta_j = -g u - reg v_j
          const float4 dj = bpr_axpy(-g, u[c], -decay, vj[c]);
          n2 += dj.x * dj.x + dj.y * dj.y + dj.z * dj.z + dj.w * dj.w;
        }
        s_j = fps_group_sum<LPR>(n2) * inv_k;
      }
      if (!live) continue;
      float step_j = 0.f;
      if constexpr (ADA) {
        step_j = fps_adagrad_scale(a.lr, G_j, s_j);
        if (!(fabsf(g) <= 3.0e38f) || !(fabsf(step_j) <= 3.0e38f)) bad = true;
      } else {
        g = a.lr / (1.f + __expf(x));                // lr * sigmoid(-x)
        if (!(fabsf(g) <= 3.0e38f)) bad = true;      // NaN/Inf guard (Vector.scala:78-80)
      }
      if (lane == 0) {
        loss_acc += fmaxf(-x, 0.f) + log1pf(expf(-fabsf(x)));   // softplus(-x), stable for any |x|
        cnt_acc += 1.f;
        ok_acc += x > 0.f ? 1.f : 0.f;
        if constexpr (ADA) fps_red_add1(gjp, s_j);
      }
      g_sum += g;
      ++n_live;
      float* pj = (!ADA && a.cand_sharded && a.use_push_tab) ? fps_row_t<IdT>(a.push_tab, (IdT)neg) : vjp;
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        if (q < nvec) {
          du[c] = bpr_axpy(g, make_float4(vi[c].x - vj[c].x, vi[c].y - vj[c].y, vi[c].z - vj[c].z,
                                          vi[c].w - vj[c].w), 1.f, du[c]);
          const float4 dj = bpr_axpy(-g, u[c], -decay, vj[c]);
          fps_red_add4(pj + 4 * q, ADA ? make_float4(step_j * dj.x, step_j * dj.y, step_j * dj.z, step_j * dj.w)
                                       : dj);   // the PUSH of v_j
        }
      }
    }
    const float dec = decay * (float)n_live;
    if constexpr (ADA) {
      // the anchor and positive deltas, summed over the live negatives, and their squared norms
      float nu = 0.f, ni = 0.f;
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        du[c] = bpr_axpy(-dec, u[c], 1.f, du[c]);
        vi[c] = bpr_axpy(g_sum, u[c], -dec, vi[c]);
        nu += du[c].x * du[c].x + du[c].y * du[c].y + du[c].z * du[c].z + du[c].w * du[c].w;
        ni += vi[c].x * vi[c].x + vi[c].y * vi[c].y + vi[c].z * vi[c].z + vi[c].w * vi[c].w;
      }
      const float s_u = fps_group_sum<LPR>(nu) * inv_k;
      const float s_i = fps_group_sum<LPR>(ni) * inv_k;
      if (n_live > 0) {
        const float step_u = fps_adagrad_scale(a.lr, G_u, s_u);
        const float step_i = fps_adagrad_scale(a.lr, G_i, s_i);
        if (!(fabsf(step_u) <= 3.0e38f) || !(fabsf(step_i) <= 3.0e38f)) bad = true;
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const int q = lane + c * LPR;
          if (q < nvec) {
            fps_red_add4(up + 4 * q, make_float4(step_u * du[c].x, step_u * du[c].y, step_u * du[c].z,
                                                 step_u * du[c].w));       // anchor update
            fps_red_add4(vip + 4 * q, make_float4(step_i * vi[c].x, step_i * vi[c].y, step_i * vi[c].z,
                                                  step_i * vi[c].w));      // the PUSH of v_i
          }
        }
        if (lane == 0) {
          fps_red_add1(gup, s_u);
          fps_red_add1(gip, s_i);
        }
      }
    } else if (n_live > 0) {
      float* pi = (a.cand_sharded && a.use_push_tab) ? fps_row_t<IdT>(a.push_tab, item) : vip;
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        if (q < nvec) {
          fps_red_add4(up + 4 * q, bpr_axpy(-dec, u[c], 1.f, du[c]));       // anchor update
          fps_red_add4(pi + 4 * q, bpr_axpy(g_sum, u[c], -dec, vi[c]));     // the PUSH of v_i
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);
    cnt_acc += __shfl_xor_sync(0xffffffffu, cnt_acc, o);
    ok_acc += __shfl_xor_sync(0xffffffffu, ok_acc, o);
  }
  if ((threadIdx.x & 31) == 0 && a.stats != nullptr && cnt_acc > 0.f) {
    atomicAdd(a.stats + 0, loss_acc);
    atomicAdd(a.stats + 1, cnt_acc);
    atomicAdd(a.stats + 2, ok_acc);
  }
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
}

// Static pull limiter: a lane-group has up to 3 rows in flight (u, v_i, v_j), so the grid is capped at
// max_inflight_rows / (3 * lane-groups per CTA).  `reserve_total` CTA slots stay free for the replica
// exchange that runs next to the step (as in launch_mf of fps_core.cu).
template <typename IdT, int LPR, int VPL, int MINB, int FMT, bool ADA>
static int launch_bpr(const BprArgs& a, int max_inflight_rows, int num_sms, cudaStream_t stream) {
  const int threads = 256;
  auto kern = fps_mf_bpr_kernel<IdT, LPR, VPL, MINB, FMT, ADA>;
  const long long blocks = fps_row_grid(kern, threads, threads / LPR, num_sms, a.reserve_total, max_inflight_rows, 3,
                                        a.n_pos, 1);
  kern<<<(int)blocks, threads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// Lane geometry of dispatch_mf (fps_core.cu): LPR lanes per row, VPL float4 per lane.  MINB is chosen for 0
// spills (ptxas -v); row-wise AdaGrad needs more registers on the 32- and 64-float4 rungs.
template <typename IdT, int FMT, bool ADA>
static int dispatch_bpr(const BprArgs& a, int max_inflight, int num_sms, cudaStream_t s) {
  if (ADA && (!a.cand_sharded || a.use_push_tab)) return -1009;
  const int nvec = a.stride >> 2;
  if (nvec <= 1) return launch_bpr<IdT, 1, 1, ADA ? 3 : 4, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 2) return launch_bpr<IdT, 2, 1, ADA ? 3 : 4, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 4) return launch_bpr<IdT, 4, 1, ADA ? 3 : 4, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 8) return launch_bpr<IdT, 8, 1, ADA ? 3 : 4, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 16) return launch_bpr<IdT, 16, 1, ADA ? 3 : 4, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 32) return launch_bpr<IdT, 32, 1, ADA ? 3 : 4, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 64) return launch_bpr<IdT, 32, 2, ADA ? 2 : 3, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 96) return launch_bpr<IdT, 32, 3, 2, FMT, ADA>(a, max_inflight, num_sms, s);
  if (nvec <= 128) return launch_bpr<IdT, 32, 4, 2, FMT, ADA>(a, max_inflight, num_sms, s);
  return -1000;  // rows wider than 512 floats
}

extern "C" int fps_mf_bpr_fused(const BprArgs* args, int id_bytes, int max_inflight_rows, int num_sms,
                                cudaStream_t stream) {
  if (args->n_pos <= 0 || args->n_neg <= 0) return 0;
  if ((args->stride & 3) != 0) return -1000;
  return fps_with_id_form(args->format, id_bytes, [&](auto form) {
    using F = decltype(form);
    if (args->cand_acc.base[0] != nullptr)   // row-wise AdaGrad
      return dispatch_bpr<typename F::Id, F::fmt, true>(*args, max_inflight_rows, num_sms, stream);
    return dispatch_bpr<typename F::Id, F::fmt, false>(*args, max_inflight_rows, num_sms, stream);
  });
}
