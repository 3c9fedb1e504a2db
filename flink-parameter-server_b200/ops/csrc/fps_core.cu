// Core parameter-server kernels for sm_90a: lazy-init materialisation (K4), fused
// pull + SGD + push for matrix factorisation (K1+K3+K2), standalone pull gather (K1),
// push accumulate (K2) and pull-fused-with-dot scoring.  All "communication" is done by
// the kernels themselves through peer-mapped shard pointers (NVLink/NVSwitch one-sided
// loads and REDG.ADD.F32x4 reductions); no NCCL call sits on these paths.
//
// Reference behaviour being reproduced (not code): SimplePSLogic.scala:13-25 (init on
// first pull, additive update), SGDUpdater.scala:5-14 (delta rule),
// PSOnlineMatrixFactorizationWorker.scala:42-89 (worker step + negative sampling).
#include "fps_common.cuh"
#include "fps_mf_args.cuh"

// ----------------------------------------------------------------------------------------
// K4: materialise rows as a pure function of (seed, id, column).
//   value(id, j) = lo + (hi - lo) * u01(philox(id_lo, id_hi, j / 4, 0; seed_lo, seed_hi)[j % 4])
// "init on first pull" (RangedRandomFactorInitializer.scala:7-9, PseudoRandomFactorInitializer
// .scala:9-12) becomes "every slot already holds what init(id) would return".
// ----------------------------------------------------------------------------------------
__global__ void fps_init_rows_kernel(float* __restrict__ rows, long long n_rows, int dim,
                                     int stride, int shard, int num_shards, int mode,
                                     long long div, unsigned long long seed, float lo,
                                     float hi) {
  const int nvec = stride >> 2;
  const long long total = n_rows * nvec;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const long long slot = t / nvec;
    const int q = (int)(t - slot * nvec);
    const long long id = (mode == FPS_PART_HASH) ? slot * num_shards + shard
                                                 : (long long)shard * div + slot;
    Philox4 r = fps_philox((uint32_t)id, (uint32_t)((unsigned long long)id >> 32), (uint32_t)q,
                           0u, (uint32_t)seed, (uint32_t)(seed >> 32));
    float4 v;
    const float sc = hi - lo;
    v.x = (4 * q + 0 < dim) ? lo + sc * fps_u01(r.x) : 0.f;
    v.y = (4 * q + 1 < dim) ? lo + sc * fps_u01(r.y) : 0.f;
    v.z = (4 * q + 2 < dim) ? lo + sc * fps_u01(r.z) : 0.f;
    v.w = (4 * q + 3 < dim) ? lo + sc * fps_u01(r.w) : 0.f;
    *reinterpret_cast<float4*>(rows + slot * (long long)stride + 4 * q) = v;
  }
}

extern "C" int fps_init_rows(float* rows, long long n_rows, int dim, int stride, int shard,
                             int num_shards, int mode, long long div, unsigned long long seed,
                             float lo, float hi, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  long long total = n_rows * (stride / 4);
  int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > 132 * 32) blocks = 132 * 32;  // 32 CTAs per H100 SM, grid-stride beyond
  fps_init_rows_kernel<<<(int)blocks, threads, 0, stream>>>(rows, n_rows, dim, stride, shard,
                                                            num_shards, mode, div, seed, lo, hi);
  return (int)cudaGetLastError();
}

// Device-side pull limiter (WL:196-250 as a credit counter): `credits[0]` holds the number of pulls that
// may still be issued; a lane-group takes one credit before it touches the owner's memory and returns
// it when the answer has been consumed (stored), so at most `pullLimit` row pulls are un-answered at any
// time whatever the grid size.  `credits[1]` counts the stalls (acquisitions that had to wait).
__device__ __forceinline__ void fps_credit_acquire(int* credits, int n = 1) {
  bool stalled = false;
  unsigned ns = 256;
  while (true) {
    // compare-and-swap on a positive value only: the counter never goes negative, so waiters cannot hold it
    // down (a sub-then-add-back scheme livelocks once thousands of lane-groups retry at the same time);
    // waiters poll with a plain load and back off exponentially
    const int cur = *reinterpret_cast<volatile int*>(credits);
    if (cur >= n && atomicCAS(credits, cur, cur - n) == cur) break;
    if (cur < n) {
      stalled = true;
      __nanosleep(ns);
      if (ns < 8192) ns <<= 1;
    }
  }
  if (stalled) atomicAdd(credits + 1, 1);
}

// ----------------------------------------------------------------------------------------
// K1+K3+K2: fused matrix-factorisation step.
//   for each (user, item, rating):          [+ neg_rate sampled (user, item', 0)]
//     v  = pull(item)      -- 16-byte loads from the owning shard (local HBM or NVLink peer)
//     u  = user row (worker-local HBM)
//     e  = err_mode==0 ? sigmoid(r - u.v) : (r - u.v)     (SGDUpdater.scala:8)
//     u += lr*e*v          -- local REDG.ADD.F32x4 (no lost updates inside a micro-batch)
//     push(item, lr*e*u)   -- REDG.ADD.F32x4 to the owner == paramUpdate(vectorSum) applied
//                              by the owner's memory system
// LPR lanes cooperate on one row (each lane owns VPL float4 chunks); each lane-group keeps R
// ratings in flight so the peer-load latency (~2 us over NVSwitch) is covered by ILP.
// The pull limiter (WL:196-250) is the number of row slots in flight: grid * 256 / LPR * R,
// chosen by the host from pullLimit (credits pre-distributed to resident lane-groups).
// ----------------------------------------------------------------------------------------

// ADA = 1: row-wise AdaGrad (DESIGN §2.10).  e is taken with learning rate 1, each row's step is
//   s = |delta|^2 / k,  row += lr * delta / (sqrt(G + s) + eps),  G += s
// with G the row's accumulator as pulled next to the row.  ADA = 0 is the SGD step, unchanged.  AdaGrad runs
// only the default register-staged geometries (no L2 hints, output stream or credit counter; a pull limit is the
// static capped grid).
template <typename IdT, int LPR, int VPL, int R, int FMT, int HINT, int EMIT, int LIMIT, int ADA>
__device__ __forceinline__ void fps_mf_step_body(const MfArgs& a) {
  unsigned long long pol_user = 0, pol_item = 0;
  if (HINT) {
    pol_user = fps_policy_evict_first();
    pol_item = fps_policy_evict_last();
  }
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int per_pos = 1 + a.neg_rate;
  const long long n_eff = a.n_pos * per_pos;
  const int stride = a.item_tab.stride;
  const int nvec = stride >> 2;
  // the id arrays are read through these (packed records through a.users): with the record pointers taken from
  // `a` at the decode, nvcc orders this kernel's argument loads differently
  const IdT* __restrict__ users = reinterpret_cast<const IdT*>(a.users);
  const IdT* __restrict__ items = reinterpret_cast<const IdT*>(a.items);
  float sq_acc = 0.f, cnt_acc = 0.f;
  bool bad = false;

  for (long long base = 0; base < n_eff; base += n_groups * R) {
    if (a.progress != nullptr && blockIdx.x == 0 && threadIdx.x == 0)
      *reinterpret_cast<volatile unsigned int*>(a.progress) = (unsigned int)base;
    float4 u[R][VPL], v[R][VPL];
    float* up[R];
    float* vp[R];
    float* pp[R];
    float rt[R];
    bool ok[R];
    long long uid[R];
    int ncred[R];
    float* gup[R];
    float* gvp[R];
    float gu[R], gv[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const long long idx = base + (long long)r * n_groups + group;
      ok[r] = idx < n_eff;
      long long pos = idx;
      int j = 0;
      if (per_pos > 1) {
        pos = idx / per_pos;
        j = (int)(idx - pos * per_pos);
      }
      IdT user = 0, item = 0;
      rt[r] = 0.f;
      if (ok[r]) {
        const FpsRecord<IdT> rec = fps_record<IdT>(FMT, FMT == 1 ? a.users : users, items, a.ratings, pos);
        user = rec.user;
        item = rec.item;
        const float rating = rec.rating;
        if (FMT == 0 && user < 0) ok[r] = false;  // record voided upstream (fps_neg_sample: no unseen item found)
        // j > 0: the K5 negative (the host requires num_items >= 2)
        if (j == 0) rt[r] = rating;
        else item = (IdT)fps_k5_negative(a, pos, j, item);
      }
      uid[r] = (long long)user;
      if (LIMIT) {
        // One credit per pull, taken for the whole warp at once (all or nothing): the lane-groups of a warp
        // meet again in the full-warp shuffles below, so a group must never hold a credit while a
        // warp-mate waits for one.  Returned once the pushes are issued.
        ncred[r] = __popc(__ballot_sync(0xffffffffu, ok[r] && lane == 0));
        if ((threadIdx.x & 31) == 0 && ncred[r] > 0) fps_credit_acquire(a.credits, ncred[r]);
        __syncwarp();
      }
      up[r] = a.user_sharded ? fps_row_t<IdT>(a.user_tab, user)
                             : a.user_table + fps_user_slot<IdT>(user, a.user_div, a.user_shift) * (size_t)stride;
      vp[r] = fps_row_t<IdT>(a.item_tab, item);
      pp[r] = a.use_push_tab ? fps_row_t<IdT>(a.push_tab, item) : vp[r];
      if (ADA) {   // the two accumulators, pulled with the rows
        gup[r] = a.user_sharded ? fps_row_t<IdT>(a.user_acc_tab, user)
                                : a.user_acc + fps_user_slot<IdT>(user, a.user_div, a.user_shift);
        gvp[r] = fps_row_t<IdT>(a.item_acc, item);
        gu[r] = ok[r] ? fps_ld_f32(gup[r]) : 0.f;
        gv[r] = ok[r] ? fps_ld_f32(gvp[r]) : 0.f;
      }
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        if (ok[r] && q < nvec) {
          if (HINT) {
            v[r][c] = fps_ld_row4_hint(vp[r] + 4 * q, pol_item);  // the PULL
            u[r][c] = fps_ld_row4_hint(up[r] + 4 * q, pol_user);
          } else {
            v[r][c] = fps_ld_row4(vp[r] + 4 * q);  // the PULL
            u[r][c] = *reinterpret_cast<const float4*>(up[r] + 4 * q);
          }
        } else {
          v[r][c] = make_float4(0.f, 0.f, 0.f, 0.f);
          u[r][c] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float d = 0.f, nu = 0.f, nv = 0.f;
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        d += fps_mf_dot4(u[r][c], v[r][c]);
        if (ADA) {
          nu += fps_mf_dot4(u[r][c], u[r][c]);
          nv += fps_mf_dot4(v[r][c], v[r][c]);
        }
      }
      d = fps_group_sum<LPR>(d);
      const float resid = rt[r] - d;
      const float g = fps_mf_grad(a.err_mode, ADA ? 1.f : a.lr, rt[r], d, resid);
      float g_u = g, g_v = g, s_u = 0.f, s_v = 0.f;   // SGD: both rows step by lr * e
      if (ADA) {   // delta_u = e v, delta_v = e u
        nu = fps_group_sum<LPR>(nu);
        nv = fps_group_sum<LPR>(nv);
        const float ee = g * g / (float)a.item_tab.dim;
        s_u = ee * nv;
        s_v = ee * nu;
        g_u = g * fps_adagrad_scale(a.lr, gu[r], s_u);
        g_v = g * fps_adagrad_scale(a.lr, gv[r], s_v);
      }
      if (LIMIT) {
        __syncwarp();                               // every lane holds its part of the answer
        if ((threadIdx.x & 31) == 0 && ncred[r] > 0) atomicAdd(a.credits, ncred[r]);
      }
      if (ok[r]) {
        if (!(fabsf(g) <= 3.0e38f)) bad = true;  // NaN/Inf guard (Vector.scala:78-80)
        if (ADA && !(fabsf(g_u) <= 3.0e38f && fabsf(g_v) <= 3.0e38f)) bad = true;
        if (lane == 0) {
          sq_acc += resid * resid;
          cnt_acc += 1.f;
          if (ADA) {
            fps_red_add1(gup[r], s_u);
            fps_red_add1(gvp[r], s_v);
          }
        }
        long long out_slot = -1;
        if (EMIT) {   // E5: this update's view of the new user vector goes to the output staging area
          const long long idx = base + (long long)r * n_groups + group;
          if (idx % a.out_every == 0) {
            out_slot = (long long)*a.out_staged + idx / a.out_every;
            if (out_slot >= a.out_cap) out_slot = -1;
            else if (lane == 0) a.out_ids[out_slot] = uid[r];
          }
        }
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const int q = lane + c * LPR;
          if (q < nvec) {
            float4 du = make_float4(g_u * v[r][c].x, g_u * v[r][c].y, g_u * v[r][c].z, g_u * v[r][c].w);
            float4 dv = make_float4(g_v * u[r][c].x, g_v * u[r][c].y, g_v * u[r][c].z, g_v * u[r][c].w);
            if (EMIT && out_slot >= 0)
              *reinterpret_cast<float4*>(a.out_vecs + out_slot * (long long)stride + 4 * q) =
                  make_float4(u[r][c].x + du.x, u[r][c].y + du.y, u[r][c].z + du.z, u[r][c].w + du.w);
            if (HINT) {
              fps_red_add4_hint(up[r] + 4 * q, du, pol_user);
              fps_red_add4_hint(pp[r] + 4 * q, dv, pol_item);
            } else {
              fps_red_add4(up[r] + 4 * q, du);   // worker-local user update
              fps_red_add4(pp[r] + 4 * q, dv);   // the PUSH, fused with paramUpdate
            }
          }
        }
      }
    }
  }
  // statistics: one atomic pair per warp
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sq_acc += __shfl_xor_sync(0xffffffffu, sq_acc, o);
    cnt_acc += __shfl_xor_sync(0xffffffffu, cnt_acc, o);
  }
  if ((threadIdx.x & 31) == 0 && a.stats != nullptr && cnt_acc > 0.f) {
    atomicAdd(a.stats + 0, sq_acc);
    atomicAdd(a.stats + 1, cnt_acc);
  }
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
}

// The step is a function the kernel calls, not the kernel's own body: written out in the kernel, it compiles to
// other register assignments in some 64-bit-id instantiations.
template <typename IdT, int LPR, int VPL, int R, int MINB, int FMT, int HINT = 0, int EMIT = 0, int LIMIT = 0,
          int ADA = 0>
__global__ void __launch_bounds__(256, MINB)
    fps_mf_sgd_fused_kernel(const __grid_constant__ MfArgs a) {
  fps_mf_step_body<IdT, LPR, VPL, R, FMT, HINT, EMIT, LIMIT, ADA>(a);
}

// A lane-group keeps R records, and so R row pairs, in flight.
template <typename IdT, int LPR, int VPL, int R, int MINB, int FMT, int HINT = 0, int EMIT = 0, int LIMIT = 0,
          int ADA = 0>
static int launch_mf(const MfArgs& a, int max_inflight_rows, int num_sms, cudaStream_t stream) {
  const int threads = 256;
  auto kern = fps_mf_sgd_fused_kernel<IdT, LPR, VPL, R, MINB, FMT, HINT, EMIT, LIMIT, ADA>;
  const long long blocks = fps_row_grid(kern, threads, threads / LPR, num_sms, a.reserve_total, max_inflight_rows, R,
                                        a.n_pos * (1 + a.neg_rate), R);
  kern<<<(int)blocks, threads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

static int g_mf_reg_variant = 0;  // tuning knob: (rows in flight per lane-group, min blocks/SM)
extern "C" void fps_set_mf_reg_variant(int v) { g_mf_reg_variant = v; }

// Defaults come from the measured sweep in profiles/mf_fused_history.md: for 16-byte-per-lane rows
// one row in flight per lane-group at full occupancy (8 CTAs/SM, 32 registers) wins on local HBM.
template <typename IdT, int FMT>
static int dispatch_mf(const MfArgs& a, int max_inflight, int num_sms, cudaStream_t s) {
  const int nvec = a.item_tab.stride >> 2;
  const int v = g_mf_reg_variant;
  if (a.item_acc.base[0] != nullptr) {   // row-wise AdaGrad: the default geometries, 0 spills (ptxas -v)
    if (a.credits != nullptr || a.out_every > 0 || a.use_push_tab) return -1009;
    if (nvec <= 1) return launch_mf<IdT, 1, 1, 2, 4, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 2) return launch_mf<IdT, 2, 1, 2, 4, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 4) return launch_mf<IdT, 4, 1, 2, 4, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 8) return launch_mf<IdT, 8, 1, 1, 6, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 16) return launch_mf<IdT, 16, 1, 1, 6, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 32) return launch_mf<IdT, 32, 1, 1, 6, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 64) return launch_mf<IdT, 32, 2, 1, 4, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 96) return launch_mf<IdT, 32, 3, 1, 4, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 128) return launch_mf<IdT, 32, 4, 1, 2, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 256) return launch_mf<IdT, 32, 8, 1, 2, FMT, 0, 0, 0, 1>(a, max_inflight, num_sms, s);
    return -1000;
  }
  if (a.credits != nullptr) {   // device credit-counter pull limiter: the counter bounds the pulls in flight;
    const int cap = 2 * max_inflight;  // the grid is trimmed to ~2x the credits (fewer contenders on the counter)
    if (nvec <= 4) return launch_mf<IdT, 4, 1, 1, 4, FMT, 0, 0, 1>(a, cap, num_sms, s);
    if (nvec <= 8) return launch_mf<IdT, 8, 1, 1, 4, FMT, 0, 0, 1>(a, cap, num_sms, s);
    if (nvec <= 16) return launch_mf<IdT, 16, 1, 1, 4, FMT, 0, 0, 1>(a, cap, num_sms, s);
    if (nvec <= 32) return launch_mf<IdT, 32, 1, 1, 4, FMT, 0, 0, 1>(a, cap, num_sms, s);
    if (nvec <= 128) return launch_mf<IdT, 32, 4, 1, 2, FMT, 0, 0, 1>(a, cap, num_sms, s);
    return -1000;
  }
  if (a.out_every > 0) {   // with the E5 output stream (one row in flight per lane-group, 4 CTAs/SM)
    if (a.out_ids == nullptr || a.out_vecs == nullptr || a.out_staged == nullptr) return -1002;
    if (nvec <= 4) return launch_mf<IdT, 4, 1, 1, 4, FMT, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 8) return launch_mf<IdT, 8, 1, 1, 4, FMT, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 16) return launch_mf<IdT, 16, 1, 1, 4, FMT, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 32) return launch_mf<IdT, 32, 1, 1, 4, FMT, 0, 1>(a, max_inflight, num_sms, s);
    if (nvec <= 128) return launch_mf<IdT, 32, 4, 1, 2, FMT, 0, 1>(a, max_inflight, num_sms, s);
    return -1000;
  }
  if (nvec <= 1) return launch_mf<IdT, 1, 1, 2, 4, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 2) return launch_mf<IdT, 2, 1, 2, 4, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 4) return launch_mf<IdT, 4, 1, 2, 4, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 8) return launch_mf<IdT, 8, 1, 1, 8, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 16) {
    if (a.l2_hints) return launch_mf<IdT, 16, 1, 1, 8, FMT, 1>(a, max_inflight, num_sms, s);
    switch (v) {
      case 1: return launch_mf<IdT, 16, 1, 4, 3, FMT>(a, max_inflight, num_sms, s);
      case 3: return launch_mf<IdT, 16, 1, 2, 4, FMT>(a, max_inflight, num_sms, s);
      case 5: return launch_mf<IdT, 16, 1, 2, 5, FMT>(a, max_inflight, num_sms, s);
      case 9: return launch_mf<IdT, 8, 2, 2, 4, FMT>(a, max_inflight, num_sms, s);
      default: return launch_mf<IdT, 16, 1, 1, 8, FMT>(a, max_inflight, num_sms, s);
    }
  }
  if (nvec <= 32) return launch_mf<IdT, 32, 1, 1, 8, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 64) return launch_mf<IdT, 32, 2, 1, 4, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 96) return launch_mf<IdT, 32, 3, 1, 4, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 128) return launch_mf<IdT, 32, 4, 1, 2, FMT>(a, max_inflight, num_sms, s);
  if (nvec <= 256) return launch_mf<IdT, 32, 8, 1, 2, FMT>(a, max_inflight, num_sms, s);
  return -1000;  // dim > 1024 not supported by the fused MF kernel
}

extern "C" int fps_mf_sgd_fused(const MfArgs* args, int id_bytes, int max_inflight_rows,
                                int num_sms, cudaStream_t stream) {
  if (args->n_pos <= 0) return 0;
  return fps_with_id_form(args->format, id_bytes, [&](auto form) {
    using F = decltype(form);
    return dispatch_mf<typename F::Id, F::fmt>(*args, max_inflight_rows, num_sms, stream);
  });
}

// ----------------------------------------------------------------------------------------
// K1 standalone: out[i, :] = table[ids[i], :]   (pull for the generic tensor tier)
// K2 standalone: table[ids[i], :] += delta[i, :] (push fused with additive paramUpdate)
// pull_dot:      score[i] = table[ids[i], :] . local[i, :]   (pull fused with the consumer)
// One lane-group of LPR lanes per row, VPL chunks per lane, generic in dim via nvec bound.
// ----------------------------------------------------------------------------------------
template <typename IdT, int LPR>
__global__ void __launch_bounds__(256)
    fps_pull_gather_kernel(const __grid_constant__ ShardTable t, const IdT* __restrict__ ids,
                           long long n, float* __restrict__ out, int out_stride, int touch,
                           int* __restrict__ credits) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int nvec = t.stride >> 2;
  const unsigned gmask = LPR == 32 ? 0xffffffffu : (((1u << LPR) - 1u) << ((threadIdx.x & 31) & ~(LPR - 1)));
  for (long long i = group; i < n; i += n_groups) {
    const long long id = (long long)ids[i];
    const float* src = fps_row_t<IdT>(t, ids[i]);
    if (touch && lane == 0) fps_touch(t, id);
    if (credits != nullptr) {
      if (lane == 0) fps_credit_acquire(credits);
      __syncwarp(gmask);
    }
    for (int q = lane; q < nvec; q += LPR) {
      float4 v = fps_ld_row4(src + 4 * q);
      float* o = out + i * (long long)out_stride + 4 * q;
      if ((out_stride & 3) == 0 && 4 * q + 3 < out_stride) {
        *reinterpret_cast<float4*>(o) = v;
      } else {
        if (4 * q + 0 < out_stride) o[0] = v.x;
        if (4 * q + 1 < out_stride) o[1] = v.y;
        if (4 * q + 2 < out_stride) o[2] = v.z;
        if (4 * q + 3 < out_stride) o[3] = v.w;
      }
    }
    if (credits != nullptr) {
      __syncwarp(gmask);                       // the answer has been consumed by every lane
      if (lane == 0) atomicAdd(credits, 1);    // release the credit
    }
  }
}

template <typename IdT, int LPR>
__global__ void __launch_bounds__(256)
    fps_push_add_kernel(const __grid_constant__ ShardTable t, const IdT* __restrict__ ids,
                        long long n, const float* __restrict__ delta, int delta_stride, float scale,
                        int touch, int* nan_flag) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int nvec = t.stride >> 2;
  bool bad = false;
  for (long long i = group; i < n; i += n_groups) {
    const long long id = (long long)ids[i];
    float* dst = fps_row_t<IdT>(t, ids[i]);
    if (touch && lane == 0) fps_touch(t, id);
    for (int q = lane; q < nvec; q += LPR) {
      const float* d = delta + i * (long long)delta_stride + 4 * q;
      float4 v;
      if (4 * q + 3 < delta_stride && (delta_stride & 3) == 0) {
        v = *reinterpret_cast<const float4*>(d);
      } else {
        v.x = (4 * q + 0 < delta_stride) ? d[0] : 0.f;
        v.y = (4 * q + 1 < delta_stride) ? d[1] : 0.f;
        v.z = (4 * q + 2 < delta_stride) ? d[2] : 0.f;
        v.w = (4 * q + 3 < delta_stride) ? d[3] : 0.f;
      }
      v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
      if (!(fabsf(v.x) <= 3.0e38f) || !(fabsf(v.y) <= 3.0e38f) || !(fabsf(v.z) <= 3.0e38f) ||
          !(fabsf(v.w) <= 3.0e38f))
        bad = true;
      fps_red_add4(dst + 4 * q, v);
    }
  }
  if (bad && nan_flag != nullptr) *nan_flag = 1;
}

// Model load (transformWithModelLoad, FPS:715-908): table[ids[i], :] = values[i, :] (one-sided store).
template <typename IdT, int LPR>
__global__ void __launch_bounds__(256)
    fps_push_assign_kernel(const __grid_constant__ ShardTable t, const IdT* __restrict__ ids,
                           long long n, const float* __restrict__ vals, int val_stride, int touch) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int nvec = t.stride >> 2;
  for (long long i = group; i < n; i += n_groups) {
    float* dst = fps_row_t<IdT>(t, ids[i]);
    if (touch && lane == 0) fps_touch(t, (long long)ids[i]);
    for (int q = lane; q < nvec; q += LPR) {
      const float* d = vals + i * (long long)val_stride + 4 * q;
      float4 v;
      v.x = (4 * q + 0 < val_stride) ? d[0] : 0.f;
      v.y = (4 * q + 1 < val_stride) ? d[1] : 0.f;
      v.z = (4 * q + 2 < val_stride) ? d[2] : 0.f;
      v.w = (4 * q + 3 < val_stride) ? d[3] : 0.f;
      *reinterpret_cast<float4*>(dst + 4 * q) = v;
    }
  }
}

template <typename IdT, int LPR>
__global__ void __launch_bounds__(256)
    fps_pull_dot_kernel(const __grid_constant__ ShardTable t, const IdT* __restrict__ ids,
                        long long n, const float* __restrict__ local, int local_stride,
                        float* __restrict__ score) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int nvec = t.stride >> 2;
  const long long n_round = ((n + n_groups - 1) / n_groups) * n_groups;
  for (long long i = group; i < n_round; i += n_groups) {
    float d = 0.f;
    if (i < n) {
      const float* src = fps_row_t<IdT>(t, ids[i]);
      for (int q = lane; q < nvec; q += LPR) {
        float4 v = fps_ld_row4(src + 4 * q);
        const float* l = local + i * (long long)local_stride + 4 * q;
        float4 w;
        w.x = (4 * q + 0 < local_stride) ? l[0] : 0.f;
        w.y = (4 * q + 1 < local_stride) ? l[1] : 0.f;
        w.z = (4 * q + 2 < local_stride) ? l[2] : 0.f;
        w.w = (4 * q + 3 < local_stride) ? l[3] : 0.f;
        d += v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
      }
    }
    d = fps_group_sum<LPR>(d);
    if (i < n && lane == 0) score[i] = d;
  }
}

// Wide rows (dim > 1024 floats, e.g. the 16K..1M-float vectors of the bandwidth sweep): one lane-group
// per row would leave the GPU idle, so the work item is (row, 4 KiB segment) and every lane keeps
// 8 independent 16-byte transfers in flight.  OP 0: pull (peer -> out), 1: push-add, 2: assign.
#define FPS_WIDE_SEG_VEC 256   // float4 per segment
template <typename IdT, int OP>
__global__ void __launch_bounds__(256)
    fps_wide_rows_kernel(const __grid_constant__ ShardTable t, const IdT* __restrict__ ids, long long n,
                         float* __restrict__ buf, int buf_stride, float scale) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int nvec = t.stride >> 2;
  const int n_seg = (nvec + FPS_WIDE_SEG_VEC - 1) / FPS_WIDE_SEG_VEC;
  const long long total = n * n_seg;
  for (long long w = warp; w < total; w += n_warps) {
    const long long i = w / n_seg;
    const int seg = (int)(w - i * n_seg);
    float* row = fps_row_t<IdT>(t, ids[i]);
    float* b = buf + i * (long long)buf_stride;
    float4 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int q = seg * FPS_WIDE_SEG_VEC + k * 32 + lane;
      if (q < nvec && 4 * q + 3 < buf_stride) {
        v[k] = (OP == 0) ? fps_ld_row4(row + 4 * q) : *reinterpret_cast<const float4*>(b + 4 * q);
      } else {
        v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int q = seg * FPS_WIDE_SEG_VEC + k * 32 + lane;
      if (q < nvec && 4 * q + 3 < buf_stride) {
        if (OP == 0) {
          *reinterpret_cast<float4*>(b + 4 * q) = v[k];
        } else if (OP == 1) {
          fps_red_add4(row + 4 * q, make_float4(v[k].x * scale, v[k].y * scale, v[k].z * scale, v[k].w * scale));
        } else {
          *reinterpret_cast<float4*>(row + 4 * q) = v[k];
        }
      }
    }
  }
}

template <int OP>
static int launch_wide(const ShardTable* t, const void* ids, int id_bytes, long long n, float* buf,
                       int buf_stride, float scale, int num_sms, cudaStream_t stream) {
  const int nvec = t->stride >> 2;
  const long long total = n * ((nvec + FPS_WIDE_SEG_VEC - 1) / FPS_WIDE_SEG_VEC);
  long long blocks = (total + 7) / 8;
  if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
  if (blocks < 1) blocks = 1;
  if (id_bytes == 4)
    fps_wide_rows_kernel<int, OP><<<(int)blocks, 256, 0, stream>>>(*t, (const int*)ids, n, buf, buf_stride, scale);
  else
    fps_wide_rows_kernel<long long, OP><<<(int)blocks, 256, 0, stream>>>(*t, (const long long*)ids, n, buf, buf_stride, scale);
  return (int)cudaGetLastError();
}
static inline bool use_wide(const ShardTable* t, int buf_stride, int touch) {
  return (t->stride >> 2) > 256 && (buf_stride & 3) == 0 && buf_stride == t->stride && !touch;
}

static inline int pick_lpr(int nvec) {
  int l = 1;
  while (l < nvec && l < 32) l <<= 1;
  return l;
}
static inline int row_grid(long long n, int lpr, int num_sms) {
  long long groups_per_block = 256 / lpr;
  long long blocks = (n + groups_per_block - 1) / groups_per_block;
  long long cap = (long long)num_sms * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

#define FPS_DISPATCH_LPR(KERNEL, IDT, LPRV, GRID, STREAM, ...)                               \
  switch (LPRV) {                                                                            \
    case 1: KERNEL<IDT, 1><<<GRID, 256, 0, STREAM>>>(__VA_ARGS__); break;                    \
    case 2: KERNEL<IDT, 2><<<GRID, 256, 0, STREAM>>>(__VA_ARGS__); break;                    \
    case 4: KERNEL<IDT, 4><<<GRID, 256, 0, STREAM>>>(__VA_ARGS__); break;                    \
    case 8: KERNEL<IDT, 8><<<GRID, 256, 0, STREAM>>>(__VA_ARGS__); break;                    \
    case 16: KERNEL<IDT, 16><<<GRID, 256, 0, STREAM>>>(__VA_ARGS__); break;                  \
    default: KERNEL<IDT, 32><<<GRID, 256, 0, STREAM>>>(__VA_ARGS__); break;                  \
  }

// max_inflight_rows > 0 is the device-side pull limiter (WL:196-250) of the generic tier: the grid is
// capped so that at most that many row pulls are in flight (one per resident lane-group).
static inline int limit_grid(int grid, int lpr, int max_inflight_rows) {
  if (max_inflight_rows <= 0) return grid;
  int cap = max_inflight_rows / (256 / lpr);
  if (cap < 1) cap = 1;
  return grid < cap ? grid : cap;
}

// credits != nullptr: device credit counter (credits[0] must hold pullLimit, credits[1] counts stalls);
// otherwise max_inflight_rows > 0 caps the grid (static variant of the limiter).
extern "C" int fps_pull_gather(const ShardTable* t, const void* ids, int id_bytes, long long n,
                               float* out, int out_stride, int touch, int num_sms,
                               int max_inflight_rows, int* credits, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (use_wide(t, out_stride, touch) && max_inflight_rows <= 0 && credits == nullptr)
    return launch_wide<0>(t, ids, id_bytes, n, out, out_stride, 1.f, num_sms, stream);
  const int lpr = pick_lpr(t->stride >> 2);
  int grid = row_grid(n, lpr, num_sms);
  // static limiter: the grid IS the bound.  Credit counter: the counter is the bound; the grid is only
  // trimmed to ~2x the credits so that thousands of lane-groups do not fight over a handful of credits
  grid = limit_grid(grid, lpr, credits == nullptr ? max_inflight_rows : 2 * max_inflight_rows);
  if (id_bytes == 4) {
    FPS_DISPATCH_LPR(fps_pull_gather_kernel, int, lpr, grid, stream, *t, (const int*)ids, n, out,
                     out_stride, touch, credits)
  } else {
    FPS_DISPATCH_LPR(fps_pull_gather_kernel, long long, lpr, grid, stream, *t,
                     (const long long*)ids, n, out, out_stride, touch, credits)
  }
  return (int)cudaGetLastError();
}

extern "C" int fps_push_add(const ShardTable* t, const void* ids, int id_bytes, long long n,
                            const float* delta, int delta_stride, float scale, int touch,
                            int* nan_flag, int num_sms, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (use_wide(t, delta_stride, touch))  // wide rows: no per-element NaN scan (bandwidth path)
    return launch_wide<1>(t, ids, id_bytes, n, const_cast<float*>(delta), delta_stride, scale, num_sms, stream);
  const int lpr = pick_lpr(t->stride >> 2);
  const int grid = row_grid(n, lpr, num_sms);
  if (id_bytes == 4) {
    FPS_DISPATCH_LPR(fps_push_add_kernel, int, lpr, grid, stream, *t, (const int*)ids, n, delta,
                     delta_stride, scale, touch, nan_flag)
  } else {
    FPS_DISPATCH_LPR(fps_push_add_kernel, long long, lpr, grid, stream, *t, (const long long*)ids,
                     n, delta, delta_stride, scale, touch, nan_flag)
  }
  return (int)cudaGetLastError();
}

extern "C" int fps_pull_dot(const ShardTable* t, const void* ids, int id_bytes, long long n,
                            const float* local, int local_stride, float* score, int num_sms,
                            cudaStream_t stream) {
  if (n <= 0) return 0;
  const int lpr = pick_lpr(t->stride >> 2);
  const int grid = row_grid(n, lpr, num_sms);
  if (id_bytes == 4) {
    FPS_DISPATCH_LPR(fps_pull_dot_kernel, int, lpr, grid, stream, *t, (const int*)ids, n, local,
                     local_stride, score)
  } else {
    FPS_DISPATCH_LPR(fps_pull_dot_kernel, long long, lpr, grid, stream, *t, (const long long*)ids,
                     n, local, local_stride, score)
  }
  return (int)cudaGetLastError();
}

extern "C" int fps_push_assign(const ShardTable* t, const void* ids, int id_bytes, long long n,
                               const float* vals, int val_stride, int touch, int num_sms,
                               cudaStream_t stream) {
  if (n <= 0) return 0;
  const int lpr = pick_lpr(t->stride >> 2);
  const int grid = row_grid(n, lpr, num_sms);
  if (id_bytes == 4) {
    FPS_DISPATCH_LPR(fps_push_assign_kernel, int, lpr, grid, stream, *t, (const int*)ids, n, vals,
                     val_stride, touch)
  } else {
    FPS_DISPATCH_LPR(fps_push_assign_kernel, long long, lpr, grid, stream, *t, (const long long*)ids,
                     n, vals, val_stride, touch)
  }
  return (int)cudaGetLastError();
}


// ----------------------------------------------------------------------------------------
// K2 with PS output: table[ids[i], :] += delta[i, :] and out[i, :] = the value AFTER this update --
// SimplePSLogic emits (id, newValue) on EVERY push (SimplePSLogic.scala:16-25).  Returning atomics
// (one per element), so concurrent pushes to one id each see a distinct prefix sum.
// ----------------------------------------------------------------------------------------
template <typename IdT>
__global__ void __launch_bounds__(256)
    fps_push_add_fetch_kernel(const __grid_constant__ ShardTable t, const IdT* __restrict__ ids,
                              long long n, const float* __restrict__ delta, int delta_stride,
                              float* __restrict__ out, int out_stride) {
  const int dim = t.dim;
  const long long total = n * dim;
  for (long long x = blockIdx.x * (long long)blockDim.x + threadIdx.x; x < total;
       x += (long long)gridDim.x * blockDim.x) {
    const long long i = x / dim;
    const int j = (int)(x - i * dim);
    float* row = fps_row_t<IdT>(t, ids[i]);
    const float d = j < delta_stride ? delta[i * (long long)delta_stride + j] : 0.f;
    const float old = atomicAdd_system(row + j, d);
    if (j < out_stride) out[i * (long long)out_stride + j] = old + d;
  }
}

extern "C" int fps_push_add_fetch(const ShardTable* t, const void* ids, int id_bytes, long long n,
                                  const float* delta, int delta_stride, float* out, int out_stride,
                                  int num_sms, cudaStream_t stream) {
  if (n <= 0) return 0;
  long long blocks = (n * t->dim + 255) / 256;
  if (blocks > (long long)num_sms * 8) blocks = (long long)num_sms * 8;
  if (id_bytes == 4)
    fps_push_add_fetch_kernel<int><<<(int)blocks, 256, 0, stream>>>(*t, (const int*)ids, n, delta, delta_stride, out, out_stride);
  else
    fps_push_add_fetch_kernel<long long><<<(int)blocks, 256, 0, stream>>>(*t, (const long long*)ids, n, delta, delta_stride, out, out_stride);
  return (int)cudaGetLastError();
}
