// K7: passive-aggressive step on a CSR micro-batch, fused with the pulls and pushes.
//
// One CTA per example.  Phase 1 pulls the rows w[idx] of every active feature (16-byte loads from
// the owning shard -- local HBM or NVLink peer) and accumulates the decision vector d = W^T x.
// Phase 2 computes the update multipliers (binary PA / PA-I / PA-II, one-versus-all PA variants,
// cost-based PB / ML).  Phase 3 pushes x_i * mult to every active feature's row with
// red.global.add.v4.f32, i.e. the additive paramUpdate runs in the owner's memory system.
// Unlabelled examples only predict.  This is the reference's worker
// (PassiveAggressiveParameterServer.scala:283-340: nnz pulls + nnz pushes per example, ~10^4 each in
// its test) as ONE kernel per micro-batch; examples inside a micro-batch race like the reference's
// asynchronous workers do.
//
// Update rules reproduced: PassiveAggressiveBinaryAlgorithm.scala:44-112,
// PassiveAggressiveOneVersusAll.scala:38-123, PassiveAggressiveCostBased.scala:30-140.
#include "fps_common.cuh"

enum FpsPaAlgo : int { PA_PA = 0, PA_PAI = 1, PA_PAII = 2, PA_PB = 3, PA_ML = 4 };
#define PA_UNLABELLED (-2147483647 - 1)
#define PA_MAX_LABELS 1024
#define PA_THREADS 128

struct PaArgs {
  const long long* row_ptr;  // [n + 1]
  const void* col_idx;       // [nnz] feature ids
  const float* values;       // [nnz]
  const int* labels;         // [n]: binary: +1 / -1, multiclass: class index, PA_UNLABELLED: predict
  int* pred;                 // [n] out: binary 1/0, multiclass argmax
  float* loss;               // [n] out (optional): suffered loss (binary) / max label loss
  const float* cost;         // [L, L] cost matrix for PB / ML (may be null)
  long long n;
  int binary;                // 1: scalar weights, labels are +-1
  int num_labels;            // L (1 for binary)
  int algo;                  // FpsPaAlgo
  float aggressiveness;      // C
  int* nan_flag;
  ShardTable tab;            // one row per feature: [stride >= L] floats
};

// Arg-max order of both kernels: (v, i) beats (best, arg) if v is larger, or equal with a lower index;
// NaN ranks above every number.  This is np.argmax (first maximum, first NaN), it is a total order, so
// every lane of a shuffle reduction ends on the same winner, and a seed of (-inf, INT_MAX) loses to
// every real column, even when all of them are -inf.
__device__ __forceinline__ bool pa_beats(float v, int i, float best, int arg) {
  const bool vn = v != v, bn = best != best;
  if (vn != bn) return vn;
  return v > best || (!(v < best) && i < arg);
}

template <typename IdT, int LPR>
__global__ void __launch_bounds__(PA_THREADS)
    fps_pa_step_kernel(const __grid_constant__ PaArgs a) {
  __shared__ float s_dec[PA_MAX_LABELS];   // decision vector, then the multipliers
  __shared__ float s_norm;
  __shared__ int s_aux[2];
  const IdT* __restrict__ cols = reinterpret_cast<const IdT*>(a.col_idx);
  const int L = a.num_labels;
  const int nvec = a.tab.stride >> 2;
  const int lane = threadIdx.x & (LPR - 1);
  const int grp = threadIdx.x / LPR;
  constexpr int NGRP = PA_THREADS / LPR;
  // rows of up to LPR chunks use one chunk per lane; only the widest variant (LPR = 32) loops
  constexpr int VPL = LPR < 32 ? 1 : PA_MAX_LABELS / 4 / 32;

  for (long long ex = blockIdx.x; ex < a.n; ex += gridDim.x) {
    const long long b = a.row_ptr[ex], e = a.row_ptr[ex + 1];
    for (int i = threadIdx.x; i < L; i += PA_THREADS) s_dec[i] = 0.f;
    if (threadIdx.x == 0) s_norm = 0.f;
    __syncthreads();
    // ---- phase 1: d = W^T x, ||x||^2 ------------------------------------------------------
    float4 acc[VPL];
#pragma unroll
    for (int c = 0; c < VPL; ++c) acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    float n2 = 0.f;
    for (long long j = b + grp; j < e; j += NGRP) {
      const float x = a.values[j];
      const float* row = fps_row_t<IdT>(a.tab, cols[j]);
      if (lane == 0) n2 += x * x;
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        if (q < nvec) {
          const float4 w = fps_ld_row4(row + 4 * q);  // the PULL
          acc[c].x += x * w.x; acc[c].y += x * w.y; acc[c].z += x * w.z; acc[c].w += x * w.w;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int q = lane + c * LPR;
      if (q < nvec) {
        if (4 * q + 0 < L) atomicAdd(&s_dec[4 * q + 0], acc[c].x);
        if (4 * q + 1 < L) atomicAdd(&s_dec[4 * q + 1], acc[c].y);
        if (4 * q + 2 < L) atomicAdd(&s_dec[4 * q + 2], acc[c].z);
        if (4 * q + 3 < L) atomicAdd(&s_dec[4 * q + 3], acc[c].w);
      }
    }
    if (lane == 0 && n2 != 0.f) atomicAdd(&s_norm, n2);
    __syncthreads();
    // ---- phase 2: prediction + multipliers (thread 0 for scalars, all threads for OVA) -----
    const int label = a.labels[ex];
    const float nsq = s_norm;
    if (threadIdx.x == 0) {
      int arg = 0;
      float best = s_dec[0];
      for (int i = 1; i < L; ++i)
        if (pa_beats(s_dec[i], i, best, arg)) { best = s_dec[i]; arg = i; }
      a.pred[ex] = a.binary ? (s_dec[0] > 0.f ? 1 : 0) : arg;
      s_aux[0] = arg;
      s_aux[1] = -1;
    }
    __syncthreads();
    bool push = (label != PA_UNLABELLED) && (e > b) && nsq > 0.f;
    if (push) {
      if (a.binary || a.algo <= PA_PAII) {
        // binary: y = label (+-1); OVA: y_i = +1 for the true class, -1 otherwise
        float max_loss = 0.f;
        for (int i = threadIdx.x; i < L; i += PA_THREADS) {
          const float y = a.binary ? (float)label : (i == label ? 1.f : -1.f);
          const float l = fmaxf(0.f, 1.f - y * s_dec[i]);
          float tau;
          if (a.algo == PA_PA) tau = l / nsq;
          else if (a.algo == PA_PAI) tau = fminf(a.aggressiveness, l / nsq);
          else tau = l / (nsq + 1.f / (2.f * a.aggressiveness));
          s_dec[i] = tau * y;  // multiplier for label column i
          max_loss = fmaxf(max_loss, l);
        }
        if (a.loss != nullptr && threadIdx.x == 0 && L == 1) a.loss[ex] = max_loss;
      } else {
        // cost based PB / ML: two columns get +-tau, everything else 0
        if (threadIdx.x == 0) {
          int q = s_aux[0];
          if (a.algo == PA_ML) {
            float bestv = -INFINITY;
            q = 0x7fffffff;
            for (int i = 0; i < L; ++i) {
              const float c = a.cost ? a.cost[label * L + i] : (i == label ? 0.f : 1.f);
              const float v = s_dec[i] - s_dec[label] + sqrtf(c);
              if (pa_beats(v, i, bestv, q)) { bestv = v; q = i; }
            }
          }
          float tau = 0.f;
          if (q != label) {
            const float c = a.cost ? a.cost[label * L + q] : 1.f;
            const float l = s_dec[q] - s_dec[label] + sqrtf(c);
            tau = l / (2.f * nsq);
            if (a.loss != nullptr) a.loss[ex] = l;
          }
          s_aux[1] = q;
          s_norm = tau;
        }
        __syncthreads();
        const int q = s_aux[1];
        const float tau = s_norm;
        for (int i = threadIdx.x; i < L; i += PA_THREADS)
          s_dec[i] = (q == label) ? 0.f : (i == label ? tau : (i == q ? -tau : 0.f));
      }
    }
    __syncthreads();
    // ---- phase 3: push x_i * mult to every active feature --------------------------------
    if (push) {
      bool bad = false;
      for (long long j = b + grp; j < e; j += NGRP) {
        const float x = a.values[j];
        float* row = fps_row_t<IdT>(a.tab, cols[j]);
#pragma unroll
        for (int c = 0; c < VPL; ++c) {
          const int q = lane + c * LPR;
          if (q < nvec && 4 * q < L) {
            float4 d;
            d.x = x * s_dec[4 * q + 0];
            d.y = (4 * q + 1 < L) ? x * s_dec[4 * q + 1] : 0.f;
            d.z = (4 * q + 2 < L) ? x * s_dec[4 * q + 2] : 0.f;
            d.w = (4 * q + 3 < L) ? x * s_dec[4 * q + 3] : 0.f;
            if (d.x != 0.f || d.y != 0.f || d.z != 0.f || d.w != 0.f) {
              // all four columns, like the warp kernel: one inf or NaN anywhere in the chunk flags it
              if (!(fabsf(d.x) + fabsf(d.y) + fabsf(d.z) + fabsf(d.w) <= 3.0e38f)) bad = true;
              fps_red_add4(row + 4 * q, d);  // the PUSH fused with paramUpdate (+)
            }
          }
        }
      }
      if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
    }
    __syncthreads();
  }
}

// ---- warp-per-example variant for rows of up to 32 16-byte chunks (<= 128 labels) ------------------
// The block kernel above spends most of its time in __syncthreads and single-thread phases when an
// example has a few hundred features (ncu: 34 % warps active, DRAM 6 %).  Here one warp owns an
// example: LPR lanes cooperate on a feature row (lane l holds labels 4*(l % LPR) .. +3), 32/LPR rows
// are pulled per step with 4 independent steps in flight, the decision vector is reduced with
// shuffles and stays distributed over the LPR lanes, multipliers are computed in registers and the
// pushes follow immediately -- no shared memory, no block barrier.
__device__ __forceinline__ float pa_sel4(const float4& v, int i) {
  return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}
__device__ __forceinline__ void pa_red_add1(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
// (value, index) arg-max over the LPR lanes of a group in pa_beats order (first maximum wins, like the
// sequential scans of the host algorithms)
template <int LPR>
__device__ __forceinline__ void pa_group_argmax(float& v, int& idx) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (pa_beats(ov, oi, v, idx)) { v = ov; idx = oi; }
  }
}
// component `label` of the distributed decision vector, broadcast to every lane
template <int LPR>
__device__ __forceinline__ float pa_group_get(const float4& mine, int label, int lane) {
  const float cand = pa_sel4(mine, label & 3);
  return __shfl_sync(0xffffffffu, cand, (lane & ~(LPR - 1)) + (label >> 2));
}

template <typename IdT, int LPR>
__global__ void __launch_bounds__(256, 4) fps_pa_step_warp_kernel(const __grid_constant__ PaArgs a) {
  constexpr int G = 32 / LPR;  // feature rows per warp step
  const IdT* __restrict__ cols = reinterpret_cast<const IdT*>(a.col_idx);
  const int L = a.num_labels;  // <= 4 * LPR
  const int lane = threadIdx.x & 31;
  const int q = lane & (LPR - 1);   // my 16-byte chunk of every row: labels 4q .. 4q+3
  const int grp = lane / LPR;
  const bool chunk_ok = 4 * q < L;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  bool bad = false;
  for (long long ex = warp; ex < a.n; ex += n_warps) {
    const long long b = a.row_ptr[ex], e = a.row_ptr[ex + 1];
    // ---- phase 1: d = W^T x, ||x||^2 ------------------------------------------------------
    float4 dec = make_float4(0.f, 0.f, 0.f, 0.f);
    float n2 = 0.f;
    for (long long j = b + grp; j < e; j += 4 * G) {
      float x[4];
      float4 w[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long jj = j + G * u;
        x[u] = 0.f;
        w[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (jj < e) {
          x[u] = a.values[jj];
          if (chunk_ok) w[u] = fps_ld_row4(fps_row_t<IdT>(a.tab, cols[jj]) + 4 * q);  // the PULL
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        dec.x += x[u] * w[u].x; dec.y += x[u] * w[u].y; dec.z += x[u] * w[u].z; dec.w += x[u] * w[u].w;
        if (q == 0) n2 += x[u] * x[u];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      if (o >= LPR) {  // sum the 32/LPR row groups; lanes with equal q end up with the same chunk
        dec.x += __shfl_xor_sync(0xffffffffu, dec.x, o);
        dec.y += __shfl_xor_sync(0xffffffffu, dec.y, o);
        dec.z += __shfl_xor_sync(0xffffffffu, dec.z, o);
        dec.w += __shfl_xor_sync(0xffffffffu, dec.w, o);
      }
      n2 += __shfl_xor_sync(0xffffffffu, n2, o);
    }
    // ---- phase 2: prediction + multipliers ---------------------------------------------------
    const int label = a.labels[ex];
    // the seed loses to every column, -inf and NaN included; a lane past L keeps it and loses the reduction
    float best = -INFINITY;
    int arg = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float v = pa_sel4(dec, i);
      if (4 * q + i < L && pa_beats(v, 4 * q + i, best, arg)) { best = v; arg = 4 * q + i; }
    }
    pa_group_argmax<LPR>(best, arg);
    if (lane == 0) a.pred[ex] = a.binary ? (best > 0.f ? 1 : 0) : arg;
    if (label == PA_UNLABELLED || e <= b || !(n2 > 0.f)) continue;
    float4 mult = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.binary || a.algo <= PA_PAII) {
      float m[4];
      float max_loss = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        m[i] = 0.f;
        if (4 * q + i < L) {
          const float y = a.binary ? (float)label : (4 * q + i == label ? 1.f : -1.f);
          const float l = fmaxf(0.f, 1.f - y * pa_sel4(dec, i));
          float tau;
          if (a.algo == PA_PA) tau = l / n2;
          else if (a.algo == PA_PAI) tau = fminf(a.aggressiveness, l / n2);
          else tau = l / (n2 + 1.f / (2.f * a.aggressiveness));
          m[i] = tau * y;
          max_loss = fmaxf(max_loss, l);
        }
      }
      mult = make_float4(m[0], m[1], m[2], m[3]);
      if (a.loss != nullptr && lane == 0 && L == 1) a.loss[ex] = max_loss;
    } else {
      // cost based PB / ML: the true label's column gets +tau, the offending column -tau
      int qq = arg;
      const float d_label = pa_group_get<LPR>(dec, label, lane);
      if (a.algo == PA_ML) {
        float bestv = -INFINITY;
        int bi = 0x7fffffff;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int li = 4 * q + i;
          if (li < L) {
            const float c = a.cost ? a.cost[label * L + li] : (li == label ? 0.f : 1.f);
            const float v = pa_sel4(dec, i) - d_label + sqrtf(c);
            if (pa_beats(v, li, bestv, bi)) { bestv = v; bi = li; }
          }
        }
        pa_group_argmax<LPR>(bestv, bi);
        qq = bi;
      }
      float tau = 0.f;
      const float d_q = pa_group_get<LPR>(dec, qq, lane);
      if (qq != label) {
        const float c = a.cost ? a.cost[label * L + qq] : 1.f;
        const float l = d_q - d_label + sqrtf(c);
        tau = l / (2.f * n2);
        if (a.loss != nullptr && lane == 0) a.loss[ex] = l;
      }
      float m[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int li = 4 * q + i;
        m[i] = (qq == label) ? 0.f : (li == label ? tau : (li == qq ? -tau : 0.f));
      }
      mult = make_float4(m[0], m[1], m[2], m[3]);
    }
    // ---- phase 3: push x_i * mult to every active feature --------------------------------
    if (chunk_ok && (mult.x != 0.f || mult.y != 0.f || mult.z != 0.f || mult.w != 0.f)) {
      for (long long j = b + grp; j < e; j += G) {
        const float x = a.values[j];
        float* row = fps_row_t<IdT>(a.tab, cols[j]) + 4 * q;
        const float4 d = make_float4(x * mult.x, x * mult.y, x * mult.z, x * mult.w);
        if (d.x != 0.f || d.y != 0.f || d.z != 0.f || d.w != 0.f) {
          if (!(fabsf(d.x) + fabsf(d.y) + fabsf(d.z) + fabsf(d.w) <= 3.0e38f)) bad = true;
          if (L == 1) pa_red_add1(row, d.x);   // the PUSH fused with paramUpdate (+)
          else fps_red_add4(row, d);
        }
      }
    }
  }
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
}

static int g_pa_variant = 0;  // 0: auto (warp kernel for one-chunk rows), 1: always the block kernel
extern "C" void fps_set_pa_variant(int v) { g_pa_variant = v; }

template <typename IdT>
static int dispatch_pa(const PaArgs& a, int num_sms, cudaStream_t s) {
  const int nvec = a.tab.stride >> 2;
  long long blocks = a.n;
  const long long cap = (long long)num_sms * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  const int g = (int)blocks;
  if (nvec <= 32 && a.num_labels <= 128 && g_pa_variant == 0) {
    long long warps = a.n;
    if (warps > (long long)num_sms * 32) warps = (long long)num_sms * 32;
    const int wg = (int)((warps + 7) / 8);
    if (nvec <= 1) fps_pa_step_warp_kernel<IdT, 1><<<wg, 256, 0, s>>>(a);
    else if (nvec <= 2) fps_pa_step_warp_kernel<IdT, 2><<<wg, 256, 0, s>>>(a);
    else if (nvec <= 4) fps_pa_step_warp_kernel<IdT, 4><<<wg, 256, 0, s>>>(a);
    else if (nvec <= 8) fps_pa_step_warp_kernel<IdT, 8><<<wg, 256, 0, s>>>(a);
    else if (nvec <= 16) fps_pa_step_warp_kernel<IdT, 16><<<wg, 256, 0, s>>>(a);
    else fps_pa_step_warp_kernel<IdT, 32><<<wg, 256, 0, s>>>(a);
    return (int)cudaGetLastError();
  }
  if (nvec <= 1) fps_pa_step_kernel<IdT, 1><<<g, PA_THREADS, 0, s>>>(a);
  else if (nvec <= 2) fps_pa_step_kernel<IdT, 2><<<g, PA_THREADS, 0, s>>>(a);
  else if (nvec <= 4) fps_pa_step_kernel<IdT, 4><<<g, PA_THREADS, 0, s>>>(a);
  else if (nvec <= 8) fps_pa_step_kernel<IdT, 8><<<g, PA_THREADS, 0, s>>>(a);
  else if (nvec <= 16) fps_pa_step_kernel<IdT, 16><<<g, PA_THREADS, 0, s>>>(a);
  else fps_pa_step_kernel<IdT, 32><<<g, PA_THREADS, 0, s>>>(a);
  return (int)cudaGetLastError();
}

extern "C" int fps_pa_step(const PaArgs* args, int id_bytes, int num_sms, cudaStream_t stream) {
  if (args->n <= 0) return 0;
  if (args->num_labels > PA_MAX_LABELS || args->num_labels < 1) return -1006;
  if (args->num_labels > args->tab.stride) return -1006;
  if (id_bytes == 4) return dispatch_pa<int>(*args, num_sms, stream);
  if (id_bytes == 8) return dispatch_pa<long long>(*args, num_sms, stream);
  return -1001;
}
