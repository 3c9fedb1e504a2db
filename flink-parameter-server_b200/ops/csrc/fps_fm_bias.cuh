// What fps_fm.cu and fps_ffm.cu share (DESIGN §2.15, §2.16): the losses and the end of a launch: the error flags,
// per-warp sums of the loss, the labelled count and sum g into `stats` and `bias_acc`, then the w0 rule.  Every
// example reads w0 as it was before the launch; the last CTA to finish (a launch counter that resets itself, behind
// __threadfence) pushes -lr * sum g / n_labelled to column 0 of the bias row, once per launch.
#pragma once
#include "fps_common.cuh"

enum FmLoss : int { FM_LOGISTIC = 0, FM_SQUARED = 1 };

__device__ __forceinline__ void fps_red_add1(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// An AdaGrad accumulator table (DESIGN §2.17) must address H exactly as the parameter table addresses the row.
__host__ __device__ inline bool fps_same_geometry(const ShardTable& acc, const ShardTable& tab) {
  return acc.stride == tab.stride && acc.dim == tab.dim && acc.rows_per_shard == tab.rows_per_shard &&
         acc.div == tab.div && acc.num_shards == tab.num_shards && acc.mode == tab.mode;
}

// libffm's AdaGrad step of one element (DESIGN §2.17): gam is what plain SGD would scale by -lr, h the element's
// H = G - 1 as pulled.  Returns the delta; gg receives gam^2, the push to H.  sqrtf and the division are IEEE
// round-to-nearest (no fast-math), so the replay's error model charges one rounding each.
__device__ __forceinline__ float fps_adagrad1(float gam, float h, float lr, float& gg) {
  gg = gam * gam;
  return -lr * gam / sqrtf(1.f + h + gg);
}
__device__ __forceinline__ float4 fps_adagrad4(float4 gam, float4 h, float lr, float4& gg) {
  return make_float4(fps_adagrad1(gam.x, h.x, lr, gg.x), fps_adagrad1(gam.y, h.y, lr, gg.y),
                     fps_adagrad1(gam.z, h.z, lr, gg.z), fps_adagrad1(gam.w, h.w, lr, gg.w));
}

// Args: FmArgs or FfmArgs (nan_flag, bad_id, predict_only, stats, bias, bias_acc, bias_done, lr, tab,
// num_features).  Every thread of the CTA calls it after its last example: bad and bad_id raise the flags, and
// unless the launch only predicts, loss_acc, lab_acc and g_acc (the thread's own sums) go on to the w0 rule.
template <typename Args>
__device__ __forceinline__ void fps_fm_bias_tail(const Args& a, bool bad, bool bad_id, float loss_acc, float lab_acc,
                                                 double g_acc) {
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
  if (bad_id && a.bad_id != nullptr) *a.bad_id = 1;
  if (a.predict_only) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);
    lab_acc += __shfl_xor_sync(0xffffffffu, lab_acc, o);
    g_acc += __shfl_xor_sync(0xffffffffu, g_acc, o);
  }
  if ((threadIdx.x & 31) == 0 && lab_acc > 0.f) {
    if (a.stats != nullptr) {
      atomicAdd(a.stats + 0, loss_acc);
      atomicAdd(a.stats + 1, lab_acc);
    }
    if (a.bias) {
      atomicAdd(a.bias_acc + 0, g_acc);
      atomicAdd(a.bias_acc + 1, (double)lab_acc);
    }
  }
  if (!a.bias) return;
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(a.bias_done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last || threadIdx.x != 0) return;
  __threadfence();
  volatile double* acc = a.bias_acc;
  const double sg = acc[0], nl = acc[1];
  float d = 0.f;
  if (nl > 0.0) {
    d = -a.lr * (float)(sg / nl);
    if (!(fabsf(d) <= 3.0e38f) && a.nan_flag != nullptr) *a.nan_flag = 1;
    fps_red_add1(fps_row(a.tab, a.num_features), d);
  }
  acc[0] = 0.0;
  acc[1] = 0.0;
  acc[2] = (double)d;
  acc[3] = acc[3] + (double)d;
  *a.bias_done = 0u;
}
