// Argument block of the fused matrix-factorisation step (fps_core.cu register-staged kernel and
// fps_mf_tma.cu TMA-pipelined kernel).  Mirrored by ops/native.py::MfArgsC.
#pragma once
#include "fps_common.cuh"
#include "fps_launch.cuh"

struct MfArgs {
  const void* users;
  const void* items;
  const float* ratings;
  long long n_pos;
  int neg_rate;
  long long num_items;        // negative-sample id range [0, num_items)
  unsigned long long seed;    // negative-sample stream key
  unsigned long long step;    // negative-sample stream counter (micro-batch number)
  float* user_table;          // worker-local [n_local_users, stride]
  int user_div;               // workerParallelism: local slot = user / user_div
  int user_shift;             // log2(user_div) if power of two, else -1
  float lr;
  int err_mode;               // 0: reference parity sigmoid(r - u.v); 1: plain residual r - u.v;
                              // 2: logistic r - sigmoid(u.v) (skip-gram negative sampling)
  int format;                 // 0: users/items/ratings arrays; 1: packed64 records in `users`
                              //    (user:26 | item:22 | rating fp16:16) -- 8 B/update over PCIe
  float* stats;               // [0] += sum (r-u.v)^2, [1] += #updates
  int* nan_flag;              // set to 1 if a non-finite update was produced
  ShardTable item_tab;
  ShardTable user_tab;        // used when user_sharded != 0: the "user" rows also live on the PS
  int user_sharded;           //   (word2vec: input vectors and output vectors are both PS tables)
  int use_push_tab;           // != 0: item deltas are pushed into push_tab instead of item_tab
  ShardTable push_tab;        //   (worker-side delta staging of the item-cache mode, see fps_cache_sync)
  int l2_hints;               // != 0: item rows evict_last, user rows evict_first (L2-blocked batches)
  int pad2_;
  unsigned int* progress;    // optional: CTA 0 publishes the record index it has reached (replica
                             //   exchange kernels follow the sweep over the L2-blocked batch)
  // E5 worker output stream (ps.output((user, userVector)) after every update,
  // PSOnlineMatrixFactorizationWorker.scala:52): record idx is emitted iff idx % out_every == 0, into the
  // device staging area of an OutputRing at slot *out_staged + idx / out_every (dropped beyond out_cap)
  long long* out_ids;
  float* out_vecs;
  const unsigned long long* out_staged;
  long long out_cap;
  int out_every;             // 0 = no output stream
  int reserve_total;         // CTA slots left free on the whole GPU (the replica exchange CTAs)
  int* credits;              // device-side pull limiter (WL:196-250): credits[0] = pulls that may still be
                             //   issued, credits[1] = stall counter; nullptr = unlimited
  // Row-wise AdaGrad (one fp32 accumulator per row, partitioned like its table; stride 1).
  // item_acc.base[0] == nullptr means plain SGD.
  ShardTable item_acc;       // item accumulators, addressed like item_tab (peer shards over NVLink)
  ShardTable user_acc_tab;   // user accumulators when user_sharded != 0 (skip-gram W_in)
  float* user_acc;           // worker-local [n_local_users] user accumulators otherwise
};

// Argument block of the pairwise steps: fps_mf_bpr.cu (BPR) and fps_mf_warp.cu (WARP).  Mirrored by
// ops/native.py::BprArgsC.
struct BprArgs {
  const void* users;          // anchor ids, or packed64 records (user:26 | item:22 | rating fp16:16)
  const void* items;          // positive candidate ids
  const float* ratings;       // records with rating <= 0 are skipped
  const void* negatives;      // [n_pos, n_neg] candidate ids, -1 = void; nullptr = sampled in the kernel
  long long n_pos;
  int n_neg;
  int format;                 // 0: users/items/ratings arrays; 1: packed64 records in `users`
  long long num_items;        // sampled negatives: id range [0, num_items)
  unsigned long long seed;    // sampled negatives: stream key
  unsigned long long step;    // sampled negatives: stream counter (micro-batch number)
  float lr;
  float reg;
  float* anchor_table;        // worker-local [rows, stride] when anchor_sharded == 0
  int anchor_div;             //   slot = id / anchor_div
  int anchor_shift;           //   log2(anchor_div) if a power of two, else -1
  int anchor_sharded;         // != 0: anchor rows are read and pushed through anchor_tab
  int cand_sharded;           // != 0: candidate rows are read through cand_tab
  ShardTable anchor_tab;
  float* cand_table;          // worker-local [rows, stride] when cand_sharded == 0
  int cand_div;
  int cand_shift;
  ShardTable cand_tab;
  int use_push_tab;           // != 0 (with cand_sharded): candidate deltas go to push_tab
  int stride;                 // row stride in floats, shared by every table
  ShardTable push_tab;
  float* stats;               // [0] += softplus(-x), [1] += #triples, [2] += #(x > 0)
  int* nan_flag;              // set to 1 if a non-finite update was produced
  int reserve_total;          // CTA slots left free on the whole GPU (the replica exchange CTAs)
  int pad_;
  // Row-wise AdaGrad accumulators (one fp32 per row, stride 1); cand_acc.base[0] == nullptr means SGD
  ShardTable anchor_acc_tab;  // anchor accumulators when anchor_sharded != 0
  ShardTable cand_acc;        // candidate accumulators, addressed like cand_tab
  float* anchor_acc;          // worker-local anchor accumulators (slot = id / anchor_div) otherwise
  // WARP (fps_mf_warp.cu): a candidate violates when u . (v_i - v_j) < margin; the rank estimate of a
  // positive whose first violator was its n-th live candidate is (rank_items - 1) / n
  long long rank_items;
  float margin;
  int pad2_;
};

// Row address of `id` in a worker-local table (slot = id / div) or through a ShardTable.
template <typename IdT>
__device__ __forceinline__ float* bpr_row(float* local, int div, int shift, int sharded,
                                          const ShardTable& t, IdT id, int stride) {
  if (sharded) return fps_row_t<IdT>(t, id);
  return local + fps_user_slot<IdT>(id, div, shift) * (size_t)stride;
}

__device__ __forceinline__ float4 bpr_axpy(float a, float4 x, float b, float4 y) {
  return make_float4(a * x.x + b * y.x, a * x.y + b * y.y, a * x.z + b * y.z, a * x.w + b * y.w);
}

// Row-wise AdaGrad accumulator access: a scalar load of G as pulled, and the one-sided G += s.
__device__ __forceinline__ float fps_ld_f32(const float* p) {
  float v;
  asm volatile("ld.global.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void fps_red_add1(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
// lr / (sqrt(G + s) + eps): the step of a row whose accumulator read G and whose squared delta mean is s
__device__ __forceinline__ float fps_adagrad_scale(float lr, float G, float s) {
  return lr / (sqrtf(G + s) + 1e-8f);
}

// The pointwise update rule, shared by every fp32 kernel that applies it (fps_core.cu per-launch kernel,
// fps_mf_window.cu windowed drain): one lane's part of u.v, and the step g = lr * e from the group's dot.
// Keeping one copy keeps the two paths bitwise equal.  The dot is spelled as the FMA chain nvcc contracts
// u.x*v.x + u.y*v.y + u.z*v.z + u.w*v.w to (SASS: FMUL y, FFMA x, FFMA z, FFMA w), so that contraction cannot
// differ between kernels.
__device__ __forceinline__ float fps_mf_dot4(float4 u, float4 v) {
  return fmaf(u.w, v.w, fmaf(u.z, v.z, fmaf(u.x, v.x, u.y * v.y)));
}
__device__ __forceinline__ float fps_mf_grad(int err_mode, float lr, float rating, float d, float resid) {
  const float e = (err_mode == 0)   ? 1.f / (1.f + __expf(-resid))
                  : (err_mode == 1) ? resid
                                    : rating - 1.f / (1.f + __expf(-d));
  return lr * e;
}
