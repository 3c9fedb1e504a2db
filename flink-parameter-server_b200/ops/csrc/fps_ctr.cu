// Wide-&-deep CTR dense tower (BASELINE.json config 3), one fused kernel per micro-batch:
//
//   x_e   = the F pulled embedding rows of example e, concatenated (IN = F * E inputs) + F "wide" weights
//   h     = relu(W1^T x + b1)                       (H hidden units)
//   logit = w2 . h + b2 + sum_f wide_f ;  p = sigmoid(logit) ;  loss = BCE(p, y)
//   backward in the same kernel: dW1, db1, dw2, db2 accumulated (red.add), and the gradient with respect
//   to every pulled row written out already scaled by -lr, ready to be PUSHED (red.add into the shards).
//
// The embedding rows arrive from the one-sided gather kernel under the device credit-counter pull limiter
// (fps_pull_gather with credits, pull-limiter = 64 in the named config); this kernel replaces the torch
// autograd + cuBLAS tower of round 1: no library GEMM, no host synchronisation (the loss stays on the
// device).  5 GFLOP per 16K-example batch on the CUDA cores -- the step is bound by the 64-credit
// limiter, not by this math, so the tensor cores are not worth a second weight layout here.
//
// Mapping: a CTA of H threads (H == 256) walks tiles of TB = 32 examples.  Forward and dW1: thread j owns
// hidden unit j (W1 is [IN][H], row i contiguous in j -> coalesced loads and coalesced REDs).  dX: thread
// i owns input i and reads the transposed copy W1T [H][IN] (kept in sync by fps_ctr_apply).
#include "fps_common.cuh"

#define CTR_H 256
#define CTR_TB 32
#define CTR_MAX_IN 256

struct CtrArgs {
  const float* rows;     // [B * F, stride]   pulled rows: E embedding values, then the wide weight
  const float* labels;   // [B]
  long long batch;
  int fields, emb, stride;
  const float* W1;       // [IN][H]
  const float* W1T;      // [H][IN]
  const float* b1;       // [H]
  const float* w2;       // [H]
  const float* b2;       // [1]
  float* gW1;            // [IN][H]   gradient sums (zeroed by fps_ctr_apply)
  float* gb1;            // [H]
  float* gw2;            // [H]
  float* gb2;            // [1]
  float* d_rows;         // [B * F, stride]  OUT: -lr * dLoss/d(row)
  float* loss;           // [2]: sum of BCE, number of examples
  float* prob;           // optional [B]: sigmoid(logit)
  float lr;
  int train;             // 0: forward only (predict)
};

__global__ void __launch_bounds__(CTR_H, 1) fps_ctr_tower_kernel(const __grid_constant__ CtrArgs a) {
  extern __shared__ float ctr_smem[];
  const int IN = a.fields * a.emb;
  float* X = ctr_smem;                       // [TB][IN]
  float* D = X + CTR_TB * IN;                // [TB][H]   dH tile
  float* red = D + CTR_TB * CTR_H;           // [8][TB]   per-warp logit partials
  float* dlog = red + 8 * CTR_TB;            // [TB]
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float b1j = a.b1[t], w2j = a.w2[t], b2 = a.b2[0];
  float gw2_acc = 0.f, gb1_acc = 0.f, gb2_acc = 0.f, loss_acc = 0.f, cnt_acc = 0.f;
  const long long n_tiles = (a.batch + CTR_TB - 1) / CTR_TB;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long e0 = tile * CTR_TB;
    const int ne = (int)min((long long)CTR_TB, a.batch - e0);
    // ---- stage the tile's inputs: X[e][f*E + c] = rows[(e0+e)*F + f][c] ---------------------------------
    for (int x = t; x < CTR_TB * IN; x += CTR_H) {
      const int e = x / IN, i = x - e * IN;
      const int f = i / a.emb, c = i - f * a.emb;
      X[x] = e < ne ? a.rows[((e0 + e) * a.fields + f) * (long long)a.stride + c] : 0.f;
    }
    __syncthreads();
    // ---- forward: thread j = hidden unit j ------------------------------------------------------------------
    float acc[CTR_TB];
#pragma unroll
    for (int e = 0; e < CTR_TB; ++e) acc[e] = b1j;
    for (int i = 0; i < IN; ++i) {
      const float w = a.W1[i * CTR_H + t];
#pragma unroll
      for (int e = 0; e < CTR_TB; ++e) acc[e] = fmaf(X[e * IN + i], w, acc[e]);
    }
#pragma unroll
    for (int e = 0; e < CTR_TB; ++e) {
      acc[e] = fmaxf(acc[e], 0.f);                       // h[e][j]
      float p = acc[e] * w2j;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
      if (lane == 0) red[warp * CTR_TB + e] = p;
    }
    __syncthreads();
    if (t < CTR_TB) {
      float logit = b2;
      for (int w = 0; w < CTR_H / 32; ++w) logit += red[w * CTR_TB + t];
      float d = 0.f;
      if (t < ne) {
        for (int f = 0; f < a.fields; ++f)
          logit += a.rows[((e0 + t) * a.fields + f) * (long long)a.stride + a.emb];   // wide term
        const float y = a.labels[e0 + t];
        const float p = 1.f / (1.f + __expf(-logit));
        d = p - y;
        if (a.prob != nullptr) a.prob[e0 + t] = p;
        // numerically safe BCE with logits
        loss_acc += fmaxf(logit, 0.f) - logit * y + log1pf(__expf(-fabsf(logit)));
        cnt_acc += 1.f;
        gb2_acc += d;
      }
      dlog[t] = d;
    }
    __syncthreads();
    if (!a.train) continue;     // predict: forward only (uniform branch, no barrier is skipped unevenly)
    // ---- backward through the hidden layer (thread j) -----------------------------------------------------------
#pragma unroll
    for (int e = 0; e < CTR_TB; ++e) {
      const float d = dlog[e];
      gw2_acc = fmaf(d, acc[e], gw2_acc);
      const float dh = acc[e] > 0.f ? d * w2j : 0.f;
      gb1_acc += dh;
      acc[e] = dh;
      D[e * CTR_H + t] = dh;
    }
    // dW1[i][j] += sum_e X[e][i] * dh[e][j]   (coalesced RED over j)
    for (int i = 0; i < IN; ++i) {
      float g = 0.f;
#pragma unroll
      for (int e = 0; e < CTR_TB; ++e) g = fmaf(X[e * IN + i], acc[e], g);
      if (g != 0.f) atomicAdd(a.gW1 + i * CTR_H + t, g);
    }
    __syncthreads();
    // ---- dX (thread i = input i, transposed weights) -> row gradients, scaled by -lr ---------------------
    if (t < IN) {
      float dx[CTR_TB];
#pragma unroll
      for (int e = 0; e < CTR_TB; ++e) dx[e] = 0.f;
      for (int j = 0; j < CTR_H; ++j) {
        const float w = a.W1T[j * IN + t];
#pragma unroll
        for (int e = 0; e < CTR_TB; ++e) dx[e] = fmaf(D[e * CTR_H + j], w, dx[e]);
      }
      const int f = t / a.emb, c = t - f * a.emb;
#pragma unroll
      for (int e = 0; e < CTR_TB; ++e)
        if (e < ne) a.d_rows[((e0 + e) * a.fields + f) * (long long)a.stride + c] = -a.lr * dx[e];
    }
    // wide weights and padding columns of the pushed rows
    for (int x = t; x < ne * a.fields; x += CTR_H) {
      const int e = x / a.fields, f = x - e * a.fields;
      float* dr = a.d_rows + ((e0 + e) * a.fields + f) * (long long)a.stride;
      dr[a.emb] = -a.lr * dlog[e];
      for (int c = a.emb + 1; c < a.stride; ++c) dr[c] = 0.f;
    }
    __syncthreads();
  }
  if (a.train) {
    atomicAdd(a.gw2 + t, gw2_acc);
    atomicAdd(a.gb1 + t, gb1_acc);
  }
  if (t < CTR_TB) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      gb2_acc += __shfl_xor_sync(0xffffffffu, gb2_acc, o);
      loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);
      cnt_acc += __shfl_xor_sync(0xffffffffu, cnt_acc, o);
    }
    if (t == 0) {
      if (a.train) atomicAdd(a.gb2, gb2_acc);
      atomicAdd(a.loss, loss_acc);
      atomicAdd(a.loss + 1, cnt_acc);
    }
  }
}

// SGD on the dense weights with the mean gradient of the micro-batch, both weight layouts kept in sync,
// gradient buffers zeroed for the next step.
__global__ void fps_ctr_apply_kernel(float* W1, float* W1T, float* b1, float* w2, float* b2, float* gW1,
                                     float* gb1, float* gw2, float* gb2, int IN, float scale) {
  const int n = IN * CTR_H;
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
    const int i = x / CTR_H, j = x - i * CTR_H;
    const float w = W1[x] - scale * gW1[x];
    W1[x] = w;
    W1T[j * IN + i] = w;
    gW1[x] = 0.f;
    if (i == 0) {
      b1[j] -= scale * gb1[j]; gb1[j] = 0.f;
      w2[j] -= scale * gw2[j]; gw2[j] = 0.f;
    }
    if (x == 0) { b2[0] -= scale * gb2[0]; gb2[0] = 0.f; }
  }
}

extern "C" int fps_ctr_step(const CtrArgs* a, float* W1, float* W1T, float* b1, float* w2, float* b2,
                            int num_sms, cudaStream_t stream) {
  const int train = a->train;
  if (a->batch <= 0) return 0;
  const int IN = a->fields * a->emb;
  if (IN > CTR_MAX_IN || IN > CTR_H) return -1501;
  // the wide weight is column `emb` of every pulled row: a narrower stride would read the next row's first float
  if (a->stride < a->emb + 1) return -1801;
  const size_t smem = (size_t)(CTR_TB * IN + CTR_TB * CTR_H + 8 * CTR_TB + CTR_TB) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(fps_ctr_tower_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  long long tiles = (a->batch + CTR_TB - 1) / CTR_TB;
  int grid = (int)(tiles < num_sms ? tiles : num_sms);
  fps_ctr_tower_kernel<<<grid, CTR_H, smem, stream>>>(*a);
  e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  if (train) {
    fps_ctr_apply_kernel<<<(IN * CTR_H + 255) / 256, 256, 0, stream>>>(W1, W1T, b1, w2, b2, a->gW1, a->gb1, a->gw2,
                                                                       a->gb2, IN, a->lr / (float)a->batch);
    e = cudaGetLastError();
  }
  return (int)e;
}
