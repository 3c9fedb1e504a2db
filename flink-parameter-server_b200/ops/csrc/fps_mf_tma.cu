// Flagship kernel, pipelined variant: fused pull + SGD + push for matrix factorisation with the
// PULL executed by the TMA engine (cp.async.bulk, SASS UBLKCP) into a deep shared-memory ring.
//
//   producer warp : for each tile of up to 32 ratings, lane l resolves rating l to
//                   (user row pointer, item row pointer in the OWNER's HBM -- local or NVLink peer),
//                   stores the row metadata in smem and issues two bulk copies
//                   (user row, item row) that complete on the stage's "full" mbarrier.
//   consumer warps: wait "full", read rows from smem, dot -> error -> deltas, and PUSH with
//                   red.global.add.v4.f32 (REDG.E.ADD.F32x4) straight to the owning shard /
//                   the local user table, then release the stage on the "empty" mbarrier.
//
// One persistent CTA per SM; ~190 KB of row data in flight per SM (vs ~64 KB for the
// register-staged kernel in fps_core.cu), which is what covers HBM (~1 us) and NVSwitch (~2-3 us)
// latency at full bandwidth.  The number of stages is the device-side credit pool of the pull
// limiter (WL:196-250): at most stages*32 pulls are un-consumed per CTA at any time.
//
// Reference behaviour reproduced: PSOnlineMatrixFactorizationWorker.scala:42-89, SGDUpdater.scala:8,
// SimplePSLogic.scala:13-25 (see fps_core.cu for the semantics notes).
#include "fps_common.cuh"
#include "fps_mf_args.cuh"
#include "fps_tma.cuh"


#define TILE_ROWS 32
#define N_PRODUCER_WARPS 2
#define N_CONSUMER_WARPS 8
#define TMA_THREADS (32 * (N_PRODUCER_WARPS + N_CONSUMER_WARPS))

struct RowMeta {
  float* up;     // user row (worker-local HBM)
  float* vp;     // item row in the owner shard (local or peer)
  float rating;
  int valid;
};

template <typename IdT, int LPR>
__global__ void __launch_bounds__(TMA_THREADS, 1)
    fps_mf_sgd_tma_kernel(const __grid_constant__ MfArgs a, const int n_stages) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int stride = a.item_tab.stride;
  const int nvec = stride >> 2;
  const uint32_t row_bytes = (uint32_t)stride * 4u;
  // layout: [stages][2][TILE_ROWS][stride] floats | [stages][TILE_ROWS] RowMeta | full[], empty[]
  float* rows = reinterpret_cast<float*>(smem_raw);
  const size_t stage_floats = (size_t)2 * TILE_ROWS * stride;
  RowMeta* meta = reinterpret_cast<RowMeta*>(smem_raw + (size_t)n_stages * stage_floats * 4);
  uint64_t* full = reinterpret_cast<uint64_t*>(meta + (size_t)n_stages * TILE_ROWS);
  uint64_t* empty = full + n_stages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < n_stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], N_CONSUMER_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  const int per_pos = 1 + a.neg_rate;
  const long long n_eff = a.n_pos * per_pos;
  const long long n_tiles = (n_eff + TILE_ROWS - 1) / TILE_ROWS;

  if (warp < N_PRODUCER_WARPS) {
    // ============================== PRODUCERS (TMA issue) ==============================
    // CTA-local tile sequence k = 0,1,2,... maps to global tile t = blockIdx.x + k*gridDim.x and to
    // stage k % n_stages; producer warp pw owns the tiles with k % N_PRODUCER_WARPS == pw
    // (n_stages is a multiple of N_PRODUCER_WARPS, so each producer owns a fixed set of stages).
    const IdT* __restrict__ users = reinterpret_cast<const IdT*>(a.users);
    const IdT* __restrict__ items = reinterpret_cast<const IdT*>(a.items);
    constexpr int PF = 4;  // tiles whose ids are fetched together (hides the id-load latency)
    for (long long k0 = warp;; k0 += (long long)N_PRODUCER_WARPS * PF) {
      if (blockIdx.x + k0 * gridDim.x >= n_tiles) break;
      IdT user[PF], item[PF];
      float rt[PF];
      bool ok[PF];
      int jj[PF];
      long long pp[PF];
#pragma unroll
      for (int p = 0; p < PF; ++p) {
        const long long t = blockIdx.x + (k0 + (long long)p * N_PRODUCER_WARPS) * gridDim.x;
        const long long idx = t * TILE_ROWS + lane;
        ok[p] = (t < n_tiles) && (idx < n_eff);
        user[p] = 0; item[p] = 0; rt[p] = 0.f; jj[p] = 0; pp[p] = 0;
        if (ok[p]) {
          long long pos = idx;
          int j = 0;
          if (per_pos > 1) {
            pos = idx / per_pos;
            j = (int)(idx - pos * per_pos);
          }
          user[p] = users[pos];
          item[p] = items[pos];
          if (user[p] < 0) ok[p] = false;  // record voided upstream (fps_neg_sample: no unseen item found)
          if (j == 0) rt[p] = a.ratings[pos];
          jj[p] = j; pp[p] = pos;
        }
      }
#pragma unroll
      for (int p = 0; p < PF; ++p) {
        const long long k = k0 + (long long)p * N_PRODUCER_WARPS;
        const long long t = blockIdx.x + k * gridDim.x;
        if (t >= n_tiles) break;
        const int stage = (int)(k % n_stages);
        const uint32_t phase = (uint32_t)((k / n_stages) & 1);
        if (ok[p] && jj[p] != 0)  // K5: device-side negative sample
          item[p] = (IdT)fps_k5_negative(a, pp[p], jj[p], item[p]);
        float* up = a.user_sharded
                        ? fps_row_t<IdT>(a.user_tab, user[p])
                        : a.user_table + fps_user_slot<IdT>(user[p], a.user_div, a.user_shift) * (size_t)stride;
        float* vp = fps_row_t<IdT>(a.item_tab, item[p]);
        mbar_wait(&empty[stage], phase ^ 1u);  // slot free (credit available)
        RowMeta m;
        m.up = up; m.vp = vp; m.rating = rt[p]; m.valid = ok[p] ? 1 : 0;
        meta[stage * TILE_ROWS + lane] = m;
        const unsigned okmask = __ballot_sync(0xffffffffu, ok[p]);
        __syncwarp();
        if (lane == 0)
          mbar_arrive_expect_tx(&full[stage], (uint32_t)__popc(okmask) * 2u * row_bytes);
        __syncwarp();
        if (ok[p]) {
          float* su = rows + (size_t)stage * stage_floats + (size_t)lane * stride;
          float* sv = su + (size_t)TILE_ROWS * stride;
          tma_bulk_g2s(sv, vp, row_bytes, &full[stage]);  // the PULL (peer HBM over NVLink or local)
          tma_bulk_g2s(su, up, row_bytes, &full[stage]);
        }
      }
    }
  } else {
    // ============================== CONSUMERS (SGD + PUSH) ==============================
    const int cw = warp - N_PRODUCER_WARPS;
    constexpr int ROWS_PER_PASS = 32 / LPR;
    const int sub = lane / LPR;
    const int l = lane & (LPR - 1);
    float sq_acc = 0.f, cnt_acc = 0.f;
    bool bad = false;
    int stage = 0;
    uint32_t phase = 0;
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      mbar_wait(&full[stage], phase);
      const float* su = rows + (size_t)stage * stage_floats;
      const float* sv = su + (size_t)TILE_ROWS * stride;
      const RowMeta* mt = meta + stage * TILE_ROWS;
#pragma unroll 2
      for (int r0 = cw * ROWS_PER_PASS; r0 < TILE_ROWS; r0 += N_CONSUMER_WARPS * ROWS_PER_PASS) {
        const int r = r0 + sub;
        const RowMeta m = mt[r];
        float d = 0.f;
        if (m.valid) {
          for (int q = l; q < nvec; q += LPR) {
            const float4 u = *reinterpret_cast<const float4*>(su + (size_t)r * stride + 4 * q);
            const float4 v = *reinterpret_cast<const float4*>(sv + (size_t)r * stride + 4 * q);
            d += u.x * v.x + u.y * v.y + u.z * v.z + u.w * v.w;
          }
        }
        d = fps_group_sum<LPR>(d);
        const float resid = m.rating - d;
        const float e = (a.err_mode == 0)   ? 1.f / (1.f + __expf(-resid))
                        : (a.err_mode == 1) ? resid
                                            : m.rating - 1.f / (1.f + __expf(-d));
        const float g = a.lr * e;
        if (m.valid) {
          if (!(fabsf(g) <= 3.0e38f)) bad = true;
          if (l == 0) { sq_acc += resid * resid; cnt_acc += 1.f; }
          for (int q = l; q < nvec; q += LPR) {
            const float4 u = *reinterpret_cast<const float4*>(su + (size_t)r * stride + 4 * q);
            const float4 v = *reinterpret_cast<const float4*>(sv + (size_t)r * stride + 4 * q);
            fps_red_add4(m.up + 4 * q, make_float4(g * v.x, g * v.y, g * v.z, g * v.w));
            fps_red_add4(m.vp + 4 * q, make_float4(g * u.x, g * u.y, g * u.z, g * u.w));  // PUSH
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);  // release the credit
      if (++stage == n_stages) { stage = 0; phase ^= 1u; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sq_acc += __shfl_xor_sync(0xffffffffu, sq_acc, o);
      cnt_acc += __shfl_xor_sync(0xffffffffu, cnt_acc, o);
    }
    if (lane == 0 && a.stats != nullptr && cnt_acc > 0.f) {
      atomicAdd(a.stats + 0, sq_acc);
      atomicAdd(a.stats + 1, cnt_acc);
    }
    if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
  }
}

template <typename IdT, int LPR>
static int launch_tma(const MfArgs& a, int max_inflight_rows, int num_sms, cudaStream_t stream) {
  const int stride = a.item_tab.stride;
  const size_t stage_bytes = (size_t)2 * TILE_ROWS * stride * 4 + TILE_ROWS * sizeof(RowMeta) + 16;
  const size_t budget = 200 * 1024;
  int stages = (int)(budget / stage_bytes);
  if (stages > 16) stages = 16;
  if (max_inflight_rows > 0) {  // pull limiter: stages * 32 * grid <= pullLimit
    long long per_cta = max_inflight_rows / (long long)num_sms;
    int cap = (int)(per_cta / TILE_ROWS);
    if (cap < 2) cap = 2;
    if (stages > cap) stages = cap;
  }
  stages -= stages % N_PRODUCER_WARPS;
  if (stages < 2) return -1002;  // rows too large for the smem ring: caller falls back
  const size_t smem = (size_t)stages * stage_bytes + 64;
  auto kern = fps_mf_sgd_tma_kernel<IdT, LPR>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const long long n_eff = a.n_pos * (1 + a.neg_rate);
  long long n_tiles = (n_eff + TILE_ROWS - 1) / TILE_ROWS;
  long long grid = num_sms;
  if (max_inflight_rows > 0 && max_inflight_rows < (long long)num_sms * 2 * TILE_ROWS) {
    grid = max_inflight_rows / (2 * TILE_ROWS);
    if (grid < 1) grid = 1;
  }
  if (grid > n_tiles) grid = n_tiles;
  kern<<<(int)grid, TMA_THREADS, smem, stream>>>(a, stages);
  return (int)cudaGetLastError();
}

template <typename IdT>
static int dispatch_tma(const MfArgs& a, int max_inflight, int num_sms, cudaStream_t s) {
  const int nvec = a.item_tab.stride >> 2;
  if (nvec <= 1) return launch_tma<IdT, 1>(a, max_inflight, num_sms, s);
  if (nvec <= 2) return launch_tma<IdT, 2>(a, max_inflight, num_sms, s);
  if (nvec <= 4) return launch_tma<IdT, 4>(a, max_inflight, num_sms, s);
  if (nvec <= 8) return launch_tma<IdT, 8>(a, max_inflight, num_sms, s);
  if (nvec <= 16) return launch_tma<IdT, 16>(a, max_inflight, num_sms, s);
  return launch_tma<IdT, 32>(a, max_inflight, num_sms, s);
}

extern "C" int fps_mf_sgd_tma(const MfArgs* args, int id_bytes, int max_inflight_rows, int num_sms,
                              cudaStream_t stream) {
  if (args->n_pos <= 0) return 0;
  if (id_bytes == 4) return dispatch_tma<int>(*args, max_inflight_rows, num_sms, stream);
  if (id_bytes == 8) return dispatch_tma<long long>(*args, max_inflight_rows, num_sms, stream);
  return -1001;
}
