// fp64 variant of the fused matrix-factorisation step (pull + SGD + push), for a like-for-like row
// against the reference, whose vectors are Array[Double] (M/matrix/factorization/utils/Vector.scala:8).
//
// Rows hold k doubles; the ShardTable machinery is unchanged (stride is counted in 4-byte cells: 2 * k,
// rows stay 16-byte aligned).  LPR lanes cooperate on one row, each lane owning VPL double2 chunks:
// pull = ld.global.v2.f64 from the owner's HBM (local or NVLink peer), push = red.global.add.f64 (there is
// no vector form of the fp64 reduction), user update = local red.global.add.f64.  Same update rules as
// fps_core.cu (SGDUpdater.scala:5-14).  Twice the bytes per update of the fp32 kernel: it runs at about
// half its updates/s on the same memory system.
#include "fps_common.cuh"
#include "fps_mf_args.cuh"

__device__ __forceinline__ double2 fps_ld_row2d(const double* p) {
  double2 v;
  asm volatile("ld.global.v2.f64 {%0,%1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ void fps_red_add_d(double* p, double v) {
  asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}

template <typename IdT, int LPR, int VPL, int FMT>
__global__ void __launch_bounds__(256, 4) fps_mf_sgd_fused_f64_kernel(const __grid_constant__ MfArgs a) {
  const int lane = threadIdx.x & (LPR - 1);
  const long long group = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LPR;
  const long long n_groups = ((long long)gridDim.x * blockDim.x) / LPR;
  const int stride = a.item_tab.stride;          // 4-byte cells per row
  const int nvec = stride >> 2;                  // double2 chunks per row
  const IdT* __restrict__ users = reinterpret_cast<const IdT*>(a.users);
  const IdT* __restrict__ items = reinterpret_cast<const IdT*>(a.items);
  double sq_acc = 0.0;
  float cnt_acc = 0.f;
  bool bad = false;
  const long long n_round = ((a.n_pos + n_groups - 1) / n_groups) * n_groups;
  for (long long idx = group; idx < n_round; idx += n_groups) {
    const bool in = idx < a.n_pos;
    IdT user = 0, item = 0;
    double rating = 0.0;
    bool ok = in;
    if (in) {
      // not fps_record: with it nvcc contracts this kernel's dot u.x*v.x + u.y*v.y the other way round in some
      // instantiations (an fp64 rounding change)
      if (FMT == 1) {
        const unsigned long long rec = reinterpret_cast<const unsigned long long*>(a.users)[idx];
        user = (IdT)(rec >> FPS_REC_USER_SHIFT);
        item = (IdT)((rec >> FPS_REC_ITEM_SHIFT) & FPS_REC_ITEM_MASK);
        rating = (double)__half2float(__ushort_as_half((unsigned short)(rec & 0xFFFFull)));
      } else {
        user = users[idx];
        item = items[idx];
        rating = (double)a.ratings[idx];
        if (user < 0) ok = false;
      }
    }
    double* up = reinterpret_cast<double*>(a.user_table + fps_user_slot<IdT>(user, a.user_div, a.user_shift) * (size_t)stride);
    double* vp = reinterpret_cast<double*>(fps_row_t<IdT>(a.item_tab, item));
    double2 u[VPL], v[VPL];
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int q = lane + c * LPR;
      if (ok && q < nvec) {
        v[c] = fps_ld_row2d(vp + 2 * q);   // the PULL
        u[c] = *reinterpret_cast<const double2*>(up + 2 * q);
      } else {
        v[c] = make_double2(0.0, 0.0);
        u[c] = make_double2(0.0, 0.0);
      }
    }
    double d = 0.0;
#pragma unroll
    for (int c = 0; c < VPL; ++c) d += u[c].x * v[c].x + u[c].y * v[c].y;
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    const double resid = rating - d;
    const double e = (a.err_mode == 0) ? 1.0 / (1.0 + exp(-resid)) : (a.err_mode == 1) ? resid
                                                                                        : rating - 1.0 / (1.0 + exp(-d));
    const double g = (double)a.lr * e;
    if (ok) {
      if (!(fabs(g) <= 1.0e300)) bad = true;
      if (lane == 0) { sq_acc += resid * resid; cnt_acc += 1.f; }
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int q = lane + c * LPR;
        if (q < nvec) {
          fps_red_add_d(up + 2 * q, g * v[c].x);       // worker-local user update
          fps_red_add_d(up + 2 * q + 1, g * v[c].y);
          fps_red_add_d(vp + 2 * q, g * u[c].x);       // the PUSH, fused with paramUpdate
          fps_red_add_d(vp + 2 * q + 1, g * u[c].y);
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sq_acc += __shfl_xor_sync(0xffffffffu, sq_acc, o);
    cnt_acc += __shfl_xor_sync(0xffffffffu, cnt_acc, o);
  }
  if ((threadIdx.x & 31) == 0 && a.stats != nullptr && cnt_acc > 0.f) {
    atomicAdd(a.stats + 0, (float)sq_acc);
    atomicAdd(a.stats + 1, cnt_acc);
  }
  if (bad && a.nan_flag != nullptr) *a.nan_flag = 1;
}

// No reserve and no pull limit: the fp64 step runs alone.
template <typename IdT, int LPR, int VPL, int FMT>
static int launch_f64(const MfArgs& a, int num_sms, cudaStream_t stream) {
  const long long blocks = fps_row_grid(fps_mf_sgd_fused_f64_kernel<IdT, LPR, VPL, FMT>, 256, 256 / LPR, num_sms, 0, 0,
                                        1, a.n_pos, 1);
  fps_mf_sgd_fused_f64_kernel<IdT, LPR, VPL, FMT><<<(int)blocks, 256, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

template <typename IdT, int FMT>
static int dispatch_f64(const MfArgs& a, int num_sms, cudaStream_t s) {
  const int nvec = a.item_tab.stride >> 2;   // double2 chunks
  if (nvec <= 4) return launch_f64<IdT, 4, 1, FMT>(a, num_sms, s);
  if (nvec <= 8) return launch_f64<IdT, 8, 1, FMT>(a, num_sms, s);
  if (nvec <= 16) return launch_f64<IdT, 16, 1, FMT>(a, num_sms, s);
  if (nvec <= 32) return launch_f64<IdT, 32, 1, FMT>(a, num_sms, s);
  if (nvec <= 64) return launch_f64<IdT, 32, 2, FMT>(a, num_sms, s);
  if (nvec <= 128) return launch_f64<IdT, 32, 4, FMT>(a, num_sms, s);
  return -1000;
}

// MfArgs as for fps_mf_sgd_fused, with every row (user_table, item_tab shards) holding doubles; negative
// sampling, output stream and the credit counter are fp32-kernel features and must be off.
extern "C" int fps_mf_sgd_fused_f64(const MfArgs* args, int id_bytes, int num_sms, cudaStream_t stream) {
  if (args->n_pos <= 0) return 0;
  if (args->neg_rate != 0 || args->user_sharded || args->use_push_tab || args->out_every > 0 || args->credits != nullptr)
    return -1004;
  return fps_with_id_form(args->format, id_bytes, [&](auto form) {
    using F = decltype(form);
    return dispatch_f64<typename F::Id, F::fmt>(*args, num_sms, stream);
  });
}

// K4 for fp64 rows: value(id, j) = lo + (hi - lo) * u53(philox(id, j / 2; seed)[2 * (j % 2) .. +1])
__global__ void fps_init_rows_f64_kernel(double* __restrict__ rows, long long n_rows, int dim, int stride_d,
                                         int shard, int num_shards, int mode, long long div,
                                         unsigned long long seed, double lo, double hi) {
  const int npair = stride_d >> 1;
  const long long total = n_rows * npair;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const long long slot = t / npair;
    const int q = (int)(t - slot * npair);
    const long long id = (mode == FPS_PART_HASH) ? slot * num_shards + shard : (long long)shard * div + slot;
    Philox4 r = fps_philox((uint32_t)id, (uint32_t)((unsigned long long)id >> 32), (uint32_t)q, 1u,
                           (uint32_t)seed, (uint32_t)(seed >> 32));
    const double sc = hi - lo;
    const double u0 = (double)((((unsigned long long)r.x << 32) | r.y) >> 11) * (1.0 / 9007199254740992.0);
    const double u1 = (double)((((unsigned long long)r.z << 32) | r.w) >> 11) * (1.0 / 9007199254740992.0);
    double2 v;
    v.x = (2 * q + 0 < dim) ? lo + sc * u0 : 0.0;
    v.y = (2 * q + 1 < dim) ? lo + sc * u1 : 0.0;
    *reinterpret_cast<double2*>(rows + slot * (long long)stride_d + 2 * q) = v;
  }
}

extern "C" int fps_init_rows_f64(double* rows, long long n_rows, int dim, int stride_d, int shard,
                                 int num_shards, int mode, long long div, unsigned long long seed, double lo,
                                 double hi, cudaStream_t stream) {
  if (n_rows <= 0) return 0;
  long long total = n_rows * (stride_d / 2);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;  // 32 CTAs per H100 SM, grid-stride beyond
  fps_init_rows_f64_kernel<<<(int)blocks, 256, 0, stream>>>(rows, n_rows, dim, stride_d, shard, num_shards, mode,
                                                            div, seed, lo, hi);
  return (int)cudaGetLastError();
}
