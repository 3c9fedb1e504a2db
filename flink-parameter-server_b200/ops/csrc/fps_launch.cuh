// Host-side launch helpers shared by the fused row kernels: the id-form dispatch of the MF entry points and the
// grid sizing of the occupancy-sized launchers (fps_core.cu, fps_mf_bpr.cu, fps_mf_warp.cu, fps_mf_f64.cu,
// fps_w2v_window.cu).
#pragma once
#include <cuda_runtime.h>

// Calls f(FpsIdForm<IdT, FMT>{}) for the record form of a batch: packed64 records (ids decoded as int) or
// arrays of 4- or 8-byte ids.  -1001: any other id width.
template <typename IdT, int FMT>
struct FpsIdForm {
  using Id = IdT;
  static constexpr int fmt = FMT;
};
template <typename F>
static inline int fps_with_id_form(int format, int id_bytes, F&& f) {
  if (format == 1) return f(FpsIdForm<int, 1>{});
  if (id_bytes == 4) return f(FpsIdForm<int, 0>{});
  if (id_bytes == 8) return f(FpsIdForm<long long, 0>{});
  return -1001;
}

// Grid of a fused row kernel with `groups_per_block` lane-groups per CTA of `threads` threads:
// - every CTA slot the occupancy allows, less `reserve_total` slots left free for the replica exchange that runs
//   next to it, and at least one CTA per SM;
// - with a static pull limit (max_inflight_rows > 0), at most max_inflight_rows rows in flight, a lane-group
//   holding `rows_per_group`;
// - no more CTAs than `work` records fill, a lane-group taking `records_per_group` per round.
template <typename Kernel>
static inline long long fps_row_grid(Kernel kern, int threads, int groups_per_block, int num_sms, int reserve_total,
                                     int max_inflight_rows, int rows_per_group, long long work,
                                     int records_per_group) {
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, 0);
  if (occ < 1) occ = 1;
  long long blocks = (long long)num_sms * occ - reserve_total;
  if (blocks < num_sms) blocks = num_sms;
  if (max_inflight_rows > 0) {
    long long cap = max_inflight_rows / ((long long)rows_per_group * groups_per_block);
    if (cap < 1) cap = 1;
    if (blocks > cap) blocks = cap;
  }
  const long long per_block = (long long)groups_per_block * records_per_group;
  long long need = (work + per_block - 1) / per_block;
  if (need < 1) need = 1;
  if (blocks > need) blocks = need;
  return blocks;
}
