// K6: pull (query vectors from the PS shards over NVLink) fused with a wgmma GEMM against the
// worker-local item table and a top-K candidate-filter epilogue.  sm_90a (Hopper).
//
//   scores[q, i] = <query[q, :], item[i, :]>        (TF32 tensor-core MMA, FP32 accumulate in registers)
//
//   A operand (queries, 128 rows per query block): gathered ONCE per CTA from the owning PS shards with
//       16-byte peer loads and written into shared memory in the canonical K-major SWIZZLE_128B layout
//       (manual XOR swizzle), then published to the async proxy with fence.proxy.async.
//   B operand (items): streamed by TMA (cp.async.bulk.tensor.2d, SASS UTMALDG) through a 2..4-stage
//       mbarrier ring by one producer warp, hardware-swizzled by the tensor map.
//   MMA: 2 * MB consumer warpgroups of 64 query rows issue wgmma.m64n128k8 TF32 from smem descriptors
//       into register accumulators; a retired stage is released before the epilogue (TMA overlaps it).
//   Epilogue (wgmma fragment: each thread holds 32 columns of 2 rows, 4 lanes share a row):
//       mode 0: write raw scores                    (small problems / validation)
//       mode 1: per-(row, tile) maximum             (pass 1: gives an exact top-K lower bound theta)
//       mode 2: append (score, item) >= theta[row]  (pass 2: exact candidate set, usually << N)
//
// Exactness: theta[row] = K-th largest tile-maximum of pass 1 is attained by K distinct items, so the
// true K-th best score >= theta and pass 2 (bitwise identical scores) keeps every top-K item.
// This replaces the pointer-chasing LEMP scan (PSTopKGeneratorWorker.scala:49-113) with tile-level
// pruning that is validated against brute force (tests/test_gpu_topk.py).
//
// Two mainloops share the interface (modes, TopkArgs, tile dealing, candidate segments):
//   fps_topk_mma_kernel       stride <= 128 (KB <= 4): a whole item tile (KB K blocks) per ring stage.
//   fps_topk_mma_wide_kernel  128 < stride <= 512 (5 <= KB <= 16): the queries stay resident, the
//       items stream one 128-item x 32-float K block per ring stage (see the comment of that kernel).
//       The K blocks of a tile are accumulated in a fixed order (kb = 0, 1, ..., KB-1, each as 4
//       wgmma k8 steps) by the same instruction sequence in every mode, so pass 1 and pass 2 agree
//       bit for bit and the theta argument above holds unchanged.
#include <cuda.h>
#include "fps_common.cuh"

#define TK_M 128          // query rows per query block (two wgmma M=64 warpgroups)
#define TK_N 128          // items per tile (wgmma N)
#define TK_KB_FLOATS 32   // floats per 128-byte swizzle atom row
#define TK_MAX_STAGES 4
#define TK_MAX_KB 4       // whole-tile stages: A block + >= 2 tile stages fit in 227 KB of smem
#define TK_WIDE_MAX_KB 16       // K-streamed kernel: stride <= 512
#define TK_WIDE_M128_MAX_KB 10  // 128 query rows while KB x 16 KB of A leaves >= 3 stages; 64 above
#define TK_WIDE_MAX_STAGES 16
#define TK_WIDE_MIN_STAGES 3

struct TopkArgs {
  const void* q_ids;        // [n_queries] ids of the query vectors in q_tab (null -> q_local)
  const float* q_local;     // [n_queries, stride] already-local queries (used when q_ids == null)
  ShardTable q_tab;         // PS table of the query vectors (users)
  int n_queries;
  int n_items;              // rows of the local item table
  int stride;               // floats per row (multiple of 4)
  int n_tiles;              // ceil(n_items / TK_N)
  int tiles_per_split;
  int n_splits;
  int mode;
  int n_stages;             // B-operand ring depth (2..4, from the smem budget)
  float* out_scores;        // mode 0: [n_queries, out_ld]
  long long out_ld;
  float* tile_max;          // mode 1: [n_queries, n_tiles]
  const float* theta;       // mode 2: [n_queries]
  int* cand_count;          // mode 2: [n_queries, n_splits] candidates found by each split (may exceed seg_cap)
  float* cand_score;        // mode 2: [n_queries, cand_cap], split s owns columns [s*seg_cap, (s+1)*seg_cap)
  int* cand_item;           // mode 2: [n_queries, cand_cap]
  int cand_cap;
  int seg_cap;              // cand_cap / n_splits (set by the launcher)
  int tile_lo;              // first tile to score
  int pad_;
  const int* tile_limit;    // optional device scalar: score only tiles < min(n_tiles, *tile_limit)
                            // (length-pruning bound computed on the device, no host round trip)
};

__device__ __forceinline__ uint32_t tk_smem(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void tk_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(tk_smem(bar)), "r"(count));
}
__device__ __forceinline__ void tk_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tk_smem(bar)) : "memory");
}
__device__ __forceinline__ void tk_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tk_smem(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tk_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "TK_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra TK_DONE;\n"
      "bra TK_WAIT;\n"
      "TK_DONE:\n"
      "}\n" ::"r"(tk_smem(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tk_tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1,
                                               uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(tk_smem(dst)),
      "l"(map), "r"(tk_smem(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA descriptor): start address,
// leading byte offset (unused by swizzled K-major layouts), stride byte offset = 8 rows * 128 B,
// layout type 1 = SWIZZLE_128B.  Every operand block starts 1024-byte aligned (base offset 0).
__device__ __forceinline__ uint64_t tk_desc(uint32_t smem_addr) {
  uint64_t d = (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// d[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T, both K-major in shared memory; scale_d == 0 overwrites d.
__device__ __forceinline__ void tk_wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}

// MB = number of 128-row query blocks per CTA.  With MB = 2 every item tile fetched by TMA feeds four
// 64-row warpgroups (256 query rows), which halves the L2 -> SM item traffic per FLOP.
// Warps 0 .. 8*MB-1 are the consumer warpgroups, warp 8*MB is the TMA producer.
template <typename IdT, int MODE, int MB>
__global__ void __launch_bounds__(256 * MB + 32, 1)
    fps_topk_mma_kernel(const __grid_constant__ CUtensorMap item_map,
                        const __grid_constant__ TopkArgs a) {
  extern __shared__ __align__(1024) unsigned char tk_smem_raw[];
  const int KB = (a.stride + TK_KB_FLOATS - 1) / TK_KB_FLOATS;  // 128-byte K blocks
  const uint32_t kb_bytes = TK_M * 128;                         // one K block of a 128-row tile
  // SWIZZLE_128B operands start 1024-byte aligned (the launcher adds 1 KB of slack for this)
  unsigned char* sA = tk_smem_raw + ((1024u - (tk_smem(tk_smem_raw) & 1023u)) & 1023u);  // [MB][KB][128][128 B]
  unsigned char* sB = sA + (size_t)MB * KB * kb_bytes;          // [STAGES][KB][128 rows][128 B]
  const int NS = a.n_stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + (size_t)NS * KB * kb_bytes);
  uint64_t* full = bars;                      // [STAGES] TMA -> MMA
  uint64_t* empty = bars + TK_MAX_STAGES;     // [STAGES] MMA -> TMA (one arrive per consumer warp)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qb = blockIdx.x / a.n_splits;
  const int split = blockIdx.x - qb * a.n_splits;
  // tiles are dealt round-robin to the splits (tile = tile_lo + split + i * n_splits): a device-side
  // tile limit or a hot region of the table (length-sorted items) then stays balanced over the CTAs
  int tiles_hi = a.n_tiles;
  if (a.tile_limit != nullptr) tiles_hi = min(tiles_hi, *a.tile_limit);
  const int first_tile = a.tile_lo + split;
  const int my_tiles = first_tile < tiles_hi ? (tiles_hi - first_tile + a.n_splits - 1) / a.n_splits : 0;
  const int row0 = qb * TK_M * MB;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      tk_mbar_init(&full[s], 1);
      tk_mbar_init(&empty[s], 8 * MB);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }

  // ---- A operand: pull the query rows (peer loads) into swizzled smem ------------------------
  {
    const IdT* qids = reinterpret_cast<const IdT*>(a.q_ids);
    const int nvec = a.stride >> 2;
    const int chunks_per_row = KB * 8;
    for (int t = threadIdx.x; t < MB * TK_M * chunks_per_row; t += blockDim.x) {
      const int r = t / chunks_per_row;
      const int cc = t - r * chunks_per_row;  // 16-byte chunk index along K
      const int kb = cc >> 3, c = cc & 7;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      const int row = row0 + r;
      if (row < a.n_queries && cc < nvec) {
        const float* src = (qids != nullptr) ? fps_row_t<IdT>(a.q_tab, qids[row])
                                             : a.q_local + (size_t)row * a.stride;
        v = fps_ld_row4(src + 4 * cc);  // the PULL (local HBM or NVLink peer)
      }
      const int mb = r >> 7, rr = r & 127;
      unsigned char* dst = sA + ((size_t)mb * KB + kb) * kb_bytes + (size_t)rr * 128 + ((c ^ (rr & 7)) << 4);
      *reinterpret_cast<float4*>(dst) = v;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes -> async proxy
  }
  __syncthreads();

  if (warp == 8 * MB) {
    // =============================== TMA producer (items) ===============================
    if (lane == 0) {
      for (int i = 0; i < my_tiles; ++i) {
        const int s = i % NS;
        const uint32_t ph = (uint32_t)((i / NS) & 1);
        tk_mbar_wait(&empty[s], ph ^ 1u);
        tk_mbar_expect_tx(&full[s], (uint32_t)KB * kb_bytes);
        const int item0 = (first_tile + i * a.n_splits) * TK_N;
        for (int kb = 0; kb < KB; ++kb)
          tk_tma_load_2d(sB + ((size_t)s * KB + kb) * kb_bytes, &item_map, kb * TK_KB_FLOATS, item0,
                         &full[s]);
      }
    }
    return;
  }

  // =============================== MMA + epilogue (consumer warpgroups) ===============================
  const int wg = warp >> 2;                 // consumer warpgroup: 64 query rows
  const int emb = wg >> 1;                  // which 128-row query block (A operand block)
  const int half = wg & 1;                  // which 64-row half of it
  // fragment of m64nNk8 with f32 accumulators: d[i] is (row rq + 8 * ((i >> 1) & 1),
  // column 8 * (i >> 2) + 2 * (lane & 3) + (i & 1)) of the warpgroup's 64 x 128 tile
  const int rq = emb * TK_M + half * 64 + (warp & 3) * 16 + (lane >> 2);
  const int rowA = row0 + rq, rowB = rowA + 8;
  const bool okA = rowA < a.n_queries, okB = rowB < a.n_queries;
  const int col0 = 2 * (lane & 3);
  const float thA = (MODE == 2 && okA) ? a.theta[rowA] : 0.f;
  const float thB = (MODE == 2 && okB) ? a.theta[rowB] : 0.f;
  int candA = 0, candB = 0;                 // per-(row, split) cursor, identical in the row's 4 lanes
  const uint32_t a_base = tk_smem(sA + (size_t)emb * KB * kb_bytes + (size_t)half * 64 * 128);
  float d[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) d[j] = 0.f;

  for (int i = 0; i < my_tiles; ++i) {
    const int s = i % NS;
    const uint32_t ph = (uint32_t)((i / NS) & 1);
    const int tile = first_tile + i * a.n_splits;
    const int item0 = tile * TK_N;
    const bool full_tile = item0 + TK_N <= a.n_items;   // no per-element bound check needed
    tk_mbar_wait(&full[s], ph);                         // TMA landed the item tile
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
    const uint32_t b_base = tk_smem(sB + (size_t)s * KB * kb_bytes);
#pragma unroll 1
    for (int kb = 0; kb < KB; ++kb) {
#pragma unroll
      for (int k = 0; k < 4; ++k)  // wgmma K = 8 tf32 = 32 bytes inside the 128-byte atom
        tk_wgmma_tf32(d, tk_desc(a_base + kb * kb_bytes + k * 32), tk_desc(b_base + kb * kb_bytes + k * 32),
                      (kb | k) != 0 ? 1u : 0u);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    __syncwarp();
    if (lane == 0) tk_mbar_arrive(&empty[s]);           // smem stage reusable: the MMAs have read it

    if (MODE == 1) {
      float mA = -3.0e38f, mB = -3.0e38f;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
        if (full_tile || item < a.n_items) {
          if ((j >> 1) & 1) mB = fmaxf(mB, d[j]); else mA = fmaxf(mA, d[j]);
        }
      }
      mA = fmaxf(mA, __shfl_xor_sync(0xffffffffu, mA, 1));
      mA = fmaxf(mA, __shfl_xor_sync(0xffffffffu, mA, 2));
      mB = fmaxf(mB, __shfl_xor_sync(0xffffffffu, mB, 1));
      mB = fmaxf(mB, __shfl_xor_sync(0xffffffffu, mB, 2));
      if ((lane & 3) == 0) {
        if (okA) a.tile_max[(size_t)rowA * a.n_tiles + tile] = mA;
        if (okB) a.tile_max[(size_t)rowB * a.n_tiles + tile] = mB;
      }
    } else if (MODE == 2) {
      // candidates are rare: first a branch-free "any >= theta" test over the thread's 64 values; the
      // warp walks the append path only when one of its rows reached theta.  Each (row, split) owns a
      // private segment of the row's buffer and a register cursor shared by the row's 4 lanes: no
      // atomics (a returning atomic per candidate made pass 2 latency bound).
      float mA = -3.0e38f, mB = -3.0e38f;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        if ((j >> 1) & 1) mB = fmaxf(mB, d[j]); else mA = fmaxf(mA, d[j]);
      }
      const bool hit = (okA && mA >= thA) || (okB && mB >= thB);
      if (__any_sync(0xffffffffu, hit)) {
        int nA = 0, nB = 0;
#pragma unroll
        for (int j = 0; j < 64; ++j) {
          const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
          const bool in = full_tile || item < a.n_items;
          if ((j >> 1) & 1) nB += (okB && in && d[j] >= thB) ? 1 : 0;
          else nA += (okA && in && d[j] >= thA) ? 1 : 0;
        }
        // exclusive prefix of the counts over the row's 4 lanes (lane & 3 = 0..3)
        int pA = nA, pB = nB;
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          const int tA = __shfl_up_sync(0xffffffffu, pA, o, 4);
          const int tB = __shfl_up_sync(0xffffffffu, pB, o, 4);
          if ((lane & 3) >= o) { pA += tA; pB += tB; }
        }
        const int totA = __shfl_sync(0xffffffffu, pA, 3, 4);
        const int totB = __shfl_sync(0xffffffffu, pB, 3, 4);
        int wA = candA + pA - nA, wB = candB + pB - nB;
        if (nA + nB > 0) {
          float* sA_ = okA ? a.cand_score + (size_t)rowA * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
          int* iA_ = okA ? a.cand_item + (size_t)rowA * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
          float* sB_ = okB ? a.cand_score + (size_t)rowB * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
          int* iB_ = okB ? a.cand_item + (size_t)rowB * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
#pragma unroll
          for (int j = 0; j < 64; ++j) {
            const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
            const bool in = full_tile || item < a.n_items;
            if ((j >> 1) & 1) {
              if (okB && in && d[j] >= thB) {
                if (wB < a.seg_cap) { sB_[wB] = d[j]; iB_[wB] = item; }
                ++wB;
              }
            } else if (okA && in && d[j] >= thA) {
              if (wA < a.seg_cap) { sA_[wA] = d[j]; iA_[wA] = item; }
              ++wA;
            }
          }
        }
        candA += totA;
        candB += totB;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
        const bool rB = (j >> 1) & 1;
        if ((rB ? okB : okA) && (full_tile || item < a.n_items))
          a.out_scores[(size_t)(rB ? rowB : rowA) * a.out_ld + item] = d[j];
      }
    }
  }
  if (MODE == 2 && (lane & 3) == 0) {
    if (okA) a.cand_count[(size_t)rowA * a.n_splits + split] = candA;
    if (okB) a.cand_count[(size_t)rowB * a.n_splits + split] = candB;
  }
}

// K-streamed variant for 128 < stride <= 512 (KB = 5 .. 16 K blocks of 32 floats).
//   A (queries): resident, gathered once per CTA exactly as above; MW 64-row consumer warpgroups, so
//       KB x MW x 8 KB of shared memory (MW = 2 up to KB = 10, MW = 1 above).
//   B (items): the ring holds single K blocks (128 items x 128 B = 16 KB, one TMA box); a tile is KB
//       consecutive chunks of the stream, so the ring depth is independent of the width (>= 3).
//   MMA: per chunk 4 x wgmma m64n128k8 into the tile's accumulators, commit, wait_group 1: the chunk
//       before it has retired and its stage goes back to the producer while this one runs.  After the
//       last chunk of a tile wait_group 0, release, epilogue.
// The epilogue is a copy of fps_topk_mma_kernel's (rows of one 64 * MW block), kept separate so the
// code generation of the narrow kernel does not depend on this one.
// Warps 0 .. 4*MW-1 are the consumer warpgroups, warp 4*MW is the TMA producer.
template <typename IdT, int MODE, int MW>
__global__ void __launch_bounds__(128 * MW + 32, 1)
    fps_topk_mma_wide_kernel(const __grid_constant__ CUtensorMap item_map,
                             const __grid_constant__ TopkArgs a) {
  constexpr int RQ = 64 * MW;                                   // query rows per CTA
  extern __shared__ __align__(1024) unsigned char tk_smem_raw[];
  const int KB = (a.stride + TK_KB_FLOATS - 1) / TK_KB_FLOATS;
  const uint32_t a_kb_bytes = RQ * 128;                         // one K block of the query block
  const uint32_t b_bytes = TK_N * 128;                          // one K block of an item tile
  unsigned char* sA = tk_smem_raw + ((1024u - (tk_smem(tk_smem_raw) & 1023u)) & 1023u);  // [KB][RQ][128 B]
  unsigned char* sB = sA + (size_t)KB * a_kb_bytes;             // [STAGES][128 rows][128 B]
  const int NS = a.n_stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + (size_t)NS * b_bytes);
  uint64_t* full = bars;                         // [STAGES] TMA -> MMA
  uint64_t* empty = bars + TK_WIDE_MAX_STAGES;   // [STAGES] MMA -> TMA (one arrive per consumer warp)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qb = blockIdx.x / a.n_splits;
  const int split = blockIdx.x - qb * a.n_splits;
  int tiles_hi = a.n_tiles;
  if (a.tile_limit != nullptr) tiles_hi = min(tiles_hi, *a.tile_limit);
  const int first_tile = a.tile_lo + split;
  const int my_tiles = first_tile < tiles_hi ? (tiles_hi - first_tile + a.n_splits - 1) / a.n_splits : 0;
  const int row0 = qb * RQ;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      tk_mbar_init(&full[s], 1);
      tk_mbar_init(&empty[s], 4 * MW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }

  // ---- A operand: pull the query rows (peer loads) into swizzled smem ------------------------
  {
    const IdT* qids = reinterpret_cast<const IdT*>(a.q_ids);
    const int nvec = a.stride >> 2;
    const int chunks_per_row = KB * 8;
    for (int t = threadIdx.x; t < RQ * chunks_per_row; t += blockDim.x) {
      const int r = t / chunks_per_row;
      const int cc = t - r * chunks_per_row;  // 16-byte chunk index along K
      const int kb = cc >> 3, c = cc & 7;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      const int row = row0 + r;
      if (row < a.n_queries && cc < nvec) {
        const float* src = (qids != nullptr) ? fps_row_t<IdT>(a.q_tab, qids[row])
                                             : a.q_local + (size_t)row * a.stride;
        v = fps_ld_row4(src + 4 * cc);  // the PULL (local HBM or NVLink peer)
      }
      unsigned char* dst = sA + (size_t)kb * a_kb_bytes + (size_t)r * 128 + ((c ^ (r & 7)) << 4);
      *reinterpret_cast<float4*>(dst) = v;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes -> async proxy
  }
  __syncthreads();

  if (warp == 4 * MW) {
    // =============================== TMA producer (item K blocks) ===============================
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int i = 0; i < my_tiles; ++i) {
        const int item0 = (first_tile + i * a.n_splits) * TK_N;
        for (int kb = 0; kb < KB; ++kb) {
          tk_mbar_wait(&empty[s], ph ^ 1u);
          tk_mbar_expect_tx(&full[s], b_bytes);
          tk_tma_load_2d(sB + (size_t)s * b_bytes, &item_map, kb * TK_KB_FLOATS, item0, &full[s]);
          if (++s == NS) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // =============================== MMA + epilogue (consumer warpgroups) ===============================
  const int wg = warp >> 2;                 // consumer warpgroup: 64 query rows
  const int rq = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int rowA = row0 + rq, rowB = rowA + 8;
  const bool okA = rowA < a.n_queries, okB = rowB < a.n_queries;
  const int col0 = 2 * (lane & 3);
  const float thA = (MODE == 2 && okA) ? a.theta[rowA] : 0.f;
  const float thB = (MODE == 2 && okB) ? a.theta[rowB] : 0.f;
  int candA = 0, candB = 0;                 // per-(row, split) cursor, identical in the row's 4 lanes
  const uint32_t a_base = tk_smem(sA + (size_t)wg * 64 * 128);
  const uint32_t b_base = tk_smem(sB);
  float d[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) d[j] = 0.f;

  int s = 0, prev = 0;                      // ring stage of the current / previous chunk
  uint32_t ph = 0;
  for (int i = 0; i < my_tiles; ++i) {
    const int tile = first_tile + i * a.n_splits;
    const int item0 = tile * TK_N;
    const bool full_tile = item0 + TK_N <= a.n_items;   // no per-element bound check needed
#pragma unroll 1
    for (int kb = 0; kb < KB; ++kb) {
      tk_mbar_wait(&full[s], ph);                       // TMA landed this K block of the tile
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int k = 0; k < 4; ++k)  // wgmma K = 8 tf32 = 32 bytes inside the 128-byte atom
        tk_wgmma_tf32(d, tk_desc(a_base + kb * a_kb_bytes + k * 32), tk_desc(b_base + s * b_bytes + k * 32),
                      (kb | k) != 0 ? 1u : 0u);
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
      // the previous chunk's wgmma group has retired: its stage may be refilled
      if (kb > 0) {
        __syncwarp();
        if (lane == 0) tk_mbar_arrive(&empty[prev]);
      }
      prev = s;
      if (++s == NS) { s = 0; ph ^= 1u; }
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    __syncwarp();
    if (lane == 0) tk_mbar_arrive(&empty[prev]);        // last chunk of the tile

    if (MODE == 1) {
      float mA = -3.0e38f, mB = -3.0e38f;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
        if (full_tile || item < a.n_items) {
          if ((j >> 1) & 1) mB = fmaxf(mB, d[j]); else mA = fmaxf(mA, d[j]);
        }
      }
      mA = fmaxf(mA, __shfl_xor_sync(0xffffffffu, mA, 1));
      mA = fmaxf(mA, __shfl_xor_sync(0xffffffffu, mA, 2));
      mB = fmaxf(mB, __shfl_xor_sync(0xffffffffu, mB, 1));
      mB = fmaxf(mB, __shfl_xor_sync(0xffffffffu, mB, 2));
      if ((lane & 3) == 0) {
        if (okA) a.tile_max[(size_t)rowA * a.n_tiles + tile] = mA;
        if (okB) a.tile_max[(size_t)rowB * a.n_tiles + tile] = mB;
      }
    } else if (MODE == 2) {
      float mA = -3.0e38f, mB = -3.0e38f;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        if ((j >> 1) & 1) mB = fmaxf(mB, d[j]); else mA = fmaxf(mA, d[j]);
      }
      const bool hit = (okA && mA >= thA) || (okB && mB >= thB);
      if (__any_sync(0xffffffffu, hit)) {
        int nA = 0, nB = 0;
#pragma unroll
        for (int j = 0; j < 64; ++j) {
          const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
          const bool in = full_tile || item < a.n_items;
          if ((j >> 1) & 1) nB += (okB && in && d[j] >= thB) ? 1 : 0;
          else nA += (okA && in && d[j] >= thA) ? 1 : 0;
        }
        int pA = nA, pB = nB;
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          const int tA = __shfl_up_sync(0xffffffffu, pA, o, 4);
          const int tB = __shfl_up_sync(0xffffffffu, pB, o, 4);
          if ((lane & 3) >= o) { pA += tA; pB += tB; }
        }
        const int totA = __shfl_sync(0xffffffffu, pA, 3, 4);
        const int totB = __shfl_sync(0xffffffffu, pB, 3, 4);
        int wA = candA + pA - nA, wB = candB + pB - nB;
        if (nA + nB > 0) {
          float* sA_ = okA ? a.cand_score + (size_t)rowA * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
          int* iA_ = okA ? a.cand_item + (size_t)rowA * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
          float* sB_ = okB ? a.cand_score + (size_t)rowB * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
          int* iB_ = okB ? a.cand_item + (size_t)rowB * a.cand_cap + (size_t)split * a.seg_cap : nullptr;
#pragma unroll
          for (int j = 0; j < 64; ++j) {
            const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
            const bool in = full_tile || item < a.n_items;
            if ((j >> 1) & 1) {
              if (okB && in && d[j] >= thB) {
                if (wB < a.seg_cap) { sB_[wB] = d[j]; iB_[wB] = item; }
                ++wB;
              }
            } else if (okA && in && d[j] >= thA) {
              if (wA < a.seg_cap) { sA_[wA] = d[j]; iA_[wA] = item; }
              ++wA;
            }
          }
        }
        candA += totA;
        candB += totB;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int item = item0 + 8 * (j >> 2) + col0 + (j & 1);
        const bool rB = (j >> 1) & 1;
        if ((rB ? okB : okA) && (full_tile || item < a.n_items))
          a.out_scores[(size_t)(rB ? rowB : rowA) * a.out_ld + item] = d[j];
      }
    }
  }
  if (MODE == 2 && (lane & 3) == 0) {
    if (okA) a.cand_count[(size_t)rowA * a.n_splits + split] = candA;
    if (okB) a.cand_count[(size_t)rowB * a.n_splits + split] = candB;
  }
}

// ---- host side ---------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

extern "C" int fps_topk_mma(TopkArgs* args_in, const float* item_table, int id_bytes,
                            int num_sms, cudaStream_t stream) {
  TopkArgs a = *args_in;
  if (a.n_queries <= 0 || a.n_items <= 0) return 0;
  const int KB = (a.stride + TK_KB_FLOATS - 1) / TK_KB_FLOATS;
  if (KB > TK_WIDE_MAX_KB) return -1003;
  const bool wide = KB > TK_MAX_KB;
  PFN_encodeTiled enc = get_encode();
  if (enc == nullptr) return -1004;
  CUtensorMap map;
  cuuint64_t gdim[2] = {(cuuint64_t)a.stride, (cuuint64_t)a.n_items};
  cuuint64_t gstr[1] = {(cuuint64_t)a.stride * 4};
  cuuint32_t box[2] = {TK_KB_FLOATS, TK_N};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)item_table, gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return -1005;
  a.n_tiles = (a.n_items + TK_N - 1) / TK_N;
  const int MBv = (a.n_queries > TK_M && KB <= 2) ? 2 : 1;   // 2 query blocks per CTA when smem allows
  // K-streamed kernel: 64-row warpgroups per CTA (2 while the resident A operand leaves >= 3 stages)
  const int MWv = KB <= TK_WIDE_M128_MAX_KB ? 2 : 1;
  const int rows_per_cta = wide ? 64 * MWv : TK_M * MBv;
  const int qblocks = (a.n_queries + rows_per_cta - 1) / rows_per_cta;
  int splits = num_sms / qblocks;  // one wave of CTAs (1 CTA/SM: smem bound), no tail wave
  int span = a.n_tiles - a.tile_lo;  // tiles that may be scored (a device tile_limit can only lower it)
  if (span < 1) span = 1;
  if (splits > span) splits = span;
  if (splits < 1) splits = 1;
  a.tiles_per_split = (span + splits - 1) / splits;
  a.n_splits = (span + a.tiles_per_split - 1) / a.tiles_per_split;
  a.seg_cap = a.cand_cap / a.n_splits;
  args_in->n_splits = a.n_splits;   // the caller sizes cand_count [n_queries, n_splits] from these
  args_in->seg_cap = a.seg_cap;
  args_in->n_tiles = a.n_tiles;
  if (a.mode < 0) return 0;         // geometry query only
  if (a.mode == 2 && a.seg_cap < 1) return -1006;
  if (wide) {
    const size_t a_bytes = (size_t)KB * 64 * MWv * 128, b_bytes = (size_t)TK_N * 128;
    int wstages = (int)((220 * 1024 - a_bytes - 2048) / b_bytes);
    if (wstages > TK_WIDE_MAX_STAGES) wstages = TK_WIDE_MAX_STAGES;
    if (wstages < TK_WIDE_MIN_STAGES) return -1003;
    a.n_stages = wstages;
    const size_t wsmem = a_bytes + b_bytes * wstages + 2 * TK_WIDE_MAX_STAGES * 8 + 1024;
    const int wgrid = qblocks * a.n_splits;
#define TK_WLAUNCH2(IDT, MODE, MWT)                                                                \
  do {                                                                                             \
    cudaError_t e = cudaFuncSetAttribute(fps_topk_mma_wide_kernel<IDT, MODE, MWT>,                 \
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem); \
    if (e != cudaSuccess) return (int)e;                                                           \
    fps_topk_mma_wide_kernel<IDT, MODE, MWT><<<wgrid, 128 * MWT + 32, wsmem, stream>>>(map, a);    \
  } while (0)
#define TK_WLAUNCH(IDT, MODE)                                                                      \
  do {                                                                                             \
    if (MWv == 2) TK_WLAUNCH2(IDT, MODE, 2); else TK_WLAUNCH2(IDT, MODE, 1);                       \
  } while (0)
    if (id_bytes == 8) {
      if (a.mode == 0) TK_WLAUNCH(long long, 0); else if (a.mode == 1) TK_WLAUNCH(long long, 1); else TK_WLAUNCH(long long, 2);
    } else {
      if (a.mode == 0) TK_WLAUNCH(int, 0); else if (a.mode == 1) TK_WLAUNCH(int, 1); else TK_WLAUNCH(int, 2);
    }
#undef TK_WLAUNCH2
#undef TK_WLAUNCH
    return (int)cudaGetLastError();
  }
  const size_t blk = (size_t)KB * TK_M * 128;
  int stages = (int)((220 * 1024 - blk * MBv - 2048) / blk);
  if (stages > TK_MAX_STAGES) stages = TK_MAX_STAGES;
  if (stages < 2) return -1003;
  a.n_stages = stages;
  const size_t smem = blk * (MBv + stages) + 2 * TK_MAX_STAGES * 8 + 1024;
  const int grid = qblocks * a.n_splits;
#define TK_LAUNCH2(IDT, MODE, MBT)                                                                 \
  do {                                                                                             \
    cudaError_t e = cudaFuncSetAttribute(fps_topk_mma_kernel<IDT, MODE, MBT>,                      \
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  \
    if (e != cudaSuccess) return (int)e;                                                           \
    fps_topk_mma_kernel<IDT, MODE, MBT><<<grid, 256 * MBT + 32, smem, stream>>>(map, a);           \
  } while (0)
#define TK_LAUNCH(IDT, MODE)                                                                       \
  do {                                                                                             \
    if (MBv == 2) TK_LAUNCH2(IDT, MODE, 2); else TK_LAUNCH2(IDT, MODE, 1);                         \
  } while (0)
  if (id_bytes == 8) {
    if (a.mode == 0) TK_LAUNCH(long long, 0); else if (a.mode == 1) TK_LAUNCH(long long, 1); else TK_LAUNCH(long long, 2);
  } else {
    if (a.mode == 0) TK_LAUNCH(int, 0); else if (a.mode == 1) TK_LAUNCH(int, 1); else TK_LAUNCH(int, 2);
  }
#undef TK_LAUNCH2
#undef TK_LAUNCH
  return (int)cudaGetLastError();
}
