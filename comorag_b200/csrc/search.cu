// K4: fused query-block x corpus-shard bf16 inner product + exact top-k + running
// (min, max), one persistent CTA per SM.
//
// Replaces the reference's per-query  np.dot(E, q.T) -> min_max_normalize ->
// np.argsort(...)[::-1]  (ComoRAG.py:937-967, embed_utils.py:153-158) for up to
// 32 queries per pass over the shard, without ever writing the [nq, N] score
// matrix.
//
// Data flow per CTA (288 threads):
//   warp 8   TMA producer: streams the shard as 128-row x 64-col bf16 boxes
//            (16 KB, 128-byte swizzle), each with the 32 x 64 query slice of
//            the same columns (4 KB, from L2), through a STAGES-deep mbarrier
//            ring.
//   warps 4-7  wgmma warpgroup: scores[128 rows, 32 queries] accumulate in
//            registers (fp32, two m64n32k16 per 16-wide K step) over the tile,
//            then go to one of kAccStages shared-memory score tiles, so the HBM
//            stream keeps running while the select warps are busy sorting a
//            full candidate buffer.
//   warps 0-3  select: each thread owns one corpus row of the tile, reads its
//            32 scores from the score tile, updates per-query min/max in
//            registers and offers scores that beat the query's current k-th
//            best to a small shared candidate buffer; full buffers are
//            bitonic-sorted in registers by one warp (topk.cuh).
//            The admission threshold is the better of the CTA's own k-th key
//            and a floor pooled over ALL CTAs (kPoolM below).
// The shard is read exactly once from HBM: algorithmic bytes = n_rows*dim*2.
// Variants of the same pipeline: IVF = true walks a work-list of probed tiles
// (crag_ivf_search); SCORES = true stores every score (crag_search_scores) or
// keeps each row's running argmax over centroid blocks (crag_ivf_assign);
// I8 = true scans int8 rows (crag_search_topk_i8, and with IVF crag_ivf_search_i8).
// Around it in this file: the per-shard merge (merge_topk_kernel), the fused
// finalize + NVLink exchange + global merge of the row-sharded index
// (finalize_exchange_kernel), the C-ABI entry points, and crag_knn_topk -- exact
// top-k up to k = 2048 for large query batches as a score-block GEMM (gemm.cu)
// plus a per-query radix select (knn_select.cuh).
#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"
#include "topk.cuh"
#include "pool_floor.cuh"
#include "merge_kernels.cuh"
#include "ivf_kernels.cuh"
#include "search_types.cuh"
#include "select_warps.cuh"
#include "gemm.cuh"
#include "knn_select.cuh"

namespace crag {

// Dynamic shared memory of the scan, from a 1024-byte aligned base: the pipeline stages, the score tiles, the
// selector (select_warps.cuh), then the mbarriers.
template <int KLIST, int CAP, int STAGES>
struct SearchLayout {
  static constexpr size_t kTilesOff = size_t(STAGES) * kStageTotalBytes;
  static constexpr size_t kSelectOff = kTilesOff + size_t(kAccStages) * kScoreTileBytes;
  static constexpr size_t kBarsOff = kSelectOff + SelectSmem<KLIST, CAP>::bytes();
  // + the alignment pad of the base and 16 bytes of slack past the mbarriers
  __host__ __device__ static constexpr size_t smem_bytes() { return 1024 + kBarsOff + (2 * STAGES + 2 * kAccStages) * 8 + 16; }
};

// the 32 scores of row `row` of a score tile (layout: score_slot) -> r[q]
__device__ __forceinline__ void ld_score_row(const float* tile, int row, uint32_t (&r)[kNQ]) {
#pragma unroll
  for (int q = 0; q < kNQ; ++q) r[q] = __float_as_uint(tile[score_slot(row, q)]);
}

// The select warps' score-tile source: wait until the wgmma warpgroup has filled score tile `acc`, read this lane's
// row of it, and hand the buffer back once the whole warp has read.
struct SmemScoreTiles {
  const float* tiles;            // [kAccStages][128 * 32]
  uint64_t *full, *empty;        // [kAccStages] each
  int acc = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void next(int /*tile*/, int quad, int lane, uint32_t (&r)[kNQ]) {
    mbar_wait(&full[acc], phase);
    ld_score_row(tiles + acc * (kTileRows * kNQ), quad * 32 + lane, r);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[acc]);
    if (++acc == kAccStages) { acc = 0; phase ^= 1; }
  }
};

// Int8 variant of the flat top-k scan (I8 = true, crag_search_topk_i8): the shard and the query block are int8 with one
// fp32 scale per row / query (quant_kernels.cuh).  A 128-byte swizzle row holds 128 int8 instead of 64 bf16, so boxes,
// stages, descriptors and score tiles keep their byte sizes; the warpgroup issues m64n32k32.s32.s8.s8 and its epilogue
// writes S1 = float(acc) * (s_q * s_row) to the score tile, which the select warps rank as they rank bf16 scores.
struct I8Args {
  const float* row_scales;     // [n_rows]
  const float* query_scales;   // [nq] of this pass
};
// The int8 IVF scan (IVF = I8 = true, crag_ivf_search_i8) walks the IVF work-list over int8 residuals: the select warps
// see the IvfArgs base, the wgmma warpgroup the scales.
struct I8IvfArgs : IvfArgs {
  const float* row_scales;     // [n_rows_padded], 0 on padding rows
  const float* query_scales;   // [nq] of this pass
};
template <bool IVF, bool SCORES, bool I8> struct ScanParam { using type = typename IvfParam<IVF, SCORES>::type; };
template <> struct ScanParam<false, false, true> { using type = I8Args; };
template <> struct ScanParam<true, false, true> { using type = I8IvfArgs; };

template <int KLIST, int CAP, int STAGES, bool IVF = false, bool SCORES = false, bool I8 = false>
__global__ void __launch_bounds__(kSearchThreads, 1)
search_topk_kernel(const __grid_constant__ CUtensorMap tm_corpus, const __grid_constant__ CUtensorMap tm_q,
                   int n_rows, int num_kb, int nq, int k, const uint64_t* __restrict__ after_keys,
                   uint64_t* __restrict__ pool, uint32_t perm_mul, int perm_shift, uint64_t* __restrict__ part_keys,
                   float* __restrict__ part_minmax, const typename ScanParam<IVF, SCORES, I8>::type args) {
  static_assert(!(I8 && SCORES), "the int8 scan is a top-k scan");
  // elements per 128-byte swizzle row: the producer's column step per k-block
  constexpr int kBlockElems = I8 ? 128 : kBlockK;
  using L = SearchLayout<KLIST, CAP, STAGES>;
  static_assert(L::smem_bytes() <= 227 * 1024, "stages, score tiles and candidate lists exceed 227 KB of shared memory");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  uint8_t* stage_base = smem;
  float* score_tiles = reinterpret_cast<float*>(smem + L::kTilesOff);
  const auto sel = SelectSmem<KLIST, CAP>::carve(smem + L::kSelectOff);
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + L::kBarsOff);
  uint64_t* bar_empty = bar_full + STAGES;
  uint64_t* bar_tfull = bar_empty + STAGES;            // [kAccStages]
  uint64_t* bar_tempty = bar_tfull + kAccStages;       // [kAccStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int num_tiles;
  if constexpr (IVF) num_tiles = __ldg(args.n_work);
  else num_tiles = (n_rows + kTileRows - 1) / kTileRows;
  const TileOrder order(num_tiles, perm_mul, perm_shift);

  // ------------------------------------------------------------ one-time setup
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&bar_full[s], 1);
      mbar_init(&bar_empty[s], 4);   // one arrive per warp of the wgmma warpgroup
    }
    for (int a = 0; a < kAccStages; ++a) {
      mbar_init(&bar_tfull[a], 128); // every thread of the wgmma warpgroup, after its score stores
      mbar_init(&bar_tempty[a], 4);  // one arrive per select warp
    }
    fence_mbar_init();
  }
  sel.init(nq, after_keys);
  __syncthreads();

  if (warp == kProducerWarp) {
    // ================================================================ producer
    if (lane == 0) {
      tma_prefetch_desc(&tm_corpus);
      tma_prefetch_desc(&tm_q);
      const uint64_t pol = policy_evict_first();
      int stage = 0;
      uint32_t phase = 0;
      for (int j = blockIdx.x; j < num_tiles; j += gridDim.x) {
        const int tile = IVF ? j : order(j);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&bar_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&bar_full[stage], kStageTotalBytes);
          int tile_row0;
          if constexpr (IVF) tile_row0 = __ldg(&args.work[tile].x);
          else tile_row0 = tile * kTileRows;
          uint8_t* st = stage_base + stage * kStageTotalBytes;
          tma_load_2d_hint(&tm_corpus, &bar_full[stage], st, kb * kBlockElems, tile_row0, pol);
          tma_load_2d(&tm_q, &bar_full[stage], st + kStageBytes, kb * kBlockElems, 0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= kMmaWarp0) {
    // ============================================================ wgmma warpgroup
    // d[0]: rows 0-63 of the tile, d[1]: rows 64-127; this thread's rows 16 (warp % 4) + lane / 4 (+ 8) of each
    const int frag_row = (warp - kMmaWarp0) * 16 + (lane >> 2);
    const int frag_col = 2 * (lane & 3);
    int stage = 0;
    uint32_t phase = 0;
    int acc = 0;
    uint32_t acc_phase = 0;
    using Acc = std::conditional_t<I8, int32_t, float>;
    // I8: the scales of this thread's 8 query columns (0 past nq), held for the whole scan
    float q_scale[I8 ? kNQ / 4 : 1];
    if constexpr (I8) {
#pragma unroll
      for (int j = 0; j < kNQ / 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int q = 8 * j + frag_col + c;
          q_scale[2 * j + c] = q < nq ? __ldg(&args.query_scales[q]) : 0.f;
        }
    }
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      Acc d[2][16];
#pragma unroll
      for (int i = 0; i < 16; ++i) d[0][i] = d[1][i] = Acc(0);
      // I8: the scales of this thread's 4 rows of the tile (0 past n_rows), fetched while the k-blocks stream in
      float r_scale[I8 ? 4 : 1];
      if constexpr (I8) {
        int row0;
        if constexpr (IVF) row0 = __ldg(&args.work[tile].x);
        else row0 = order(tile) * kTileRows;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = row0 + (i >> 1) * 64 + frag_row + (i & 1) * 8;
          r_scale[i] = row < n_rows ? __ldg(&args.row_scales[row]) : 0.f;
        }
      }
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&bar_full[stage], phase);
        const uint32_t a_addr = smem_u32(stage_base + stage * kStageTotalBytes);
        const uint32_t b_addr = a_addr + kStageBytes;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kBlockK / 16; ++ks) {   // 32-byte K steps: 16 bf16 or 32 int8
          const uint64_t db = wgmma_desc_sw128(b_addr + ks * 32);
          if constexpr (I8) {
            wgmma_m64n32k32_s8_ss(d[0], wgmma_desc_sw128(a_addr + ks * 32), db, 1u);
            wgmma_m64n32k32_s8_ss(d[1], wgmma_desc_sw128(a_addr + 64 * 128 + ks * 32), db, 1u);
          } else {
            wgmma_m64n32k16_ss(d[0], wgmma_desc_sw128(a_addr + ks * 32), db, 1u);
            wgmma_m64n32k16_ss(d[1], wgmma_desc_sw128(a_addr + 64 * 128 + ks * 32), db, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();   // k-block kb - 1 has retired: its smem slot goes back to the producer
        if (kb > 0 && lane == 0) mbar_arrive(&bar_empty[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d[0]);
      wgmma_fence_regs(d[1]);
      if (lane == 0) mbar_arrive(&bar_empty[prev]);
      mbar_wait(&bar_tempty[acc], acc_phase ^ 1);
      float* st = score_tiles + acc * (kTileRows * kNQ);
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < kNQ / 8; ++j)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = m * 64 + frag_row + (i >> 1) * 8;
            if constexpr (I8) {   // S1 = float(acc) * (s_q * s_row); |acc| <= 127^2 * 1024 < 2^24 converts exactly
              const float scale = __fmul_rn(q_scale[2 * j + (i & 1)], r_scale[2 * m + (i >> 1)]);
              st[score_slot(row, 8 * j + frag_col + (i & 1))] = __fmul_rn(__int2float_rn(d[m][4 * j + i]), scale);
            } else {
              st[score_slot(row, 8 * j + frag_col + (i & 1))] = d[m][4 * j + i];
            }
          }
      mbar_arrive(&bar_tfull[acc]);
      if (++acc == kAccStages) { acc = 0; acc_phase ^= 1; }
    }
  } else {
    // ================================================================== select
    SmemScoreTiles tiles{score_tiles, bar_tfull, bar_tempty};
    if constexpr (I8 && !IVF) select_warps<KLIST, CAP, false, false>(sel, tiles, order, num_tiles, n_rows, nq, k, after_keys, pool, part_keys, part_minmax, NoIvfArgs{}, warp, lane);
    else select_warps<KLIST, CAP, IVF, SCORES>(sel, tiles, order, num_tiles, n_rows, nq, k, after_keys, pool, part_keys, part_minmax, args, warp, lane);
  }
}

// ------------------------------------------------------------------ host side
namespace {

struct SearchPlan {
  int grid;
  size_t keys_bytes;    // per 32-query pass
  size_t minmax_bytes;  // per 32-query pass
  size_t pool_bytes;    // pooled-floor table of one 32-query pass (0 when the grid exceeds kPoolMaxCtas)
};

SearchPlan plan_search(int k) {
  SearchPlan p;
  p.grid = sm_count();
  if (p.grid <= 0) p.grid = 132;
  p.keys_bytes = ((size_t(p.grid) * kNQ * k * 8) + 255) & ~size_t(255);
  p.minmax_bytes = ((size_t(p.grid) * kNQ * 2 * 4) + 255) & ~size_t(255);
  p.pool_bytes = p.grid <= kPoolMaxCtas ? ((size_t(kNQ) * p.grid * kPoolSlots * 8 + 255) & ~size_t(255)) : 0;
  return p;
}

// One launch of the scan.  The dynamic shared-memory limit is raised once per instantiation and device.
template <int KLIST, int CAP, int STAGES, bool IVF, bool SCORES, bool I8 = false>
int launch_scan(const CUtensorMap& tm_corpus, const CUtensorMap& tm_q, int n_rows, int num_kb, int nq, int k, int grid,
                const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul, int perm_shift, uint64_t* part_keys,
                float* part_minmax, const typename ScanParam<IVF, SCORES, I8>::type& args, cudaStream_t stream) {
  constexpr size_t smem = SearchLayout<KLIST, CAP, STAGES>::smem_bytes();
  auto kern = search_topk_kernel<KLIST, CAP, STAGES, IVF, SCORES, I8>;
  static bool attr_set[64] = {};
  int dev = 0;
  CRAG_CUDA_OK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    CRAG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  kern<<<grid, kSearchThreads, smem, stream>>>(tm_corpus, tm_q, n_rows, num_kb, nq, k, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

// A top-k scan with the selector of k: 64-key lists and 6 stages up to k = 64, 128-key lists and 4 stages above.
// I8Args / I8IvfArgs select the int8 scan.
template <bool IVF, class Args>
int launch_topk_scan(const CUtensorMap& tm_corpus, const CUtensorMap& tm_q, int n_rows, int num_kb, int nq, int k,
                     int grid, const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul, int perm_shift,
                     uint64_t* part_keys, float* part_minmax, const Args& args, cudaStream_t stream) {
  constexpr bool I8 = std::is_same<Args, I8Args>::value || std::is_same<Args, I8IvfArgs>::value;
  if (k <= 64) return launch_scan<64, 64, 6, IVF, false, I8>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
  return launch_scan<128, 128, 4, IVF, false, I8>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
}

// The merge kernels' list size for k (32, 64 or 128), passed to `launch` as a std::integral_constant.
template <class Launch>
void with_merge_tier(int k, Launch launch) {
  if (k <= 32) launch(std::integral_constant<int, 32>{});
  else if (k <= 64) launch(std::integral_constant<int, 64>{});
  else launch(std::integral_constant<int, 128>{});
}

// tensor map of queries q0 .. q0 + nqc - 1 (nqc <= 32) of a dense [nq, dim] bf16 array
int make_query_tmap(CUtensorMap* tm, const void* queries, int q0, int nqc, int dim) {
  return make_tmap_bf16_2d(tm, static_cast<const uint8_t*>(queries) + size_t(q0) * dim * 2, uint64_t(nqc), uint64_t(dim), uint64_t(dim) * 2, kNQ);
}

}  // namespace
}  // namespace crag

using namespace crag;

extern "C" size_t crag_search_workspace_bytes(int nq, int k) {
  (void)nq;
  if (k < 1 || k > 128) return 0;
  const SearchPlan p = plan_search(k);
  return p.keys_bytes + p.minmax_bytes + p.pool_bytes;
}

namespace crag {
namespace {

int check_search_args(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride, const void* queries,
                      int nq, int k, const void* workspace, size_t workspace_bytes, const SearchPlan& plan,
                      int k_max = 128) {
  if (nq < 1 || k < 1 || k > k_max) return fail(CRAG_ERR_INVALID, "search: need nq >= 1 and 1 <= k <= %d (nq=%d k=%d)", k_max, nq, k);
  if (dim < 64 || dim > 1024 || dim % 64 != 0) return fail(CRAG_ERR_INVALID, "search: dim must be a multiple of 64 in [64, 1024] (dim=%d)", dim);
  if (n_rows < 0 || n_rows >= (int64_t(1) << 31) - kTileRows) return fail(CRAG_ERR_INVALID, "search: n_rows out of range (%lld)", (long long)n_rows);
  if (corpus_row_stride < dim || corpus_row_stride % 8 != 0) return fail(CRAG_ERR_INVALID, "search: corpus_row_stride must be >= dim and a multiple of 8");
  if (!queries || !workspace || (n_rows > 0 && !corpus)) return fail(CRAG_ERR_INVALID, "search: null pointer");
  if ((reinterpret_cast<uintptr_t>(corpus) | reinterpret_cast<uintptr_t>(queries)) & 15) return fail(CRAG_ERR_INVALID, "search: corpus/queries must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(CRAG_ERR_INVALID, "search: workspace must be 256-byte aligned");
  if (workspace_bytes < plan.keys_bytes + plan.minmax_bytes) return fail(CRAG_ERR_WORKSPACE, "search: workspace %zu < %zu bytes", workspace_bytes, plan.keys_bytes + plan.minmax_bytes);
  return CRAG_OK;
}

inline int scan_grid(int64_t n_rows, const SearchPlan& plan) {
  const int num_tiles = int((n_rows + kTileRows - 1) / kTileRows);
  return num_tiles < plan.grid ? num_tiles : plan.grid;
}

// the flat scans permute groups of 2^kPermShift consecutive tiles (TileOrder)
constexpr int kPermShift = 3;

// one corpus pass for queries q0 .. q0 + nq - 1 (nq <= 32): per-CTA partial lists into the workspace.  With `i8` the
// corpus and queries are int8 [*, dim] (dim a multiple of 128) with the scales of i8 (query scales from query 0 on).
int scan_pass(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride, const void* queries, int q0,
              int nq, int k, const uint64_t* after_keys, void* workspace, size_t workspace_bytes,
              const SearchPlan& plan, cudaStream_t stream, const I8Args* i8 = nullptr) {
  const int grid = scan_grid(n_rows, plan);
  if (grid == 0) return CRAG_OK;
  uint64_t* part_keys = static_cast<uint64_t*>(workspace);
  float* part_minmax = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + plan.keys_bytes);
  // pooled floor: needs its table in the workspace and pays off once a CTA sees more than a couple of tiles
  uint64_t* pool = nullptr;
  const int64_t num_tiles = (n_rows + kTileRows - 1) / kTileRows;
  if (plan.pool_bytes && workspace_bytes >= plan.keys_bytes + plan.minmax_bytes + plan.pool_bytes && num_tiles >= 4 * int64_t(grid)) {
    pool = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(workspace) + plan.keys_bytes + plan.minmax_bytes);
    CRAG_CUDA_OK(cudaMemsetAsync(pool, 0, plan.pool_bytes, stream));
  }
  CUtensorMap tm_corpus, tm_q;
  if (i8) {
    int rc = make_tmap_u8_2d(&tm_corpus, corpus, uint64_t(n_rows), uint64_t(dim), uint64_t(corpus_row_stride), kTileRows);
    if (rc != CRAG_OK) return rc;
    rc = make_tmap_u8_2d(&tm_q, static_cast<const uint8_t*>(queries) + size_t(q0) * dim, uint64_t(nq), uint64_t(dim), uint64_t(dim), kNQ);
    if (rc != CRAG_OK) return rc;
    return launch_topk_scan<false>(tm_corpus, tm_q, int(n_rows), dim / 128, nq, k, grid, after_keys, pool,
                                   perm_multiplier(num_tiles >> kPermShift), kPermShift, part_keys, part_minmax,
                                   I8Args{i8->row_scales, i8->query_scales + q0}, stream);
  }
  int rc = make_tmap_bf16_2d(&tm_corpus, corpus, uint64_t(n_rows), uint64_t(dim), uint64_t(corpus_row_stride) * 2, kTileRows);
  if (rc != CRAG_OK) return rc;
  rc = make_query_tmap(&tm_q, queries, q0, nq, dim);
  if (rc != CRAG_OK) return rc;
  return launch_topk_scan<false>(tm_corpus, tm_q, int(n_rows), dim / kBlockK, nq, k, grid, after_keys, pool,
                                 perm_multiplier(num_tiles >> kPermShift), kPermShift, part_keys, part_minmax, NoIvfArgs{}, stream);
}

// merge the per-CTA partials of one pass into the final (ids, scores, minmax) of its <= 32 queries
int finalize_parts(const void* workspace, int grid, int nq, int k, int64_t row_offset, int64_t* out_ids,
                   float* out_scores, float* out_minmax, uint64_t* last_keys, const SearchPlan& plan, cudaStream_t stream) {
  const uint64_t* part_keys = static_cast<const uint64_t*>(workspace);
  const float* part_minmax = reinterpret_cast<const float*>(static_cast<const uint8_t*>(workspace) + plan.keys_bytes);
  with_merge_tier(k, [&](auto tier) {   // one CTA per query
    constexpr int T = decltype(tier)::value;
    merge_topk_kernel<T, T, false><<<nq, 128, 0, stream>>>(part_keys, nullptr, nullptr, part_minmax, grid, kNQ, nq, k, row_offset, 0, 0, 0,
                                                           out_ids, out_scores, out_minmax, last_keys);
  });
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

int finalize_pass(const void* workspace, int64_t n_rows, int nq, int k, int64_t row_offset, int64_t* out_ids,
                  float* out_scores, float* out_minmax, uint64_t* last_keys, const SearchPlan& plan, cudaStream_t stream) {
  return finalize_parts(workspace, scan_grid(n_rows, plan), nq, k, row_offset, out_ids, out_scores, out_minmax, last_keys,
                        plan, stream);
}

// IVF workspace = the flat scan's per-CTA partials, then the per-pass plan
struct IvfPlan {
  size_t pool_off, mask_off, coarse_off, work_off, count_off, total;
};
IvfPlan plan_ivf(const SearchPlan& sp, int nlist, int64_t total_tiles) {
  auto up = [](size_t x) { return (x + 255) & ~size_t(255); };
  IvfPlan p;
  p.pool_off = sp.keys_bytes + sp.minmax_bytes;
  p.mask_off = p.pool_off + sp.pool_bytes;
  p.coarse_off = p.mask_off + up(size_t(nlist) * 4);
  p.work_off = p.coarse_off + up(size_t(nlist) * kNQ * 4);
  p.count_off = p.work_off + up(size_t(total_tiles) * sizeof(int4));
  p.total = p.count_off + 256;
  return p;
}

}  // namespace
}  // namespace crag

extern "C" size_t crag_ivf_workspace_bytes(int nlist, int64_t total_tiles, int k) {
  if (nlist < 1 || total_tiles < 0 || k < 1 || k > 128) return 0;
  return plan_ivf(plan_search(k), nlist, total_tiles).total;
}

extern "C" int crag_ivf_search(const void* residuals, int64_t n_rows_padded, int dim, int64_t row_stride,
                               const int32_t* list_tile_start, const int32_t* list_rows, int nlist,
                               int64_t total_tiles, const int64_t* row_ids, const void* queries, int nq,
                               const int64_t* probed_ids, const float* probed_scores, int nprobe, int k,
                               int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                               size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SearchPlan sp = plan_search(k >= 1 && k <= 128 ? k : 1);
  if (nlist < 1 || nlist > (1 << 20) || nprobe < 1 || nprobe > nlist) return fail(CRAG_ERR_INVALID, "ivf: need 1 <= nprobe <= nlist <= 2^20 (nprobe=%d nlist=%d)", nprobe, nlist);
  if (total_tiles < 0 || total_tiles * kTileRows != n_rows_padded) return fail(CRAG_ERR_INVALID, "ivf: n_rows_padded (%lld) must be total_tiles (%lld) * %d", (long long)n_rows_padded, (long long)total_tiles, kTileRows);
  const IvfPlan ip = plan_ivf(sp, nlist, total_tiles);
  int rc = check_search_args(residuals, n_rows_padded, dim, row_stride, queries, nq, k, workspace, workspace_bytes, sp);
  if (rc != CRAG_OK) return rc;
  if (workspace_bytes < ip.total) return fail(CRAG_ERR_WORKSPACE, "ivf: workspace %zu < %zu bytes", workspace_bytes, ip.total);
  if (!list_tile_start || !list_rows || !row_ids || !probed_ids || !probed_scores || !out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "ivf: null pointer");
  if (n_rows_padded == 0) return fail(CRAG_ERR_INVALID, "ivf: empty index");
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  uint64_t* part_keys = reinterpret_cast<uint64_t*>(ws);
  float* part_minmax = reinterpret_cast<float*>(ws + sp.keys_bytes);
  IvfArgs ivf;
  ivf.list_mask = reinterpret_cast<uint32_t*>(ws + ip.mask_off);
  ivf.coarse = reinterpret_cast<float*>(ws + ip.coarse_off);
  ivf.work = reinterpret_cast<int4*>(ws + ip.work_off);
  ivf.n_work = reinterpret_cast<int*>(ws + ip.count_off);
  CUtensorMap tm_res;
  rc = make_tmap_bf16_2d(&tm_res, residuals, uint64_t(n_rows_padded), uint64_t(dim), uint64_t(row_stride) * 2, kTileRows);
  if (rc != CRAG_OK) return rc;
  const int num_kb = dim / kBlockK;
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    CUtensorMap tm_q;
    rc = make_query_tmap(&tm_q, queries, q0, nqc, dim);
    if (rc != CRAG_OK) return rc;
    ivf_plan_kernel<<<1, 1024, 0, stream>>>(probed_ids + size_t(q0) * nprobe, probed_scores + size_t(q0) * nprobe, nqc, nprobe,
                                            nlist, list_tile_start, list_rows, const_cast<uint32_t*>(ivf.list_mask),
                                            const_cast<float*>(ivf.coarse), const_cast<int4*>(ivf.work), const_cast<int*>(ivf.n_work));
    CRAG_CUDA_OK(cudaGetLastError());
    // every CTA of the grid publishes a (possibly empty) partial list, so the merge always reads sp.grid parts
    uint64_t* pool = nullptr;
    if (sp.pool_bytes) {
      pool = reinterpret_cast<uint64_t*>(ws + ip.pool_off);
      CRAG_CUDA_OK(cudaMemsetAsync(pool, 0, sp.pool_bytes, stream));
    }
    rc = launch_topk_scan<true>(tm_res, tm_q, 0, num_kb, nqc, k, sp.grid, nullptr, pool, 0u, 0, part_keys, part_minmax, ivf, stream);
    if (rc != CRAG_OK) return rc;
    rc = finalize_parts(workspace, sp.grid, nqc, k, 0, out_ids + size_t(q0) * k, out_scores + size_t(q0) * k,
                        out_minmax ? out_minmax + size_t(q0) * 2 : nullptr, nullptr, sp, stream);
    if (rc != CRAG_OK) return rc;
    ivf_map_ids_kernel<<<(nqc * k + 255) / 256, 256, 0, stream>>>(out_ids + size_t(q0) * k, nqc * k, row_ids);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}

// ------------------------------------------------------------------ IVF over int8 residuals
// Per 32-query pass: the IVF plan, the int8 scan of the probed tiles for n_cand candidates (S1 + coarse term), their
// merge into the workspace, the exact bf16 rescore with the coarse term of each candidate's list (quant.cu), and the
// map of stored positions to original ids.  The coarse table the rescore reads is the plan's, rebuilt every pass.
namespace crag {
namespace {
struct IvfI8Plan {
  IvfPlan ivf;
  size_t cand_ids_off, cand_scores_off, total;
};
IvfI8Plan plan_ivf_i8(int nlist, int64_t total_tiles, int n_cand) {
  IvfI8Plan p;
  p.ivf = plan_ivf(plan_search(n_cand), nlist, total_tiles);
  p.cand_ids_off = p.ivf.total;
  p.cand_scores_off = p.cand_ids_off + ((size_t(kNQ) * n_cand * 8 + 255) & ~size_t(255));
  p.total = p.cand_scores_off + ((size_t(kNQ) * n_cand * 4 + 255) & ~size_t(255));
  return p;
}
}  // namespace
}  // namespace crag

extern "C" size_t crag_ivf_i8_workspace_bytes(int nlist, int64_t total_tiles, int n_cand) {
  if (nlist < 1 || total_tiles < 0 || n_cand < 1 || n_cand > 128) return 0;
  return plan_ivf_i8(nlist, total_tiles, n_cand).total;
}

extern "C" int crag_ivf_search_i8(const void* residuals_i8, const float* row_scales, int dim8, int64_t row_stride_i8,
                                  const void* residuals_bf16, int dim, int64_t row_stride, int64_t n_rows_padded,
                                  const int32_t* list_tile_start, const int32_t* list_rows, int nlist,
                                  int64_t total_tiles, const int64_t* row_ids, const void* queries_i8,
                                  const float* query_scales, const void* queries_bf16, int nq,
                                  const int64_t* probed_ids, const float* probed_scores, int nprobe, int n_cand, int k,
                                  int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                                  size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (nlist < 1 || nlist > (1 << 20) || nprobe < 1 || nprobe > nlist) return fail(CRAG_ERR_INVALID, "ivf_i8: need 1 <= nprobe <= nlist <= 2^20 (nprobe=%d nlist=%d)", nprobe, nlist);
  if (nq < 1 || k < 1 || n_cand < k || n_cand > 128) return fail(CRAG_ERR_INVALID, "ivf_i8: need nq >= 1 and 1 <= k <= n_cand <= 128 (nq=%d k=%d n_cand=%d)", nq, k, n_cand);
  if (dim < 64 || dim > 1024 || dim % 64 != 0) return fail(CRAG_ERR_INVALID, "ivf_i8: dim must be a multiple of 64 in [64, 1024] (dim=%d)", dim);
  if (dim8 != (dim + 127) / 128 * 128) return fail(CRAG_ERR_INVALID, "ivf_i8: dim8 must be dim rounded up to a multiple of 128 (dim=%d dim8=%d)", dim, dim8);
  if (total_tiles < 1 || total_tiles * kTileRows != n_rows_padded || n_rows_padded >= (int64_t(1) << 31) - kTileRows) return fail(CRAG_ERR_INVALID, "ivf_i8: need n_rows_padded (%lld) = total_tiles (%lld) * %d, non-empty and below 2^31", (long long)n_rows_padded, (long long)total_tiles, kTileRows);
  if (row_stride_i8 < dim8 || row_stride_i8 % 16 != 0) return fail(CRAG_ERR_INVALID, "ivf_i8: row_stride_i8 must be >= dim8 and a multiple of 16");
  if (row_stride < dim || row_stride % 8 != 0) return fail(CRAG_ERR_INVALID, "ivf_i8: row_stride must be >= dim and a multiple of 8");
  if (!residuals_i8 || !row_scales || !residuals_bf16 || !list_tile_start || !list_rows || !row_ids || !queries_i8 ||
      !query_scales || !queries_bf16 || !probed_ids || !probed_scores || !out_ids || !out_scores || !workspace) return fail(CRAG_ERR_INVALID, "ivf_i8: null pointer");
  if ((reinterpret_cast<uintptr_t>(residuals_i8) | reinterpret_cast<uintptr_t>(queries_i8) | reinterpret_cast<uintptr_t>(residuals_bf16) |
       reinterpret_cast<uintptr_t>(queries_bf16)) & 15) return fail(CRAG_ERR_INVALID, "ivf_i8: residuals and queries must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(CRAG_ERR_INVALID, "ivf_i8: workspace must be 256-byte aligned");
  const IvfI8Plan plan = plan_ivf_i8(nlist, total_tiles, n_cand);
  if (workspace_bytes < plan.total) return fail(CRAG_ERR_WORKSPACE, "ivf_i8: workspace %zu < %zu bytes", workspace_bytes, plan.total);
  const void* rows_bf16 = nullptr;   // the bf16 residuals may be page-locked host memory: refused before any launch if pageable
  int rc = device_readable(residuals_bf16, &rows_bf16, "ivf_i8");
  if (rc != CRAG_OK) return rc;
  const SearchPlan sp = plan_search(n_cand);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  uint64_t* part_keys = reinterpret_cast<uint64_t*>(ws);
  float* part_minmax = reinterpret_cast<float*>(ws + sp.keys_bytes);
  int64_t* cand_ids = reinterpret_cast<int64_t*>(ws + plan.cand_ids_off);
  float* cand_scores = reinterpret_cast<float*>(ws + plan.cand_scores_off);
  I8IvfArgs args;
  args.list_mask = reinterpret_cast<uint32_t*>(ws + plan.ivf.mask_off);
  args.coarse = reinterpret_cast<float*>(ws + plan.ivf.coarse_off);
  args.work = reinterpret_cast<int4*>(ws + plan.ivf.work_off);
  args.n_work = reinterpret_cast<int*>(ws + plan.ivf.count_off);
  args.row_scales = row_scales;
  CUtensorMap tm_res;
  rc = make_tmap_u8_2d(&tm_res, residuals_i8, uint64_t(n_rows_padded), uint64_t(dim8), uint64_t(row_stride_i8), kTileRows);
  if (rc != CRAG_OK) return rc;
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    CUtensorMap tm_q;
    rc = make_tmap_u8_2d(&tm_q, static_cast<const uint8_t*>(queries_i8) + size_t(q0) * dim8, uint64_t(nqc), uint64_t(dim8), uint64_t(dim8), kNQ);
    if (rc != CRAG_OK) return rc;
    ivf_plan_kernel<<<1, 1024, 0, stream>>>(probed_ids + size_t(q0) * nprobe, probed_scores + size_t(q0) * nprobe, nqc, nprobe,
                                            nlist, list_tile_start, list_rows, const_cast<uint32_t*>(args.list_mask),
                                            const_cast<float*>(args.coarse), const_cast<int4*>(args.work), const_cast<int*>(args.n_work));
    CRAG_CUDA_OK(cudaGetLastError());
    uint64_t* pool = nullptr;
    if (sp.pool_bytes) {
      pool = reinterpret_cast<uint64_t*>(ws + plan.ivf.pool_off);
      CRAG_CUDA_OK(cudaMemsetAsync(pool, 0, sp.pool_bytes, stream));
    }
    args.query_scales = query_scales + q0;
    rc = launch_topk_scan<true>(tm_res, tm_q, int(n_rows_padded), dim8 / 128, nqc, n_cand, sp.grid, nullptr, pool, 0u, 0,
                                part_keys, part_minmax, args, stream);
    if (rc != CRAG_OK) return rc;
    rc = finalize_parts(workspace, sp.grid, nqc, n_cand, 0, cand_ids, cand_scores,
                        out_minmax ? out_minmax + size_t(q0) * 2 : nullptr, nullptr, sp, stream);
    if (rc != CRAG_OK) return rc;
    rc = launch_ivf_rescore(rows_bf16, n_rows_padded, dim, row_stride, static_cast<const uint8_t*>(queries_bf16) + size_t(q0) * dim * 2,
                            nqc, cand_ids, n_cand, k, list_tile_start, nlist, args.coarse, out_ids + size_t(q0) * k,
                            out_scores + size_t(q0) * k, stream);
    if (rc != CRAG_OK) return rc;
    ivf_map_ids_kernel<<<(nqc * k + 255) / 256, 256, 0, stream>>>(out_ids + size_t(q0) * k, nqc * k, row_ids);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}

extern "C" int crag_search_scan(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                const void* queries, int nq, int k, void* workspace, size_t workspace_bytes,
                                crag_stream_t stream) {
  const SearchPlan plan = plan_search(k >= 1 && k <= 128 ? k : 1);
  int rc = check_search_args(corpus, n_rows, dim, corpus_row_stride, queries, nq, k, workspace, workspace_bytes, plan);
  if (rc != CRAG_OK) return rc;
  if (nq > kNQ) return fail(CRAG_ERR_INVALID, "crag_search_scan handles one pass of at most %d queries (nq=%d)", kNQ, nq);
  return scan_pass(corpus, n_rows, dim, corpus_row_stride, queries, 0, nq, k, nullptr, workspace, workspace_bytes, plan, static_cast<cudaStream_t>(stream));
}

extern "C" int crag_search_finalize(const void* workspace, size_t workspace_bytes, int64_t n_rows, int nq, int k,
                                    int64_t row_offset, int64_t* out_ids, float* out_scores, float* out_minmax,
                                    crag_stream_t stream) {
  if (nq < 1 || nq > kNQ || k < 1 || k > 128) return fail(CRAG_ERR_INVALID, "crag_search_finalize: bad nq/k (nq=%d k=%d)", nq, k);
  const SearchPlan plan = plan_search(k);
  if (!workspace || !out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "crag_search_finalize: null pointer");
  if (workspace_bytes < plan.keys_bytes + plan.minmax_bytes) return fail(CRAG_ERR_WORKSPACE, "crag_search_finalize: workspace too small");
  return finalize_pass(workspace, n_rows, nq, k, row_offset, out_ids, out_scores, out_minmax, nullptr, plan, static_cast<cudaStream_t>(stream));
}

extern "C" int crag_search_topk_after(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                      int64_t row_offset, const void* queries, int nq, int k,
                                      const uint64_t* after_keys, int64_t* out_ids, float* out_scores,
                                      float* out_minmax, uint64_t* last_keys, void* workspace,
                                      size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SearchPlan plan = plan_search(k >= 1 && k <= 128 ? k : 1);
  int rc = check_search_args(corpus, n_rows, dim, corpus_row_stride, queries, nq, k, workspace, workspace_bytes, plan);
  if (rc != CRAG_OK) return rc;
  if (!out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "search: null output pointer");
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    rc = scan_pass(corpus, n_rows, dim, corpus_row_stride, queries, q0, nqc, k, after_keys ? after_keys + q0 : nullptr, workspace, workspace_bytes, plan, stream);
    if (rc != CRAG_OK) return rc;
    rc = finalize_pass(workspace, n_rows, nqc, k, row_offset, out_ids + size_t(q0) * k, out_scores + size_t(q0) * k,
                       out_minmax ? out_minmax + size_t(q0) * 2 : nullptr, last_keys ? last_keys + q0 : nullptr, plan, stream);
    if (rc != CRAG_OK) return rc;
  }
  return CRAG_OK;
}

extern "C" int crag_search_topk(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                int64_t row_offset, const void* queries, int nq, int k, int64_t* out_ids,
                                float* out_scores, float* out_minmax, void* workspace, size_t workspace_bytes,
                                crag_stream_t stream) {
  return crag_search_topk_after(corpus, n_rows, dim, corpus_row_stride, row_offset, queries, nq, k, nullptr, out_ids,
                                out_scores, out_minmax, nullptr, workspace, workspace_bytes, stream);
}

// ------------------------------------------------------------------ int8 shards (quant_kernels.cuh)
extern "C" int crag_search_topk_i8(const void* corpus_i8, const float* row_scales, int64_t n_rows, int dim8,
                                   int64_t row_stride, int64_t row_offset, const void* queries_i8,
                                   const float* query_scales, int nq, int k, int64_t* out_ids, float* out_scores,
                                   float* out_minmax, void* workspace, size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SearchPlan plan = plan_search(k >= 1 && k <= 128 ? k : 1);
  if (nq < 1 || k < 1 || k > 128) return fail(CRAG_ERR_INVALID, "search_i8: need nq >= 1 and 1 <= k <= 128 (nq=%d k=%d)", nq, k);
  if (dim8 < 128 || dim8 > 1024 || dim8 % 128 != 0) return fail(CRAG_ERR_INVALID, "search_i8: dim8 must be a multiple of 128 in [128, 1024] (dim8=%d)", dim8);
  if (n_rows < 0 || n_rows >= (int64_t(1) << 31) - kTileRows) return fail(CRAG_ERR_INVALID, "search_i8: n_rows out of range (%lld)", (long long)n_rows);
  if (row_stride < dim8 || row_stride % 16 != 0) return fail(CRAG_ERR_INVALID, "search_i8: row_stride must be >= dim8 and a multiple of 16");
  if (!queries_i8 || !query_scales || !workspace || !out_ids || !out_scores || (n_rows > 0 && (!corpus_i8 || !row_scales))) return fail(CRAG_ERR_INVALID, "search_i8: null pointer");
  if ((reinterpret_cast<uintptr_t>(corpus_i8) | reinterpret_cast<uintptr_t>(queries_i8)) & 15) return fail(CRAG_ERR_INVALID, "search_i8: corpus/queries must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(CRAG_ERR_INVALID, "search_i8: workspace must be 256-byte aligned");
  if (workspace_bytes < plan.keys_bytes + plan.minmax_bytes) return fail(CRAG_ERR_WORKSPACE, "search_i8: workspace %zu < %zu bytes", workspace_bytes, plan.keys_bytes + plan.minmax_bytes);
  const I8Args i8{row_scales, query_scales};
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    int rc = scan_pass(corpus_i8, n_rows, dim8, row_stride, queries_i8, q0, nqc, k, nullptr, workspace, workspace_bytes, plan, stream, &i8);
    if (rc != CRAG_OK) return rc;
    rc = finalize_pass(workspace, n_rows, nqc, k, row_offset, out_ids + size_t(q0) * k, out_scores + size_t(q0) * k,
                       out_minmax ? out_minmax + size_t(q0) * 2 : nullptr, nullptr, plan, stream);
    if (rc != CRAG_OK) return rc;
  }
  return CRAG_OK;
}

// ------------------------------------------------------------------ exact top-k for large k / many queries
// Per chunk of queries: the wgmma GEMM writes the fp32 score block [q_chunk, ld] into the workspace
// (gemm_scores_f32), then knn_select_kernel (knn_select.cuh) radix-selects each query's k best rows from its row.
namespace crag {
namespace {
inline int64_t knn_ld(int64_t n_rows) { return ((n_rows > 0 ? n_rows : 1) + 3) & ~int64_t(3); }
}  // namespace
}  // namespace crag

extern "C" size_t crag_knn_workspace_bytes(int64_t n_rows, int q_chunk) {
  if (n_rows < 0 || q_chunk < 1) return 0;
  return (size_t(q_chunk) * size_t(knn_ld(n_rows)) * 4 + 255) & ~size_t(255);
}

extern "C" int crag_knn_topk(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride, int64_t row_offset,
                             const void* queries, int nq, int k, int64_t* out_ids, float* out_scores, float* out_minmax,
                             void* workspace, size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SearchPlan no_scan_workspace{0, 0, 0, 0};
  int rc = check_search_args(corpus, n_rows, dim, corpus_row_stride, queries, nq, k, workspace, workspace_bytes,
                             no_scan_workspace, kKnnMaxK);
  if (rc != CRAG_OK) return rc;
  if (!out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "knn: null output pointer");
  const int64_t ld = knn_ld(n_rows);
  const size_t per_query = size_t(ld) * 4;
  const size_t fit = workspace_bytes / per_query;
  if (fit < 1) return fail(CRAG_ERR_WORKSPACE, "knn: workspace %zu < %zu bytes (one query's score row)", workspace_bytes, per_query);
  const int q_chunk = fit < size_t(nq) ? int(fit) : nq;
  float* block = static_cast<float*>(workspace);
  for (int q0 = 0; q0 < nq; q0 += q_chunk) {
    const int nqc = (nq - q0) < q_chunk ? (nq - q0) : q_chunk;
    rc = gemm_scores_f32(static_cast<const uint8_t*>(queries) + size_t(q0) * dim * 2, dim, corpus, corpus_row_stride,
                         block, ld, nqc, int(n_rows), dim, stream);
    if (rc != CRAG_OK) return rc;
    knn_select_kernel<<<nqc, kKnnThreads, 0, stream>>>(block, ld, int(n_rows), k, row_offset, out_ids + size_t(q0) * k,
                                                       out_scores + size_t(q0) * k,
                                                       out_minmax ? out_minmax + size_t(q0) * 2 : nullptr);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}

namespace crag {
namespace {
int merge_pairs(const float* scores, const int64_t* ids, const float* minmax, int64_t ids_stride, int64_t scores_stride,
                int64_t mm_stride, int parts, int nq, int k, int64_t* out_ids, float* out_scores, float* out_minmax,
                cudaStream_t stream) {
  if (parts < 0 || nq < 1 || k < 1 || k > 128 || int64_t(parts) * k > (1 << 20)) return fail(CRAG_ERR_INVALID, "crag_merge_topk: bad sizes (parts=%d nq=%d k=%d)", parts, nq, k);
  if (!out_ids || !out_scores || (parts > 0 && (!scores || !ids))) return fail(CRAG_ERR_INVALID, "crag_merge_topk: null pointer");
  const float* mm = out_minmax ? minmax : nullptr;
  with_merge_tier(k, [&](auto tier) {   // one CTA per query
    constexpr int T = decltype(tier)::value;
    merge_topk_kernel<T, T, true><<<nq, 128, 0, stream>>>(nullptr, scores, ids, mm, parts, nq, nq, k, 0, ids_stride, scores_stride, mm_stride,
                                                          out_ids, out_scores, out_minmax, nullptr);
  });
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}
}  // namespace
}  // namespace crag

extern "C" int crag_merge_topk(const float* scores, const int64_t* ids, const float* minmax, int parts, int nq,
                               int k, int64_t* out_ids, float* out_scores, float* out_minmax,
                               crag_stream_t stream) {
  return crag::merge_pairs(scores, ids, minmax, int64_t(nq) * k * 8, int64_t(nq) * k * 4, int64_t(nq) * 2 * 4, parts, nq, k,
                           out_ids, out_scores, out_minmax, static_cast<cudaStream_t>(stream));
}

extern "C" int crag_merge_topk_packed(const void* records, int64_t record_bytes, int parts, int nq, int k,
                                      int64_t* out_ids, float* out_scores, float* out_minmax, crag_stream_t stream) {
  const int64_t a = int64_t(nq) * k * 8, b = a + int64_t(nq) * k * 4, need = b + int64_t(nq) * 2 * 4;
  if (record_bytes < need || record_bytes % 8) return crag::fail(CRAG_ERR_INVALID, "crag_merge_topk_packed: record_bytes %lld < %lld or not a multiple of 8", (long long)record_bytes, (long long)need);
  if (!records && parts > 0) return crag::fail(CRAG_ERR_INVALID, "crag_merge_topk_packed: null pointer");
  const char* base = static_cast<const char*>(records);
  return crag::merge_pairs(reinterpret_cast<const float*>(base + a), reinterpret_cast<const int64_t*>(base),
                           reinterpret_cast<const float*>(base + b), record_bytes, record_bytes, record_bytes, parts, nq, k,
                           out_ids, out_scores, out_minmax, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ score-all pass
namespace crag {
namespace {
// (min, max) over the per-CTA partials of a score-all pass: one warp per query.
__global__ void minmax_reduce_kernel(const float* __restrict__ part_minmax, int parts, int nq, float* __restrict__ out) {
  const int q = blockIdx.x, lane = threadIdx.x;
  if (q >= nq) return;
  float a = INFINITY, b = -INFINITY;
  for (int p = lane; p < parts; p += 32) {
    a = fminf(a, part_minmax[(size_t(p) * kNQ + q) * 2 + 0]);
    b = fmaxf(b, part_minmax[(size_t(p) * kNQ + q) * 2 + 1]);
  }
  warp_minmax(a, b);
  if (lane == 0) {
    out[size_t(q) * 2 + 0] = a;
    out[size_t(q) * 2 + 1] = b;
  }
}

// Score-all passes (the scan with SCORES), one per block of 32 queries.  Block q0 stores its scores from row q0 of
// sa.out on, or, in assignment mode (sa.best_id set), updates every row's running argmax with ids counted from q0.
// out_minmax (may be null) receives each query's (min, max).
int score_passes(const void* corpus, int64_t n_rows, int dim, int64_t row_stride, const void* queries, int nq,
                 ScoreArgs sa, float* out_minmax, void* workspace, const SearchPlan& plan, cudaStream_t stream) {
  const int grid = scan_grid(n_rows, plan);
  if (grid == 0) {
    if (out_minmax) {   // empty shard: (+inf, -inf), as crag_search_topk
      minmax_reduce_kernel<<<nq, 32, 0, stream>>>(nullptr, 0, nq, out_minmax);
      CRAG_CUDA_OK(cudaGetLastError());
    }
    return CRAG_OK;
  }
  float* part_minmax = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + plan.keys_bytes);
  CUtensorMap tm_corpus;
  int rc = make_tmap_bf16_2d(&tm_corpus, corpus, uint64_t(n_rows), uint64_t(dim), uint64_t(row_stride) * 2, kTileRows);
  if (rc != CRAG_OK) return rc;
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    CUtensorMap tm_q;
    rc = make_query_tmap(&tm_q, queries, q0, nqc, dim);
    if (rc != CRAG_OK) return rc;
    ScoreArgs pass = sa;
    if (sa.best_id) pass.base_id = q0;
    else pass.out = sa.out + int64_t(q0) * sa.ld;
    rc = launch_scan<16, 16, 7, false, true>(tm_corpus, tm_q, int(n_rows), dim / kBlockK, nqc, 1, grid, nullptr, nullptr, 0u, 0, nullptr, part_minmax, pass, stream);
    if (rc != CRAG_OK) return rc;
    if (out_minmax) {
      minmax_reduce_kernel<<<nqc, 32, 0, stream>>>(part_minmax, grid, nqc, out_minmax + size_t(q0) * 2);
      CRAG_CUDA_OK(cudaGetLastError());
    }
  }
  return CRAG_OK;
}
}  // namespace
}  // namespace crag

extern "C" int crag_search_scores(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                  const void* queries, int nq, float* out_scores, int64_t out_ld, float* out_minmax,
                                  void* workspace, size_t workspace_bytes, crag_stream_t stream) {
  const SearchPlan plan = plan_search(1);
  int rc = check_search_args(corpus, n_rows, dim, corpus_row_stride, queries, nq, 1, workspace, workspace_bytes, plan);
  if (rc != CRAG_OK) return rc;
  if (!out_scores || out_ld < n_rows) return fail(CRAG_ERR_INVALID, "crag_search_scores: need out_scores and out_ld >= n_rows");
  return score_passes(corpus, n_rows, dim, corpus_row_stride, queries, nq, ScoreArgs{out_scores, out_ld, nullptr, nullptr, 0}, out_minmax, workspace,
                      plan, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ fused finalize + exchange (row-sharded index)
extern "C" size_t crag_exchange_buffer_bytes(int world) {
  if (world < 1 || world > kXMaxWorld) return 0;
  return (xchg_total_bytes(world) + 255) & ~size_t(255);
}

extern "C" int crag_search_finalize_exchange(const void* workspace, size_t workspace_bytes, int64_t n_rows, int nq, int k,
                                             int64_t row_offset, const uint64_t* peer_bufs, int rank, int world,
                                             uint64_t* epochs, int* status, int64_t* out_ids, float* out_scores,
                                             float* out_minmax, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (nq < 1 || nq > kNQ || k < 1 || k > 128) return fail(CRAG_ERR_INVALID, "crag_search_finalize_exchange: bad nq/k (nq=%d k=%d)", nq, k);
  if (world < 1 || world > kXMaxWorld || rank < 0 || rank >= world) return fail(CRAG_ERR_INVALID, "crag_search_finalize_exchange: bad rank/world (%d/%d)", rank, world);
  if (!workspace || !peer_bufs || !epochs || !status || !out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "crag_search_finalize_exchange: null pointer");
  const SearchPlan plan = plan_search(k);
  if (workspace_bytes < plan.keys_bytes + plan.minmax_bytes) return fail(CRAG_ERR_WORKSPACE, "crag_search_finalize_exchange: workspace too small");
  const uint64_t* part_keys = static_cast<const uint64_t*>(workspace);
  const float* part_minmax = reinterpret_cast<const float*>(static_cast<const uint8_t*>(workspace) + plan.keys_bytes);
  const int parts = scan_grid(n_rows, plan);
  with_merge_tier(k, [&](auto tier) {   // one CTA per query
    constexpr int T = decltype(tier)::value;
    finalize_exchange_kernel<T, T><<<nq, 128, 0, stream>>>(part_keys, part_minmax, parts, nq, k, row_offset, peer_bufs, rank,
                                                           world, epochs, status, out_ids, out_scores, out_minmax);
  });
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

// IVF build, assignment step: list of every row = argmax over the centroid table of bf16(row) . bf16(centroid) with fp32
// accumulation, ties to the smaller list id (oracle/ivf_oracle.py `assign`).  The rows are the "corpus" of the scan
// kernel and the centroids its query blocks (32 per pass): nlist / 32 passes over the rows, each row keeping its
// running best in (best_score, best_id).  Replaces a torch matmul + argmax over [rows, nlist] score blocks.
extern "C" int crag_ivf_assign(const void* rows, int64_t n_rows, int dim, int64_t row_stride, const void* centroids,
                               int nlist, float* best_score, int32_t* best_id, void* workspace, size_t workspace_bytes,
                               crag_stream_t stream) {
  const SearchPlan plan = plan_search(1);
  int rc = check_search_args(rows, n_rows, dim, row_stride, centroids, nlist, 1, workspace, workspace_bytes, plan);
  if (rc != CRAG_OK) return rc;
  if (!best_score || !best_id) return fail(CRAG_ERR_INVALID, "crag_ivf_assign: null output pointer");
  // the pass over centroid block 0 initialises every row's running best (-inf, list 0); later passes update it
  return score_passes(rows, n_rows, dim, row_stride, centroids, nlist, ScoreArgs{nullptr, 0, best_score, best_id, 0}, nullptr, workspace, plan,
                      static_cast<cudaStream_t>(stream));
}
