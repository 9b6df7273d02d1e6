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
// Variants of the same pipeline, named by the kernel's argument struct: IvfArgs walks a work-list of probed tiles
// (crag_ivf_search); ScoreArgs stores every score (crag_search_scores) or keeps each row's running argmax over centroid
// blocks (crag_ivf_assign); I8Args scans int8 rows (crag_search_topk_i8), I8IvfArgs int8 IVF lists (crag_ivf_search_i8).
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
#include "workspace.cuh"

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

// Int8 variant of the flat top-k scan (I8Args, crag_search_topk_i8): the shard and the query block are int8 with one
// fp32 scale per row / query (quant_kernels.cuh).  A 128-byte swizzle row holds 128 int8 instead of 64 bf16, so boxes,
// stages, descriptors and score tiles keep their byte sizes; the warpgroup issues m64n32k32.s32.s8.s8 and its epilogue
// writes S1 = float(acc) * (s_q * s_row) to the score tile, which the select warps rank as they rank bf16 scores.
struct I8Args {
  const float* row_scales;     // [n_rows], 0 on IVF padding rows
  const float* query_scales;   // [nq] of this pass
};
// The int8 IVF scan (crag_ivf_search_i8): the select warps read the IvfArgs part, the wgmma warpgroup the scales.
struct I8IvfArgs : IvfArgs, I8Args {};
template <class Args> constexpr bool kI8Scan = std::is_base_of<I8Args, Args>::value;

template <int KLIST, int CAP, int STAGES, class Args>
__global__ void __launch_bounds__(kSearchThreads, 1)
search_topk_kernel(const __grid_constant__ CUtensorMap tm_corpus, const __grid_constant__ CUtensorMap tm_q,
                   int n_rows, int num_kb, int nq, int k, const uint64_t* __restrict__ after_keys,
                   uint64_t* __restrict__ pool, uint32_t perm_mul, int perm_shift, uint64_t* __restrict__ part_keys,
                   float* __restrict__ part_minmax, const Args args) {
  constexpr bool IVF = kIvfScan<Args>, SCORES = kScoreScan<Args>, I8 = kI8Scan<Args>;
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
    select_warps<KLIST, CAP, IVF, SCORES>(sel, tiles, order, num_tiles, n_rows, nq, k, after_keys, pool, part_keys, part_minmax, args, warp, lane);
  }
}

// ------------------------------------------------------------------ host side
namespace {

// Workspace of a flat scan, per 32-query pass: the per-CTA partial keys and (min, max), then the pooled-floor table
// (0 bytes when the grid exceeds kPoolMaxCtas).  Every scan needs the partials; a flat scan uses the table if it fits.
struct SearchPlan {
  int grid;
  uint64_t* part_keys;
  float* part_minmax;
  size_t parts_bytes;
  uint64_t* pool;       // null without a table
  size_t pool_bytes;
  size_t total;
};

SearchPlan plan_search(int k, const void* ws = nullptr) {
  SearchPlan p;
  p.grid = sm_count();
  if (p.grid <= 0) p.grid = 132;
  WsCursor c(ws);
  p.part_keys = c.take<uint64_t>(size_t(p.grid) * kNQ * k);
  p.part_minmax = c.take<float>(size_t(p.grid) * kNQ * 2);
  p.parts_bytes = c.bytes;
  const bool pooled = p.grid <= kPoolMaxCtas;
  uint64_t* pool = c.take<uint64_t>(pooled ? size_t(kNQ) * p.grid * kPoolSlots : 0);
  p.pool = pooled ? pool : nullptr;
  p.pool_bytes = c.bytes - p.parts_bytes;
  p.total = c.bytes;
  return p;
}

// One launch of the scan.  The dynamic shared-memory limit is raised once per instantiation and device.
template <int KLIST, int CAP, int STAGES, class Args>
int launch_scan(const CUtensorMap& tm_corpus, const CUtensorMap& tm_q, int n_rows, int num_kb, int nq, int k, int grid,
                const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul, int perm_shift, uint64_t* part_keys,
                float* part_minmax, const Args& args, cudaStream_t stream) {
  constexpr size_t smem = SearchLayout<KLIST, CAP, STAGES>::smem_bytes();
  auto kern = search_topk_kernel<KLIST, CAP, STAGES, Args>;
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
template <class Args>
int launch_topk_scan(const CUtensorMap& tm_corpus, const CUtensorMap& tm_q, int n_rows, int num_kb, int nq, int k,
                     int grid, const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul, int perm_shift,
                     uint64_t* part_keys, float* part_minmax, const Args& args, cudaStream_t stream) {
  if (k <= 64) return launch_scan<64, 64, 6>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
  return launch_scan<128, 128, 4>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
}

// The merge kernels' list size for k (32, 64 or 128), passed to `launch` as a std::integral_constant.
template <class Launch>
void with_merge_tier(int k, Launch launch) {
  if (k <= 32) launch(std::integral_constant<int, 32>{});
  else if (k <= 64) launch(std::integral_constant<int, 64>{});
  else launch(std::integral_constant<int, 128>{});
}

// the scan arguments of the pass over queries q0 .. q0 + 31: the int8 scans read the scales of that pass's queries
template <class Args>
Args pass_args(Args args, int q0) {
  if constexpr (kI8Scan<Args>) args.query_scales += q0;
  return args;
}

// A scan operand: `rows` rows of `width` elements, `stride` elements apart; `name` heads its error messages.
enum Elem { kS8 = 1, kBf16 = 2 };   // bytes per element
struct Operand {
  const void* ptr;
  int64_t rows;
  int width;
  int64_t stride;
  Elem elem;
  const char* name;
  Operand rows_from(int64_t r0, int64_t n) const { return {static_cast<const uint8_t*>(ptr) + r0 * stride * elem, n, width, stride, elem, name}; }
  int num_kb() const { return width * elem / 128; }   // 128-byte swizzle rows per row
};

// The scan's rules for an operand, in bytes: 1 to 1024 elements per row in whole 128-byte swizzle rows (bf16 dim % 64,
// int8 dim % 128), a row stride of whole 16 bytes, a 16-byte aligned base and row indices that fit an int.
int check_operand(const char* who, const Operand& op) {
  if (op.width < 1 || op.width > 1024 || op.width * op.elem % 128 != 0) return fail(CRAG_ERR_INVALID, "%s: %s dim must be a multiple of %d in [%d, 1024] (dim=%d)", who, op.name, 128 / op.elem, 128 / op.elem, op.width);
  if (op.rows < 0 || op.rows >= (int64_t(1) << 31) - kTileRows) return fail(CRAG_ERR_INVALID, "%s: %s n_rows out of range (%lld)", who, op.name, (long long)op.rows);
  if (op.stride < op.width || op.stride * op.elem % 16 != 0) return fail(CRAG_ERR_INVALID, "%s: %s row stride must be >= dim and a multiple of %d", who, op.name, 16 / op.elem);
  if (op.rows > 0 && !op.ptr) return fail(CRAG_ERR_INVALID, "%s: null %s pointer", who, op.name);
  if (reinterpret_cast<uintptr_t>(op.ptr) & 15) return fail(CRAG_ERR_INVALID, "%s: %s must be 16-byte aligned", who, op.name);
  return CRAG_OK;
}

// nq and k, the shard and query operands of a scan, and a 256-byte aligned workspace of at least `need` bytes
int check_scan_args(const char* who, int nq, int k, int k_max, const Operand& corpus, const Operand& queries,
                    const void* workspace, size_t workspace_bytes, size_t need) {
  if (nq < 1 || k < 1 || k > k_max) return fail(CRAG_ERR_INVALID, "%s: need nq >= 1 and 1 <= k <= %d (nq=%d k=%d)", who, k_max, nq, k);
  int rc = check_operand(who, corpus);
  if (rc == CRAG_OK) rc = check_operand(who, queries);
  if (rc != CRAG_OK) return rc;
  return check_workspace(who, workspace, workspace_bytes, need);
}

// TMA map of an operand in boxes of box_rows rows by one 128-byte swizzle row
int make_tmap(CUtensorMap* tm, const Operand& op, uint32_t box_rows) {
  if (op.elem == kS8) return make_tmap_u8_2d(tm, op.ptr, uint64_t(op.rows), uint64_t(op.width), uint64_t(op.stride), box_rows);
  return make_tmap_bf16_2d(tm, op.ptr, uint64_t(op.rows), uint64_t(op.width), uint64_t(op.stride) * 2, box_rows);
}

}  // namespace
}  // namespace crag

using namespace crag;

extern "C" size_t crag_search_workspace_bytes(int nq, int k) {
  (void)nq;
  if (k < 1 || k > 128) return 0;
  return plan_search(k).total;
}

namespace crag {
namespace {

inline int scan_grid(int64_t n_rows, const SearchPlan& plan) {
  const int num_tiles = int((n_rows + kTileRows - 1) / kTileRows);
  return num_tiles < plan.grid ? num_tiles : plan.grid;
}

// the flat scans permute groups of 2^kPermShift consecutive tiles (TileOrder)
constexpr int kPermShift = 3;

// one corpus pass for the <= 32 queries of `queries`: per-CTA partial lists into the workspace
template <class Args>
int scan_pass(const Operand& corpus, const Operand& queries, int k, const uint64_t* after_keys, const Args& args,
              size_t workspace_bytes, const SearchPlan& plan, cudaStream_t stream) {
  const int grid = scan_grid(corpus.rows, plan);
  if (grid == 0) return CRAG_OK;
  // pooled floor: needs its table in the workspace and pays off once a CTA sees more than a couple of tiles
  uint64_t* pool = nullptr;
  const int64_t num_tiles = (corpus.rows + kTileRows - 1) / kTileRows;
  if (plan.pool && workspace_bytes >= plan.total && num_tiles >= 4 * int64_t(grid)) {
    pool = plan.pool;
    CRAG_CUDA_OK(cudaMemsetAsync(pool, 0, plan.pool_bytes, stream));
  }
  CUtensorMap tm_corpus, tm_q;
  int rc = make_tmap(&tm_corpus, corpus, kTileRows);
  if (rc == CRAG_OK) rc = make_tmap(&tm_q, queries, kNQ);
  if (rc != CRAG_OK) return rc;
  return launch_topk_scan(tm_corpus, tm_q, int(corpus.rows), corpus.num_kb(), int(queries.rows), k, grid, after_keys, pool,
                          perm_multiplier(num_tiles >> kPermShift), kPermShift, plan.part_keys, plan.part_minmax, args, stream);
}

// merge the per-CTA partials of one pass into the final (ids, scores, minmax) of its <= 32 queries
int finalize_parts(int grid, int nq, int k, int64_t row_offset, int64_t* out_ids, float* out_scores, float* out_minmax,
                   uint64_t* last_keys, const SearchPlan& plan, cudaStream_t stream) {
  with_merge_tier(k, [&](auto tier) {   // one CTA per query
    constexpr int T = decltype(tier)::value;
    merge_topk_kernel<T, T, false><<<nq, 128, 0, stream>>>(plan.part_keys, nullptr, nullptr, plan.part_minmax, grid, kNQ, nq, k, row_offset, 0, 0, 0,
                                                           out_ids, out_scores, out_minmax, last_keys);
  });
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

// every 32-query pass of a flat top-k scan: the scan, then the merge of its partials into the outputs
template <class Args>
int topk_passes(const Operand& corpus, const Operand& queries, int k, int64_t row_offset, const uint64_t* after_keys,
                const Args& args, int64_t* out_ids, float* out_scores, float* out_minmax, uint64_t* last_keys,
                size_t workspace_bytes, const SearchPlan& plan, cudaStream_t stream) {
  const int nq = int(queries.rows);
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    int rc = scan_pass(corpus, queries.rows_from(q0, nqc), k, after_keys ? after_keys + q0 : nullptr, pass_args(args, q0),
                       workspace_bytes, plan, stream);
    if (rc == CRAG_OK)
      rc = finalize_parts(scan_grid(corpus.rows, plan), nqc, k, row_offset, out_ids + size_t(q0) * k, out_scores + size_t(q0) * k,
                         out_minmax ? out_minmax + size_t(q0) * 2 : nullptr, last_keys ? last_keys + q0 : nullptr, plan, stream);
    if (rc != CRAG_OK) return rc;
  }
  return CRAG_OK;
}

// IVF workspace = the flat scan's, then the per-pass plan of the probed tiles
struct IvfPlan {
  SearchPlan scan;
  uint32_t* list_mask;
  float* coarse;
  int4* work;
  int* n_work;
  size_t total;
};
IvfPlan plan_ivf(int k, int nlist, int64_t total_tiles, const void* ws = nullptr) {
  IvfPlan p;
  p.scan = plan_search(k, ws);
  WsCursor c(ws, p.scan.total);
  p.list_mask = c.take<uint32_t>(size_t(nlist));
  p.coarse = c.take<float>(size_t(nlist) * kNQ);
  p.work = c.take<int4>(size_t(total_tiles));
  p.n_work = c.take<int>(1);
  p.total = c.bytes;
  return p;
}

// int8 IVF workspace = the IVF workspace for n_cand keys, then the candidates of one pass
struct IvfI8Plan {
  IvfPlan ivf;
  int64_t* cand_ids;
  float* cand_scores;
  size_t total;
};
IvfI8Plan plan_ivf_i8(int nlist, int64_t total_tiles, int n_cand, const void* ws = nullptr) {
  IvfI8Plan p;
  p.ivf = plan_ivf(n_cand, nlist, total_tiles, ws);
  WsCursor c(ws, p.ivf.total);
  p.cand_ids = c.take<int64_t>(size_t(kNQ) * n_cand);
  p.cand_scores = c.take<float>(size_t(kNQ) * n_cand);
  p.total = c.bytes;
  return p;
}

struct IvfLists {   // the list tables and probes of an IVF search, as crag_ivf_search takes them
  const int32_t* tile_start;
  const int32_t* rows;
  int nlist;
  int64_t total_tiles;
  const int64_t* row_ids;
  const int64_t* probed_ids;
  const float* probed_scores;
  int nprobe;
};

// the lists, the probes and the outputs of an IVF search over n_rows_padded stored rows in whole tiles
int check_ivf_args(const char* who, const IvfLists& l, int64_t n_rows_padded, const int64_t* out_ids, const float* out_scores) {
  if (l.nlist < 1 || l.nlist > (1 << 20) || l.nprobe < 1 || l.nprobe > l.nlist) return fail(CRAG_ERR_INVALID, "%s: need 1 <= nprobe <= nlist <= 2^20 (nprobe=%d nlist=%d)", who, l.nprobe, l.nlist);
  if (l.total_tiles < 1 || l.total_tiles * kTileRows != n_rows_padded) return fail(CRAG_ERR_INVALID, "%s: need n_rows_padded (%lld) = total_tiles (%lld) * %d, non-empty", who, (long long)n_rows_padded, (long long)l.total_tiles, kTileRows);
  if (!l.tile_start || !l.rows || !l.row_ids || !l.probed_ids || !l.probed_scores || !out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "%s: null pointer", who);
  return CRAG_OK;
}

// crag_ivf_search_i8's exact rescore: bf16 residuals (device address) and queries, and the candidates' workspace buffers
struct IvfRescore {
  Operand rows, queries;
  int64_t* cand_ids;
  float* cand_scores;
};

// Every 32-query pass of an IVF search over the residuals `res`: the plan of the probed tiles, the scan for n_scan keys
// per query, the merge of its partials, then the map of stored positions to original ids.  With `rescore` the merge
// writes n_scan candidates, which the exact rescore (quant.cu) turns into the k results, with the plan's coarse terms.
template <class Args>
int ivf_passes(const Operand& res, const Operand& queries, Args args, const IvfLists& l, int n_scan, int k,
               const IvfRescore* rescore, int64_t* out_ids, float* out_scores, float* out_minmax, const IvfPlan& ip,
               cudaStream_t stream) {
  const SearchPlan& sp = ip.scan;
  static_cast<IvfArgs&>(args) = IvfArgs{ip.work, ip.n_work, ip.list_mask, ip.coarse};
  CUtensorMap tm_res;
  int rc = make_tmap(&tm_res, res, kTileRows);
  if (rc != CRAG_OK) return rc;
  const int nq = int(queries.rows);
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    CUtensorMap tm_q;
    rc = make_tmap(&tm_q, queries.rows_from(q0, nqc), kNQ);
    if (rc != CRAG_OK) return rc;
    ivf_plan_kernel<<<1, 1024, 0, stream>>>(l.probed_ids + size_t(q0) * l.nprobe, l.probed_scores + size_t(q0) * l.nprobe, nqc,
                                            l.nprobe, l.nlist, l.tile_start, l.rows, ip.list_mask, ip.coarse, ip.work,
                                            ip.n_work);
    CRAG_CUDA_OK(cudaGetLastError());
    // every CTA of the grid publishes a (possibly empty) partial list, so the merge always reads sp.grid parts
    if (sp.pool) CRAG_CUDA_OK(cudaMemsetAsync(sp.pool, 0, sp.pool_bytes, stream));
    rc = launch_topk_scan(tm_res, tm_q, int(res.rows), res.num_kb(), nqc, n_scan, sp.grid, nullptr, sp.pool, 0u, 0,
                          sp.part_keys, sp.part_minmax, pass_args(args, q0), stream);
    if (rc != CRAG_OK) return rc;
    int64_t* ids = out_ids + size_t(q0) * k;
    float* scores = out_scores + size_t(q0) * k;
    float* minmax = out_minmax ? out_minmax + size_t(q0) * 2 : nullptr;
    if (!rescore) {
      rc = finalize_parts(sp.grid, nqc, k, 0, ids, scores, minmax, nullptr, sp, stream);
    } else {
      rc = finalize_parts(sp.grid, nqc, n_scan, 0, rescore->cand_ids, rescore->cand_scores, minmax, nullptr, sp, stream);
      if (rc == CRAG_OK)
        rc = launch_ivf_rescore(rescore->rows.ptr, rescore->rows.rows, rescore->rows.width, rescore->rows.stride,
                                rescore->queries.rows_from(q0, nqc).ptr, nqc, rescore->cand_ids, n_scan, k, l.tile_start,
                                l.nlist, ip.coarse, ids, scores, stream);
    }
    if (rc != CRAG_OK) return rc;
    ivf_map_ids_kernel<<<(nqc * k + 255) / 256, 256, 0, stream>>>(ids, nqc * k, l.row_ids);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}

}  // namespace
}  // namespace crag

extern "C" size_t crag_ivf_workspace_bytes(int nlist, int64_t total_tiles, int k) {
  if (nlist < 1 || total_tiles < 0 || k < 1 || k > 128) return 0;
  return plan_ivf(k, nlist, total_tiles).total;
}

extern "C" int crag_ivf_search(const void* residuals, int64_t n_rows_padded, int dim, int64_t row_stride,
                               const int32_t* list_tile_start, const int32_t* list_rows, int nlist,
                               int64_t total_tiles, const int64_t* row_ids, const void* queries, int nq,
                               const int64_t* probed_ids, const float* probed_scores, int nprobe, int k,
                               int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                               size_t workspace_bytes, crag_stream_t stream) {
  const Operand res{residuals, n_rows_padded, dim, row_stride, kBf16, "residuals"}, q{queries, nq, dim, dim, kBf16, "queries"};
  const IvfLists lists{list_tile_start, list_rows, nlist, total_tiles, row_ids, probed_ids, probed_scores, nprobe};
  int rc = check_ivf_args("ivf", lists, n_rows_padded, out_ids, out_scores);
  if (rc != CRAG_OK) return rc;
  const IvfPlan ip = plan_ivf(k >= 1 && k <= 128 ? k : 1, nlist, total_tiles, workspace);
  rc = check_scan_args("ivf", nq, k, 128, res, q, workspace, workspace_bytes, ip.total);
  if (rc != CRAG_OK) return rc;
  return ivf_passes(res, q, IvfArgs{}, lists, k, k, nullptr, out_ids, out_scores, out_minmax, ip,
                    static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ IVF over int8 residuals (ivf_passes with a rescore)
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
                                  size_t workspace_bytes, crag_stream_t stream) {
  const Operand res{residuals_i8, n_rows_padded, dim8, row_stride_i8, kS8, "residuals_i8"}, q{queries_i8, nq, dim8, dim8, kS8, "queries_i8"};
  IvfRescore rescore{{residuals_bf16, n_rows_padded, dim, row_stride, kBf16, "residuals_bf16"},
                     {queries_bf16, nq, dim, dim, kBf16, "queries_bf16"}, nullptr, nullptr};
  const IvfLists lists{list_tile_start, list_rows, nlist, total_tiles, row_ids, probed_ids, probed_scores, nprobe};
  int rc = check_ivf_args("ivf_i8", lists, n_rows_padded, out_ids, out_scores);
  if (rc != CRAG_OK) return rc;
  if (nq < 1 || k < 1 || n_cand < k || n_cand > 128) return fail(CRAG_ERR_INVALID, "ivf_i8: need nq >= 1 and 1 <= k <= n_cand <= 128 (nq=%d k=%d n_cand=%d)", nq, k, n_cand);
  if (dim8 != (dim + 127) / 128 * 128) return fail(CRAG_ERR_INVALID, "ivf_i8: dim8 must be dim rounded up to a multiple of 128 (dim=%d dim8=%d)", dim, dim8);
  const IvfI8Plan plan = plan_ivf_i8(nlist, total_tiles, n_cand, workspace);
  rc = check_scan_args("ivf_i8", nq, n_cand, 128, res, q, workspace, workspace_bytes, plan.total);
  if (rc == CRAG_OK) rc = check_operand("ivf_i8", rescore.rows);
  if (rc == CRAG_OK) rc = check_operand("ivf_i8", rescore.queries);
  if (rc != CRAG_OK) return rc;
  if (!row_scales || !query_scales) return fail(CRAG_ERR_INVALID, "ivf_i8: null pointer");
  // the bf16 residuals may be page-locked host memory: refused before any launch if pageable
  rc = device_readable(residuals_bf16, &rescore.rows.ptr, "ivf_i8");
  if (rc != CRAG_OK) return rc;
  rescore.cand_ids = plan.cand_ids;
  rescore.cand_scores = plan.cand_scores;
  return ivf_passes(res, q, I8IvfArgs{{}, {row_scales, query_scales}}, lists, n_cand, k, &rescore, out_ids, out_scores, out_minmax, plan.ivf,
                    static_cast<cudaStream_t>(stream));
}

extern "C" int crag_search_scan(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                const void* queries, int nq, int k, void* workspace, size_t workspace_bytes,
                                crag_stream_t stream) {
  const Operand c{corpus, n_rows, dim, corpus_row_stride, kBf16, "corpus"}, q{queries, nq, dim, dim, kBf16, "queries"};
  const SearchPlan plan = plan_search(k >= 1 && k <= 128 ? k : 1, workspace);
  int rc = check_scan_args("search", nq, k, 128, c, q, workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  if (nq > kNQ) return fail(CRAG_ERR_INVALID, "crag_search_scan handles one pass of at most %d queries (nq=%d)", kNQ, nq);
  return scan_pass(c, q, k, nullptr, NoIvfArgs{}, workspace_bytes, plan, static_cast<cudaStream_t>(stream));
}

extern "C" int crag_search_finalize(const void* workspace, size_t workspace_bytes, int64_t n_rows, int nq, int k,
                                    int64_t row_offset, int64_t* out_ids, float* out_scores, float* out_minmax,
                                    crag_stream_t stream) {
  if (nq < 1 || nq > kNQ || k < 1 || k > 128) return fail(CRAG_ERR_INVALID, "crag_search_finalize: bad nq/k (nq=%d k=%d)", nq, k);
  const SearchPlan plan = plan_search(k, workspace);
  if (!out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "crag_search_finalize: null pointer");
  const int rc = check_workspace("crag_search_finalize", workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  return finalize_parts(scan_grid(n_rows, plan), nq, k, row_offset, out_ids, out_scores, out_minmax, nullptr, plan,
                        static_cast<cudaStream_t>(stream));
}

extern "C" int crag_search_topk_after(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                      int64_t row_offset, const void* queries, int nq, int k,
                                      const uint64_t* after_keys, int64_t* out_ids, float* out_scores,
                                      float* out_minmax, uint64_t* last_keys, void* workspace,
                                      size_t workspace_bytes, crag_stream_t stream) {
  const Operand c{corpus, n_rows, dim, corpus_row_stride, kBf16, "corpus"}, q{queries, nq, dim, dim, kBf16, "queries"};
  const SearchPlan plan = plan_search(k >= 1 && k <= 128 ? k : 1, workspace);
  int rc = check_scan_args("search", nq, k, 128, c, q, workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  if (!out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "search: null output pointer");
  return topk_passes(c, q, k, row_offset, after_keys, NoIvfArgs{}, out_ids, out_scores, out_minmax, last_keys,
                     workspace_bytes, plan, static_cast<cudaStream_t>(stream));
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
                                   float* out_minmax, void* workspace, size_t workspace_bytes, crag_stream_t stream) {
  const Operand c{corpus_i8, n_rows, dim8, row_stride, kS8, "corpus"}, q{queries_i8, nq, dim8, dim8, kS8, "queries"};
  const SearchPlan plan = plan_search(k >= 1 && k <= 128 ? k : 1, workspace);
  int rc = check_scan_args("search_i8", nq, k, 128, c, q, workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  if (!query_scales || !out_ids || !out_scores || (n_rows > 0 && !row_scales)) return fail(CRAG_ERR_INVALID, "search_i8: null pointer");
  return topk_passes(c, q, k, row_offset, nullptr, I8Args{row_scales, query_scales}, out_ids, out_scores, out_minmax,
                     nullptr, workspace_bytes, plan, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ exact top-k for large k / many queries
// Per chunk of queries: the wgmma GEMM writes the fp32 score block [q_chunk, ld] into the workspace
// (gemm_scores_f32), then knn_select_kernel (knn_select.cuh) radix-selects each query's k best rows from its row.
namespace crag {
namespace {
inline int64_t knn_ld(int64_t n_rows) { return ((n_rows > 0 ? n_rows : 1) + 3) & ~int64_t(3); }

// Workspace of crag_knn_topk: the fp32 score block [q_chunk][knn_ld(n_rows)]
struct KnnWorkspace { float* block; size_t total; };
KnnWorkspace knn_workspace(int64_t n_rows, int q_chunk, void* ws = nullptr) {
  WsCursor c(ws);
  KnnWorkspace w;
  w.block = c.take<float>(size_t(q_chunk) * size_t(knn_ld(n_rows)));
  w.total = c.bytes;
  return w;
}
}  // namespace
}  // namespace crag

extern "C" size_t crag_knn_workspace_bytes(int64_t n_rows, int q_chunk) {
  if (n_rows < 0 || q_chunk < 1) return 0;
  return knn_workspace(n_rows, q_chunk).total;
}

extern "C" int crag_knn_topk(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride, int64_t row_offset,
                             const void* queries, int nq, int k, int64_t* out_ids, float* out_scores, float* out_minmax,
                             void* workspace, size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const Operand c{corpus, n_rows, dim, corpus_row_stride, kBf16, "corpus"}, q{queries, nq, dim, dim, kBf16, "queries"};
  int rc = check_scan_args("search", nq, k, kKnnMaxK, c, q, workspace, workspace_bytes, 0);
  if (rc != CRAG_OK) return rc;
  if (!out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "knn: null output pointer");
  const int64_t ld = knn_ld(n_rows);
  const size_t per_query = size_t(ld) * 4;
  const size_t fit = workspace_bytes / per_query;
  if (fit < 1) return fail(CRAG_ERR_WORKSPACE, "knn: workspace %zu < %zu bytes (one query's score row)", workspace_bytes, per_query);
  const int q_chunk = fit < size_t(nq) ? int(fit) : nq;
  float* block = knn_workspace(n_rows, q_chunk, workspace).block;
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

// Score-all passes (the scan with ScoreArgs), one per block of 32 queries.  Block q0 stores its scores from row q0 of
// sa.out on, or, in assignment mode (sa.best_id set), updates every row's running argmax with ids counted from q0.
// out_minmax (may be null) receives each query's (min, max).
int score_passes(const Operand& corpus, const Operand& queries, ScoreArgs sa, float* out_minmax, const SearchPlan& plan,
                 cudaStream_t stream) {
  const int nq = int(queries.rows);
  const int grid = scan_grid(corpus.rows, plan);
  if (grid == 0) {
    if (out_minmax) {   // empty shard: (+inf, -inf), as crag_search_topk
      minmax_reduce_kernel<<<nq, 32, 0, stream>>>(nullptr, 0, nq, out_minmax);
      CRAG_CUDA_OK(cudaGetLastError());
    }
    return CRAG_OK;
  }
  CUtensorMap tm_corpus;
  int rc = make_tmap(&tm_corpus, corpus, kTileRows);
  if (rc != CRAG_OK) return rc;
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    CUtensorMap tm_q;
    rc = make_tmap(&tm_q, queries.rows_from(q0, nqc), kNQ);
    if (rc != CRAG_OK) return rc;
    ScoreArgs pass = sa;
    if (sa.best_id) pass.base_id = q0;
    else pass.out = sa.out + int64_t(q0) * sa.ld;
    rc = launch_scan<16, 16, 7>(tm_corpus, tm_q, int(corpus.rows), corpus.num_kb(), nqc, 1, grid, nullptr, nullptr, 0u, 0, nullptr, plan.part_minmax, pass, stream);
    if (rc != CRAG_OK) return rc;
    if (out_minmax) {
      minmax_reduce_kernel<<<nqc, 32, 0, stream>>>(plan.part_minmax, grid, nqc, out_minmax + size_t(q0) * 2);
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
  const Operand c{corpus, n_rows, dim, corpus_row_stride, kBf16, "corpus"}, q{queries, nq, dim, dim, kBf16, "queries"};
  const SearchPlan plan = plan_search(1, workspace);
  int rc = check_scan_args("search", nq, 1, 128, c, q, workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  if (!out_scores || out_ld < n_rows) return fail(CRAG_ERR_INVALID, "crag_search_scores: need out_scores and out_ld >= n_rows");
  return score_passes(c, q, ScoreArgs{out_scores, out_ld, nullptr, nullptr, 0}, out_minmax, plan,
                      static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ fused finalize + exchange (row-sharded index)
extern "C" size_t crag_exchange_buffer_bytes(int world) {
  if (world < 1 || world > kXMaxWorld) return 0;
  return ws_round(xchg_total_bytes(world));
}

extern "C" int crag_search_finalize_exchange(const void* workspace, size_t workspace_bytes, int64_t n_rows, int nq, int k,
                                             int64_t row_offset, const uint64_t* peer_bufs, int rank, int world,
                                             uint64_t* epochs, int* status, int64_t* out_ids, float* out_scores,
                                             float* out_minmax, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (nq < 1 || nq > kNQ || k < 1 || k > 128) return fail(CRAG_ERR_INVALID, "crag_search_finalize_exchange: bad nq/k (nq=%d k=%d)", nq, k);
  if (world < 1 || world > kXMaxWorld || rank < 0 || rank >= world) return fail(CRAG_ERR_INVALID, "crag_search_finalize_exchange: bad rank/world (%d/%d)", rank, world);
  if (!peer_bufs || !epochs || !status || !out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "crag_search_finalize_exchange: null pointer");
  const SearchPlan plan = plan_search(k, workspace);
  const int rc = check_workspace("crag_search_finalize_exchange", workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  const int parts = scan_grid(n_rows, plan);
  with_merge_tier(k, [&](auto tier) {   // one CTA per query
    constexpr int T = decltype(tier)::value;
    finalize_exchange_kernel<T, T><<<nq, 128, 0, stream>>>(plan.part_keys, plan.part_minmax, parts, nq, k, row_offset, peer_bufs, rank,
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
  const Operand c{rows, n_rows, dim, row_stride, kBf16, "rows"}, q{centroids, nlist, dim, dim, kBf16, "centroids"};
  const SearchPlan plan = plan_search(1, workspace);
  int rc = check_scan_args("search", nlist, 1, 128, c, q, workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  if (!best_score || !best_id) return fail(CRAG_ERR_INVALID, "crag_ivf_assign: null output pointer");
  // the pass over centroid block 0 initialises every row's running best (-inf, list 0); later passes update it
  return score_passes(c, q, ScoreArgs{nullptr, 0, best_score, best_id, 0}, nullptr, plan,
                      static_cast<cudaStream_t>(stream));
}
