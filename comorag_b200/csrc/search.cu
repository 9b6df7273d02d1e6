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
// blocks (crag_ivf_assign); I8Args scans int8 rows (crag_search_topk_i8), I8IvfArgs int8 IVF lists (crag_ivf_search_i8),
// B1Args one-bit rows (crag_search_topk_b1), CodeScoreArgs every S1 of int8 or one-bit rows (crag_knn_topk_i8 / _b1).
// Around it in this file: the per-shard merge (merge_topk_kernel), the fused
// finalize + NVLink exchange + global merge of the row-sharded index
// (finalize_exchange_kernel), the C-ABI entry points, and crag_knn_topk -- exact
// top-k up to k = 2048 for large query batches as a score-block GEMM (gemm.cu)
// plus a per-query radix select (knn_select.cuh), and crag_knn_threshold -- the same score block, then a per-query
// threshold join (knn_threshold.cuh).  crag_ivf_search_pq runs the IVF plan, then the PQ table and scan kernels
// (pq_kernels.cuh), then the same merge, rescore and id map as crag_ivf_search_i8.  Their _wide forms score every
// probed row into a block (ivf_wide_kernels.cuh) and radix-select up to 2048 candidates per query.
#include <algorithm>
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
#include "knn_threshold.cuh"
#include "pq_kernels.cuh"
#include "ivf_wide_kernels.cuh"
#include "binary.cuh"
#include "workspace.cuh"

namespace crag {

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
// One-bit variant (crag_search_topk_b1, binary.cuh): row_scales are the rows' alpha, the query block is int8 as for
// I8Args, and so is the epilogue.  A stage holds one tile's code rows (128 rows x 128 bytes, 1024 columns at most) and
// nothing else: the whole query block stays resident in shared memory, loaded once per launch, because streaming its
// slice with every tile would cost about twice the code bytes in L2 reads.  The warpgroup widens its own A fragments
// from the stage's bits and issues m64n32k32.s32.s8.s8 with A in registers.
struct B1Args : I8Args {};
template <class Args> constexpr bool kB1Scan = std::is_base_of<B1Args, Args>::value;

// Score-all over codes (crag_knn_topk_i8 / _b1): the int8 or one-bit scan's warpgroup and epilogue, so S1 is the same
// expression bit for bit, and the select warps' ScoreArgs branch, which stores out[q * ld + row].  The constructor
// leaves ScoreArgs' assignment mode (best_id) off: a running argmax over code rows is not a variant of the scan.
template <class Codes>
struct CodeScoreArgs : ScoreArgs, Codes {
  CodeScoreArgs(float* out, int64_t ld, const Codes& codes) : ScoreArgs{out, ld, nullptr, nullptr, 0}, Codes(codes) {}
};

// Dynamic shared memory of the scan, from a 1024-byte aligned base: the pipeline stages, (one-bit scan) the resident
// query block, the score tiles, the selector (select_warps.cuh), then the mbarriers.
template <int KLIST, int CAP, int STAGES, class Args>
struct SearchLayout {
  static constexpr bool kB1 = kB1Scan<Args>;
  static constexpr size_t kStage = kB1 ? size_t(kStageBytes) : size_t(kStageTotalBytes);
  static constexpr size_t kQueryOff = size_t(STAGES) * kStage;
  static constexpr size_t kTilesOff = kQueryOff + (kB1 ? size_t(kB1QueryBytes) : 0);
  static constexpr size_t kSelectOff = kTilesOff + size_t(kAccStages) * kScoreTileBytes;
  static constexpr size_t kBarsOff = kSelectOff + SelectSmem<KLIST, CAP>::bytes();
  static constexpr int kBars = 2 * STAGES + 2 * kAccStages + (kB1 ? 1 : 0);
  // + the alignment pad of the base and 16 bytes of slack past the mbarriers
  __host__ __device__ static constexpr size_t smem_bytes() { return 1024 + kBarsOff + kBars * 8 + 16; }
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

// The one-bit scan's MMA over one tile (B1Args): d[m] += A_m . Q^T over the num_kb 128-column chunks, A_m the +-1 rows
// m * 64 .. m * 64 + 63 of the tile widened from the stage's bits (b1_a_fragment), Q the resident query block.  The
// stage holds row r's 16-byte chunk kb at r * 128 + 16 (kb ^ r % 8) (TMA's 128-byte swizzle), so the 8 rows of one
// load of a warp fall on distinct banks.  Chunks alternate between two register sets: the next chunk is widened while
// the wgmma group of the current one runs, and only one group is in flight at a time, which is the pipelining ptxas
// keeps without serialising register-A wgmmas (a second group in flight while A registers are written makes it
// serialise them, C7513).
__device__ __forceinline__ void b1_tile_mma(int32_t (&d)[2][16], const uint8_t* stage, int frag_row, int lane,
                                            uint32_t q_addr, int num_kb) {
  const int t = lane & 3;
  const uint8_t* row0 = stage + frag_row * 128;   // this thread's rows frag_row, + 8, + 64, + 72
  const int sw = frag_row & 7;                    // = r % 8 for all four
  auto widen = [&](int kb, uint32_t (&a)[2][4][4]) {
    const int off = (kb ^ sw) << 4;
    const uint4 c[4] = {*reinterpret_cast<const uint4*>(row0 + off), *reinterpret_cast<const uint4*>(row0 + 8 * 128 + off),
                        *reinterpret_cast<const uint4*>(row0 + 64 * 128 + off), *reinterpret_cast<const uint4*>(row0 + 72 * 128 + off)};
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const uint32_t lo[4] = {c[2 * m].x, c[2 * m].y, c[2 * m].z, c[2 * m].w};
      const uint32_t hi[4] = {c[2 * m + 1].x, c[2 * m + 1].y, c[2 * m + 1].z, c[2 * m + 1].w};
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) b1_a_fragment(lo[ks], hi[ks], t, a[m][ks]);
    }
  };
  auto mma = [&](int kb, uint32_t (&a)[2][4][4]) {
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {   // 32-column k-steps: 32 bytes of the query box's rows
      const uint64_t db = wgmma_desc_sw128(q_addr + kb * kQBlockBytes + ks * 32);
      wgmma_m64n32k32_s8_rs(d[0], a[0][ks], db, 1u);
      wgmma_m64n32k32_s8_rs(d[1], a[1][ks], db, 1u);
    }
    wgmma_commit();
  };
  uint32_t a0[2][4][4], a1[2][4][4];
  widen(0, a0);
  for (int kb = 0; kb < num_kb; kb += 2) {
    mma(kb, a0);
    if (kb + 1 < num_kb) widen(kb + 1, a1);
    wgmma_wait<0>();
    if (kb + 1 < num_kb) mma(kb + 1, a1);
    if (kb + 2 < num_kb) widen(kb + 2, a0);
    wgmma_wait<0>();
  }
}

template <int KLIST, int CAP, int STAGES, class Args>
__global__ void __launch_bounds__(kSearchThreads, 1)
search_topk_kernel(const __grid_constant__ CUtensorMap tm_corpus, const __grid_constant__ CUtensorMap tm_q,
                   int n_rows, int num_kb, int nq, int k, const uint64_t* __restrict__ after_keys,
                   uint64_t* __restrict__ pool, uint32_t perm_mul, int perm_shift, uint64_t* __restrict__ part_keys,
                   float* __restrict__ part_minmax, const Args args) {
  constexpr bool IVF = kIvfScan<Args>, SCORES = kScoreScan<Args>, I8 = kI8Scan<Args>, B1 = kB1Scan<Args>;
  static_assert(!(B1 && IVF), "the one-bit scan has no IVF variant");
  // elements per 128-byte swizzle row: the producer's column step per k-block
  constexpr int kBlockElems = I8 ? 128 : kBlockK;
  using L = SearchLayout<KLIST, CAP, STAGES, Args>;
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
  uint64_t* bar_q = bar_tempty + kAccStages;           // B1: the resident query block has landed
  uint8_t* q_block = smem + L::kQueryOff;              // B1: num_kb boxes of 32 queries x 128 int8

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
    if constexpr (B1) mbar_init(bar_q, 1);
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
      if constexpr (B1) {   // the query block, once: num_kb boxes of 32 x 128 int8, 128-byte swizzled
        mbar_arrive_expect_tx(bar_q, uint32_t(num_kb) * kQBlockBytes);
        for (int kb = 0; kb < num_kb; ++kb) tma_load_2d(&tm_q, bar_q, q_block + kb * kQBlockBytes, kb * 128, 0);
      }
      for (int j = blockIdx.x; j < num_tiles; j += gridDim.x) {
        const int tile = IVF ? j : order(j);
        if constexpr (B1) {   // one box per tile: 128 code rows of 128 bytes (zero past dim8 / 8), 128-byte swizzled
          mbar_wait(&bar_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&bar_full[stage], kStageBytes);
          tma_load_2d_hint(&tm_corpus, &bar_full[stage], stage_base + stage * L::kStage, 0, tile * kTileRows, pol);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        for (int kb = 0; kb < (B1 ? 0 : num_kb); ++kb) {
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
    if constexpr (B1) mbar_wait(bar_q, 0);
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
      if constexpr (B1) {
        mbar_wait(&bar_full[stage], phase);
        b1_tile_mma(d, stage_base + stage * L::kStage, frag_row, lane, smem_u32(q_block), num_kb);
        __syncwarp();   // every lane has read its bits: the stage goes back to the producer
        if (lane == 0) mbar_arrive(&bar_empty[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      for (int kb = 0; kb < (B1 ? 0 : num_kb); ++kb) {
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
      if (!B1 && lane == 0) mbar_arrive(&bar_empty[prev]);
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

// CTAs of a scan: one per SM (132 without a device)
inline int scan_ctas() {
  const int g = sm_count();
  return g > 0 ? g : 132;
}

SearchPlan plan_search(int k, const void* ws = nullptr) {
  SearchPlan p;
  p.grid = scan_ctas();
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
  constexpr size_t smem = SearchLayout<KLIST, CAP, STAGES, Args>::smem_bytes();
  const int rc = allow_dynamic_smem<search_topk_kernel<KLIST, CAP, STAGES, Args>>(smem);
  if (rc != CRAG_OK) return rc;
  search_topk_kernel<KLIST, CAP, STAGES, Args><<<grid, kSearchThreads, smem, stream>>>(tm_corpus, tm_q, n_rows, num_kb, nq, k, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

// A top-k scan with the selector of k: 64-key lists and 6 stages up to k = 64, 128-key lists and 4 stages above.  The
// one-bit scan's stages are whole tiles and its query block takes 32 KB: 5 and 3 stages.
template <class Args>
int launch_topk_scan(const CUtensorMap& tm_corpus, const CUtensorMap& tm_q, int n_rows, int num_kb, int nq, int k,
                     int grid, const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul, int perm_shift,
                     uint64_t* part_keys, float* part_minmax, const Args& args, cudaStream_t stream) {
  if constexpr (kB1Scan<Args>) {
    if (k <= 64) return launch_scan<64, 64, 5>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
    return launch_scan<128, 128, 3>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
  } else {
    if (k <= 64) return launch_scan<64, 64, 6>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
    return launch_scan<128, 128, 4>(tm_corpus, tm_q, n_rows, num_kb, nq, k, grid, after_keys, pool, perm_mul, perm_shift, part_keys, part_minmax, args, stream);
  }
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

// A scan operand: `rows` rows of `width` elements, `stride` elements apart; `name` heads its error messages.  `bits`
// marks a one-bit shard's sign-bit rows: dim8 / 8 bytes each, read as one zero-filled 128-byte box per row, so their
// width has no rule of its own and follows from the queries' dim8.
enum Elem { kS8 = 1, kBf16 = 2 };   // bytes per element
struct Operand {
  const void* ptr;
  int64_t rows;
  int width;
  int64_t stride;
  Elem elem;
  const char* name;
  bool bits = false;
  Operand rows_from(int64_t r0, int64_t n) const { return {static_cast<const uint8_t*>(ptr) + r0 * stride * elem, n, width, stride, elem, name, bits}; }
  int num_kb() const { return width * elem / 128; }   // 128-byte swizzle rows per row
};

// The scan's rules for an operand, in bytes: 1 to 1024 elements per row in whole 128-byte swizzle rows (bf16 dim % 64,
// int8 dim8 % 128), a row stride of whole 16 bytes, a 16-byte aligned base and row indices that fit an int.
int check_operand(const char* who, const Operand& op) {
  const char* dim = op.elem == kS8 ? "dim8" : "dim";
  if (!op.bits && (op.width < 1 || op.width > 1024 || op.width * op.elem % 128 != 0)) return fail(CRAG_ERR_INVALID, "%s: %s %s must be a multiple of %d in [%d, 1024] (%s=%d)", who, op.name, dim, 128 / op.elem, 128 / op.elem, dim, op.width);
  if (op.rows < 0 || op.rows >= (int64_t(1) << 31) - kTileRows) return fail(CRAG_ERR_INVALID, "%s: %s n_rows out of range (%lld)", who, op.name, (long long)op.rows);
  if (op.stride < op.width || op.stride * op.elem % 16 != 0) return fail(CRAG_ERR_INVALID, "%s: %s row_stride must be >= %s and a multiple of %d", who, op.name, op.bits ? "dim8 / 8 bytes" : dim, 16 / op.elem);
  if (op.rows > 0 && !op.ptr) return fail(CRAG_ERR_INVALID, "%s: null %s pointer", who, op.name);
  if (reinterpret_cast<uintptr_t>(op.ptr) & 15) return fail(CRAG_ERR_INVALID, "%s: %s must be 16-byte aligned", who, op.name);
  return CRAG_OK;
}

// nq and k, the query and shard operands of a scan, and a 256-byte aligned workspace of at least `need` bytes.  The
// queries come first: their width rule is the shard's too, and the only one a one-bit shard has.
int check_scan_args(const char* who, int nq, int k, int k_max, const Operand& corpus, const Operand& queries,
                    const void* workspace, size_t workspace_bytes, size_t need) {
  if (nq < 1 || k < 1 || k > k_max) return fail(CRAG_ERR_INVALID, "%s: need nq >= 1 and 1 <= k <= %d (nq=%d k=%d)", who, k_max, nq, k);
  int rc = check_operand(who, queries);
  if (rc == CRAG_OK) rc = check_operand(who, corpus);
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
  // k-blocks per pass over a row: 128-byte swizzle rows of a query (as many as a corpus row holds, except for one-bit
  // codes, whose whole row is one box)
  return launch_topk_scan(tm_corpus, tm_q, int(corpus.rows), queries.num_kb(), int(queries.rows), k, grid, after_keys, pool,
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

// the exact rescore of crag_ivf_search_i8 and crag_ivf_search_pq: bf16 residuals (device address) and queries, and
// the candidates' workspace buffers
struct IvfRescore {
  Operand rows, queries;
  int64_t* cand_ids;
  float* cand_scores;
};

// Every 32-query pass of an IVF search: the plan of the probed tiles, then `fine(q0, nqc, ids, scores, minmax)`, which
// writes the k results of queries q0 .. q0 + nqc - 1 as stored positions into the outputs it is given, then the map of
// stored positions to original ids.
template <class Fine>
int ivf_pass_loop(int nq, const IvfLists& l, int k, int64_t* out_ids, float* out_scores, float* out_minmax,
                  const IvfPlan& ip, cudaStream_t stream, Fine fine) {
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    ivf_plan_kernel<<<1, 1024, 0, stream>>>(l.probed_ids + size_t(q0) * l.nprobe, l.probed_scores + size_t(q0) * l.nprobe, nqc,
                                            l.nprobe, l.nlist, l.tile_start, l.rows, ip.list_mask, ip.coarse, ip.work,
                                            ip.n_work);
    CRAG_CUDA_OK(cudaGetLastError());
    int64_t* ids = out_ids + size_t(q0) * k;
    const int rc = fine(q0, nqc, ids, out_scores + size_t(q0) * k, out_minmax ? out_minmax + size_t(q0) * 2 : nullptr);
    if (rc != CRAG_OK) return rc;
    ivf_map_ids_kernel<<<(nqc * k + 255) / 256, 256, 0, stream>>>(ids, nqc * k, l.row_ids);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}

// The passes of an IVF search whose stage 1 keeps n_scan keys per query in per-CTA partial lists.
// `stage1(q0, nqc, parts)` launches stage 1 for queries q0 .. q0 + nqc - 1 and sets `parts` to the number of partial
// lists it wrote.  With `rescore` the merge writes n_scan candidates, which the exact rescore (quant.cu) turns into the
// k results, with the plan's coarse terms.
template <class Stage1>
int ivf_passes(int nq, const IvfLists& l, int n_scan, int k, const IvfRescore* rescore, int64_t* out_ids,
               float* out_scores, float* out_minmax, const IvfPlan& ip, cudaStream_t stream, Stage1 stage1) {
  const SearchPlan& sp = ip.scan;
  return ivf_pass_loop(nq, l, k, out_ids, out_scores, out_minmax, ip, stream,
                       [&](int q0, int nqc, int64_t* ids, float* scores, float* minmax) {
    int parts = 0;
    int rc = stage1(q0, nqc, parts);
    if (rc != CRAG_OK) return rc;
    if (!rescore) return finalize_parts(parts, nqc, k, 0, ids, scores, minmax, nullptr, sp, stream);
    rc = finalize_parts(parts, nqc, n_scan, 0, rescore->cand_ids, rescore->cand_scores, minmax, nullptr, sp, stream);
    if (rc == CRAG_OK)
      rc = launch_ivf_rescore(rescore->rows.ptr, rescore->rows.rows, rescore->rows.width, rescore->rows.stride,
                              rescore->queries.rows_from(q0, nqc).ptr, nqc, rescore->cand_ids, n_scan, k, l.tile_start,
                              l.nlist, ip.coarse, ids, scores, stream);
    return rc;
  });
}

// The IVF passes whose stage 1 is the scan of the probed tiles of the residuals `res` (bf16 or int8, as Args says).
// Every CTA of the grid publishes a (possibly empty) partial list, so the merge reads sp.grid parts.
template <class Args>
int ivf_scan_passes(const Operand& res, const Operand& queries, Args args, const IvfLists& l, int n_scan, int k,
                    const IvfRescore* rescore, int64_t* out_ids, float* out_scores, float* out_minmax,
                    const IvfPlan& ip, cudaStream_t stream) {
  const SearchPlan& sp = ip.scan;
  static_cast<IvfArgs&>(args) = IvfArgs{ip.work, ip.n_work, ip.list_mask, ip.coarse};
  CUtensorMap tm_res;
  int rc = make_tmap(&tm_res, res, kTileRows);
  if (rc != CRAG_OK) return rc;
  return ivf_passes(int(queries.rows), l, n_scan, k, rescore, out_ids, out_scores, out_minmax, ip, stream,
                    [&](int q0, int nqc, int& parts) {
                      CUtensorMap tm_q;
                      const int rc = make_tmap(&tm_q, queries.rows_from(q0, nqc), kNQ);
                      if (rc != CRAG_OK) return rc;
                      if (sp.pool) CRAG_CUDA_OK(cudaMemsetAsync(sp.pool, 0, sp.pool_bytes, stream));
                      parts = sp.grid;
                      return launch_topk_scan(tm_res, tm_q, int(res.rows), res.num_kb(), nqc, n_scan, sp.grid, nullptr,
                                              sp.pool, 0u, 0, sp.part_keys, sp.part_minmax, pass_args(args, q0), stream);
                    });
}

// The argument rules of the rescored IVF searches (crag_ivf_search_i8 / _pq and their _wide forms): the lists, probes
// and outputs, nq >= 1 and 1 <= k <= n_cand <= max_cand (128, or 2048 for the wide forms), then the entry's own rules
// (`entry_check()`), the bf16 residuals and queries of the rescore, and a workspace of `need` bytes.  Then points
// r.rows at the device address of the bf16 residuals, which may be page-locked host memory (pageable memory is refused
// before any launch), and r's candidates at the workspace's buffers `cand_ids` / `cand_scores`.
template <class EntryCheck>
int check_rescored_ivf(const char* who, const IvfLists& l, int64_t n_rows_padded, int nq, int n_cand, int k, int max_cand,
                       const int64_t* out_ids, const float* out_scores, IvfRescore& r, int64_t* cand_ids,
                       float* cand_scores, const void* workspace, size_t workspace_bytes, size_t need,
                       EntryCheck entry_check) {
  int rc = check_ivf_args(who, l, n_rows_padded, out_ids, out_scores);
  if (rc != CRAG_OK) return rc;
  if (nq < 1 || k < 1 || n_cand < k || n_cand > max_cand) return fail(CRAG_ERR_INVALID, "%s: need nq >= 1 and 1 <= k <= n_cand <= %d (nq=%d k=%d n_cand=%d)", who, max_cand, nq, k, n_cand);
  rc = entry_check();
  if (rc == CRAG_OK) rc = check_operand(who, r.rows);
  if (rc == CRAG_OK) rc = check_operand(who, r.queries);
  if (rc == CRAG_OK) rc = check_workspace(who, workspace, workspace_bytes, need);
  if (rc == CRAG_OK) rc = device_readable(r.rows.ptr, &r.rows.ptr, who);
  r.cand_ids = cand_ids;
  r.cand_scores = cand_scores;
  return rc;
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
  return ivf_scan_passes(res, q, IvfArgs{}, lists, k, k, nullptr, out_ids, out_scores, out_minmax, ip,
                         static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ IVF over int8 residuals (ivf_passes with a rescore)
namespace crag {
namespace {
// the int8 residuals and queries of an int8 IVF search: dim8 = dim rounded up to 128, the scan's operand rules, scales
int check_ivf_i8_codes(const char* who, int dim, const Operand& res, const Operand& q, const float* row_scales,
                       const float* query_scales) {
  if (res.width != (dim + 127) / 128 * 128) return fail(CRAG_ERR_INVALID, "%s: dim8 must be dim rounded up to a multiple of 128 (dim=%d dim8=%d)", who, dim, res.width);
  int rc = check_operand(who, res);
  if (rc == CRAG_OK) rc = check_operand(who, q);
  if (rc == CRAG_OK && (!row_scales || !query_scales)) rc = fail(CRAG_ERR_INVALID, "%s: null pointer", who);
  return rc;
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
                                  size_t workspace_bytes, crag_stream_t stream) {
  const Operand res{residuals_i8, n_rows_padded, dim8, row_stride_i8, kS8, "residuals_i8"}, q{queries_i8, nq, dim8, dim8, kS8, "queries_i8"};
  IvfRescore rescore{{residuals_bf16, n_rows_padded, dim, row_stride, kBf16, "residuals_bf16"},
                     {queries_bf16, nq, dim, dim, kBf16, "queries_bf16"}, nullptr, nullptr};
  const IvfLists lists{list_tile_start, list_rows, nlist, total_tiles, row_ids, probed_ids, probed_scores, nprobe};
  const IvfI8Plan plan = plan_ivf_i8(nlist, total_tiles, n_cand, workspace);
  const int rc = check_rescored_ivf("ivf_i8", lists, n_rows_padded, nq, n_cand, k, 128, out_ids, out_scores, rescore,
                                    plan.cand_ids, plan.cand_scores, workspace, workspace_bytes, plan.total,
                                    [&] { return check_ivf_i8_codes("ivf_i8", dim, res, q, row_scales, query_scales); });
  if (rc != CRAG_OK) return rc;
  return ivf_scan_passes(res, q, I8IvfArgs{{}, {row_scales, query_scales}}, lists, n_cand, k, &rescore, out_ids, out_scores,
                         out_minmax, plan.ivf, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ IVF over product-quantized residuals (pq_kernels.cuh)
namespace crag {
namespace {

// PQ IVF workspace = the int8 IVF workspace for n_cand candidates, then the tables of one pass's queries
struct IvfPqPlan {
  IvfI8Plan cand;
  float* lut;   // [kNQ][m][256]
  size_t total;
};
IvfPqPlan plan_ivf_pq(int nlist, int64_t total_tiles, int n_cand, int m, const void* ws = nullptr) {
  IvfPqPlan p;
  p.cand = plan_ivf_i8(nlist, total_tiles, n_cand, ws);
  WsCursor c(ws, p.cand.total);
  p.lut = c.take<float>(size_t(kNQ) * m * kPqCodewords);
  p.total = c.bytes;
  return p;
}

int check_pq_shape(const char* who, int dim, int m) {
  if (dim < 64 || dim > 1024 || dim % 64 != 0) return fail(CRAG_ERR_INVALID, "%s: dim must be a multiple of 64 in [64, 1024] (dim=%d)", who, dim);
  if (m < 1 || m > kPqMaxM || dim % m != 0 || dim / m > kPqMaxDsub) return fail(CRAG_ERR_INVALID, "%s: m must divide dim with 1 <= m <= %d and dim / m <= %d (dim=%d m=%d)", who, kPqMaxM, kPqMaxDsub, dim, m);
  return CRAG_OK;
}

// the codes and codebooks of a PQ IVF search
int check_ivf_pq_codes(const char* who, int dim, int m, const void* codes, int64_t code_stride, const float* codebooks) {
  const int rc = check_pq_shape(who, dim, m);
  if (rc != CRAG_OK) return rc;
  if (code_stride < pq_code_stride(m) || code_stride % 16 != 0) return fail(CRAG_ERR_INVALID, "%s: code_stride must be a multiple of 16 and >= %d (code_stride=%lld)", who, pq_code_stride(m), (long long)code_stride);
  if (!codes || !codebooks) return fail(CRAG_ERR_INVALID, "%s: null codes or codebooks pointer", who);
  if ((reinterpret_cast<uintptr_t>(codes) | reinterpret_cast<uintptr_t>(codebooks)) & 15) return fail(CRAG_ERR_INVALID, "%s: codes and codebooks must be 16-byte aligned", who);
  return CRAG_OK;
}

}  // namespace
}  // namespace crag

extern "C" size_t crag_ivf_pq_workspace_bytes(int nlist, int64_t total_tiles, int n_cand, int m) {
  if (nlist < 1 || total_tiles < 0 || n_cand < 1 || n_cand > 128 || m < 1 || m > kPqMaxM) return 0;
  return plan_ivf_pq(nlist, total_tiles, n_cand, m).total;
}

extern "C" int crag_ivf_search_pq(const void* codes, int m, int64_t code_stride, const float* codebooks,
                                  const void* residuals_bf16, int dim, int64_t row_stride, int64_t n_rows_padded,
                                  const int32_t* list_tile_start, const int32_t* list_rows, int nlist,
                                  int64_t total_tiles, const int64_t* row_ids, const void* queries_bf16, int nq,
                                  const int64_t* probed_ids, const float* probed_scores, int nprobe, int n_cand, int k,
                                  int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                                  size_t workspace_bytes, crag_stream_t stream) {
  IvfRescore rescore{{residuals_bf16, n_rows_padded, dim, row_stride, kBf16, "residuals_bf16"},
                     {queries_bf16, nq, dim, dim, kBf16, "queries_bf16"}, nullptr, nullptr};
  const IvfLists lists{list_tile_start, list_rows, nlist, total_tiles, row_ids, probed_ids, probed_scores, nprobe};
  const IvfPqPlan plan = plan_ivf_pq(nlist, total_tiles, n_cand, m, workspace);
  const int rc = check_rescored_ivf("ivf_pq", lists, n_rows_padded, nq, n_cand, k, 128, out_ids, out_scores, rescore,
                                    plan.cand.cand_ids, plan.cand.cand_scores, workspace, workspace_bytes, plan.total,
                                    [&] { return check_ivf_pq_codes("ivf_pq", dim, m, codes, code_stride, codebooks); });
  if (rc != CRAG_OK) return rc;
  // Stage 1: the queries' tables, then the PQ scan for n_cand candidates, about two CTAs per SM in all; every
  // (slice, query) CTA writes its part, so the merge reads `slices` parts.
  const IvfPlan& ip = plan.cand.ivf;
  const SearchPlan& sp = ip.scan;
  const IvfArgs args{ip.work, ip.n_work, ip.list_mask, ip.coarse};
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return ivf_passes(nq, lists, n_cand, k, &rescore, out_ids, out_scores, out_minmax, ip, st, [&](int q0, int nqc, int& slices) {
    const void* qp = rescore.queries.rows_from(q0, nqc).ptr;
    pq_table_kernel<<<unsigned(nqc * m), kPqTableThreads, 0, st>>>(static_cast<const uint16_t*>(qp), dim, codebooks, m, plan.lut);
    CRAG_CUDA_OK(cudaGetLastError());
    slices = std::min(sp.grid, std::max(1, (2 * sp.grid + nqc - 1) / nqc));
    int rc = CRAG_OK;
    with_merge_tier(n_cand, [&](auto tier) {
      constexpr int T = decltype(tier)::value;
      rc = allow_dynamic_smem<pq_scan_kernel<T>>(PqScanSmem<T>::bytes(kPqMaxM));
      if (rc != CRAG_OK) return;
      pq_scan_kernel<T><<<unsigned(nqc * slices), kPqThreads, PqScanSmem<T>::bytes(m), st>>>(
          static_cast<const uint8_t*>(codes), code_stride, m, plan.lut, slices, n_cand, args, sp.part_keys, sp.part_minmax);
    });
    if (rc != CRAG_OK) return rc;
    CRAG_CUDA_OK(cudaGetLastError());
    return CRAG_OK;
  });
}

// ------------------------------------------------------------------ wide IVF stage 1: up to 2048 candidates per query
// Per 32-query pass: the IVF plan, the wide plan (slot layout, ivf_kernels.cuh), a score-all fill of every probed row's
// S1 into the S1 block (ivf_wide_kernels.cuh), the ragged per-query select (knn_select.cuh), the map of slots to stored
// positions, then the IVF rescore and the id map.  DESIGN.md section 7.
namespace crag {
namespace {

constexpr int kIvfWideMaxCand = kKnnMaxK;
constexpr int64_t kIvfMaxProbeRows = (int64_t(1) << 31) - kTileRows;

// Workspace of the wide searches: the IVF plan (sized for a 1-key scan, which the wide path never launches: only its
// list mask, coarse terms and work-list are used), the wide plan, the S1 block [kNQ][round_up(max_probe_rows, 4)],
// the candidates of one pass, then (PQ, m > 0) the tables of one pass's queries.
struct IvfWideWs {
  IvfPlan ivf;
  IvfWidePlan wide;
  float* block;
  int64_t ld;
  int64_t* cand_ids;
  float* cand_scores;
  float* lut;
  size_t total;
};
IvfWideWs plan_ivf_wide(int nlist, int64_t total_tiles, int n_cand, int64_t max_probe_rows, int m, const void* ws = nullptr) {
  IvfWideWs p;
  p.ivf = plan_ivf(1, nlist, total_tiles, ws);
  WsCursor c(ws, p.ivf.total);
  p.wide.slot_base = c.take<int32_t>(size_t(nlist) * kNQ);
  p.wide.seg_list = c.take<int32_t>(size_t(kNQ) * kIvfMaxProbe);
  p.wide.seg_slot = c.take<int32_t>(size_t(kNQ) * kIvfMaxProbe);
  p.wide.n_seg = c.take<int32_t>(kNQ);
  p.wide.n_rows = c.take<int32_t>(kNQ);
  p.ld = (max_probe_rows + 3) & ~int64_t(3);
  p.block = c.take<float>(size_t(kNQ) * size_t(p.ld));
  p.cand_ids = c.take<int64_t>(size_t(kNQ) * n_cand);
  p.cand_scores = c.take<float>(size_t(kNQ) * n_cand);
  p.lut = c.take<float>(size_t(kNQ) * m * kPqCodewords);
  p.total = c.bytes;
  return p;
}

bool wide_sizes_ok(int nlist, int64_t total_tiles, int n_cand, int64_t max_probe_rows) {
  return nlist >= 1 && total_tiles >= 0 && n_cand >= 1 && n_cand <= kIvfWideMaxCand && max_probe_rows >= 1 &&
         max_probe_rows <= kIvfMaxProbeRows;
}

// The workspace layout of a wide search's arguments.  Sizes out of range are refused by the argument checks before the
// layout is used, so they carve a minimal one.
IvfWideWs plan_ivf_wide_args(int nlist, int64_t total_tiles, int n_cand, int64_t max_probe_rows, int m, const void* ws) {
  if (!wide_sizes_ok(nlist, total_tiles, n_cand, max_probe_rows)) return plan_ivf_wide(1, 0, 1, 1, 0, ws);
  return plan_ivf_wide(nlist, total_tiles, n_cand, max_probe_rows, m >= 1 && m <= kPqMaxM ? m : 0, ws);
}

// the wide forms' own rules beside their entry's: max_probe_rows, and nprobe within the wide plan's probe table
int check_wide_rows(const char* who, int nprobe, int64_t max_probe_rows) {
  if (max_probe_rows < 1 || max_probe_rows > kIvfMaxProbeRows) return fail(CRAG_ERR_INVALID, "%s: need 1 <= max_probe_rows <= %lld (max_probe_rows=%lld)", who, (long long)kIvfMaxProbeRows, (long long)max_probe_rows);
  if (nprobe > kIvfMaxProbe) return fail(CRAG_ERR_INVALID, "%s: need nprobe <= %d (nprobe=%d)", who, kIvfMaxProbe, nprobe);
  return CRAG_OK;
}

// The passes of a wide search.  `fill(q0, nqc, slices, args, out)` launches the score-all fill of the pass's S1 block
// over nqc * slices CTAs, about ctas_per_sm per SM: 2 for the PQ fill, as the PQ scan, and 8 for the int8 fill, whose
// one-warp-per-row CTAs need more warps per SM to keep enough row reads in flight.
template <class Fill>
int ivf_wide_passes(int nq, const IvfLists& l, int n_cand, int k, int cap, const IvfRescore& rescore, int64_t* out_ids,
                    float* out_scores, float* out_minmax, const IvfWideWs& w, cudaStream_t stream, int ctas_per_sm,
                    Fill fill) {
  const IvfPlan& ip = w.ivf;
  const IvfArgs args{ip.work, ip.n_work, ip.list_mask, ip.coarse};
  const IvfWideBlock out{l.tile_start, w.wide.slot_base, w.block, w.ld, cap};
  const int grid = ip.scan.grid;
  return ivf_pass_loop(nq, l, k, out_ids, out_scores, out_minmax, ip, stream,
                       [&](int q0, int nqc, int64_t* ids, float* scores, float* minmax) {
    ivf_wide_plan_kernel<<<nqc, kIvfMaxProbe, 0, stream>>>(l.probed_ids + size_t(q0) * l.nprobe, l.nprobe, l.nlist, l.rows,
                                                           cap, w.wide);
    CRAG_CUDA_OK(cudaGetLastError());
    // about ctas_per_sm CTAs per SM in all, at most half of them for one query
    const int slices = std::min(ctas_per_sm * grid / 2, std::max(1, (ctas_per_sm * grid + nqc - 1) / nqc));
    int rc = fill(q0, nqc, slices, args, out);
    if (rc != CRAG_OK) return rc;
    CRAG_CUDA_OK(cudaGetLastError());
    ivf_wide_select_kernel<<<nqc, kKnnThreads, 0, stream>>>(w.block, w.ld, w.wide.n_rows, n_cand, w.cand_ids,
                                                            w.cand_scores, minmax);
    CRAG_CUDA_OK(cudaGetLastError());
    ivf_slot_map_kernel<<<(nqc * n_cand + 255) / 256, 256, 0, stream>>>(w.cand_ids, nqc, n_cand, w.wide, l.tile_start);
    CRAG_CUDA_OK(cudaGetLastError());
    return launch_ivf_rescore(rescore.rows.ptr, rescore.rows.rows, rescore.rows.width, rescore.rows.stride,
                              rescore.queries.rows_from(q0, nqc).ptr, nqc, w.cand_ids, n_cand, k, l.tile_start, l.nlist,
                              ip.coarse, ids, scores, stream);
  });
}

}  // namespace
}  // namespace crag

extern "C" size_t crag_ivf_i8_wide_workspace_bytes(int nlist, int64_t total_tiles, int n_cand, int64_t max_probe_rows) {
  if (!wide_sizes_ok(nlist, total_tiles, n_cand, max_probe_rows)) return 0;
  return plan_ivf_wide(nlist, total_tiles, n_cand, max_probe_rows, 0).total;
}

extern "C" size_t crag_ivf_pq_wide_workspace_bytes(int nlist, int64_t total_tiles, int n_cand, int64_t max_probe_rows,
                                                   int m) {
  if (!wide_sizes_ok(nlist, total_tiles, n_cand, max_probe_rows) || m < 1 || m > kPqMaxM) return 0;
  return plan_ivf_wide(nlist, total_tiles, n_cand, max_probe_rows, m).total;
}

extern "C" int crag_ivf_search_i8_wide(const void* residuals_i8, const float* row_scales, int dim8, int64_t row_stride_i8,
                                       const void* residuals_bf16, int dim, int64_t row_stride, int64_t n_rows_padded,
                                       const int32_t* list_tile_start, const int32_t* list_rows, int nlist,
                                       int64_t total_tiles, const int64_t* row_ids, const void* queries_i8,
                                       const float* query_scales, const void* queries_bf16, int nq,
                                       const int64_t* probed_ids, const float* probed_scores, int nprobe, int n_cand,
                                       int k, int64_t max_probe_rows, int64_t* out_ids, float* out_scores,
                                       float* out_minmax, void* workspace, size_t workspace_bytes, crag_stream_t stream) {
  const char* who = "ivf_i8_wide";
  const Operand res{residuals_i8, n_rows_padded, dim8, row_stride_i8, kS8, "residuals_i8"}, q{queries_i8, nq, dim8, dim8, kS8, "queries_i8"};
  IvfRescore rescore{{residuals_bf16, n_rows_padded, dim, row_stride, kBf16, "residuals_bf16"},
                     {queries_bf16, nq, dim, dim, kBf16, "queries_bf16"}, nullptr, nullptr};
  const IvfLists lists{list_tile_start, list_rows, nlist, total_tiles, row_ids, probed_ids, probed_scores, nprobe};
  const IvfWideWs plan = plan_ivf_wide_args(nlist, total_tiles, n_cand, max_probe_rows, 0, workspace);
  const int rc = check_rescored_ivf(who, lists, n_rows_padded, nq, n_cand, k, kIvfWideMaxCand, out_ids, out_scores, rescore,
                                    plan.cand_ids, plan.cand_scores, workspace, workspace_bytes, plan.total, [&] {
    const int rc = check_wide_rows(who, nprobe, max_probe_rows);
    return rc != CRAG_OK ? rc : check_ivf_i8_codes(who, dim, res, q, row_scales, query_scales);
  });
  if (rc != CRAG_OK) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return ivf_wide_passes(nq, lists, n_cand, k, int(max_probe_rows), rescore, out_ids, out_scores, out_minmax, plan, st, 8,
                         [&](int q0, int nqc, int slices, const IvfArgs& args, const IvfWideBlock& out) {
    ivf_fill_i8_kernel<<<unsigned(nqc * slices), kIvfFillThreads, 0, st>>>(
        static_cast<const int8_t*>(residuals_i8), row_stride_i8, dim8, row_scales,
        static_cast<const int8_t*>(queries_i8) + size_t(q0) * dim8, query_scales + q0, slices, args, out);
    return CRAG_OK;
  });
}

extern "C" int crag_ivf_search_pq_wide(const void* codes, int m, int64_t code_stride, const float* codebooks,
                                       const void* residuals_bf16, int dim, int64_t row_stride, int64_t n_rows_padded,
                                       const int32_t* list_tile_start, const int32_t* list_rows, int nlist,
                                       int64_t total_tiles, const int64_t* row_ids, const void* queries_bf16, int nq,
                                       const int64_t* probed_ids, const float* probed_scores, int nprobe, int n_cand,
                                       int k, int64_t max_probe_rows, int64_t* out_ids, float* out_scores,
                                       float* out_minmax, void* workspace, size_t workspace_bytes, crag_stream_t stream) {
  const char* who = "ivf_pq_wide";
  IvfRescore rescore{{residuals_bf16, n_rows_padded, dim, row_stride, kBf16, "residuals_bf16"},
                     {queries_bf16, nq, dim, dim, kBf16, "queries_bf16"}, nullptr, nullptr};
  const IvfLists lists{list_tile_start, list_rows, nlist, total_tiles, row_ids, probed_ids, probed_scores, nprobe};
  const IvfWideWs plan = plan_ivf_wide_args(nlist, total_tiles, n_cand, max_probe_rows, m, workspace);
  const int rc = check_rescored_ivf(who, lists, n_rows_padded, nq, n_cand, k, kIvfWideMaxCand, out_ids, out_scores, rescore,
                                    plan.cand_ids, plan.cand_scores, workspace, workspace_bytes, plan.total, [&] {
    const int rc = check_wide_rows(who, nprobe, max_probe_rows);
    return rc != CRAG_OK ? rc : check_ivf_pq_codes(who, dim, m, codes, code_stride, codebooks);
  });
  if (rc != CRAG_OK) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return ivf_wide_passes(nq, lists, n_cand, k, int(max_probe_rows), rescore, out_ids, out_scores, out_minmax, plan, st, 2,
                         [&](int q0, int nqc, int slices, const IvfArgs& args, const IvfWideBlock& out) {
    const void* qp = rescore.queries.rows_from(q0, nqc).ptr;
    pq_table_kernel<<<unsigned(nqc * m), kPqTableThreads, 0, st>>>(static_cast<const uint16_t*>(qp), dim, codebooks, m, plan.lut);
    CRAG_CUDA_OK(cudaGetLastError());
    const int rc = allow_dynamic_smem<ivf_fill_pq_kernel>(size_t(kPqMaxM) * kPqCodewords * 4);
    if (rc != CRAG_OK) return rc;
    ivf_fill_pq_kernel<<<unsigned(nqc * slices), kIvfFillThreads, size_t(m) * kPqCodewords * 4, st>>>(
        static_cast<const uint8_t*>(codes), code_stride, m, plan.lut, slices, args, out);
    return CRAG_OK;
  });
}

extern "C" int crag_pq_encode(const void* rows_bf16, int64_t n_rows, int dim, int64_t row_stride, const float* codebooks,
                              int m, void* codes, int64_t code_stride, crag_stream_t stream) {
  int rc = check_pq_shape("pq_encode", dim, m);
  if (rc != CRAG_OK) return rc;
  if (n_rows < 0 || n_rows >= (int64_t(1) << 31)) return fail(CRAG_ERR_INVALID, "pq_encode: n_rows out of range (%lld)", (long long)n_rows);
  if (row_stride < dim) return fail(CRAG_ERR_INVALID, "pq_encode: row_stride must be >= dim (row_stride=%lld dim=%d)", (long long)row_stride, dim);
  if (code_stride < m) return fail(CRAG_ERR_INVALID, "pq_encode: code_stride must be >= m (code_stride=%lld m=%d)", (long long)code_stride, m);
  if (n_rows == 0) return CRAG_OK;
  if (!rows_bf16 || !codebooks || !codes) return fail(CRAG_ERR_INVALID, "pq_encode: null rows, codebooks or codes pointer");
  if ((reinterpret_cast<uintptr_t>(rows_bf16) & 1) || (reinterpret_cast<uintptr_t>(codebooks) & 3)) return fail(CRAG_ERR_INVALID, "pq_encode: rows must be 2-byte and codebooks 4-byte aligned");
  const void* rows = rows_bf16;
  rc = device_readable(rows_bf16, &rows, "pq_encode");
  if (rc != CRAG_OK) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = allow_dynamic_smem<pq_encode_kernel>(pq_encode_smem_bytes(kPqMaxDsub));
  if (rc != CRAG_OK) return rc;
  constexpr int64_t kChunk = int64_t(1) << 22;   // rows per launch: (chunk / 128) * m blocks stay far below 2^31
  for (int64_t r0 = 0; r0 < n_rows; r0 += kChunk) {
    const int64_t n = std::min(kChunk, n_rows - r0);
    const unsigned grid = unsigned((n + kPqThreads - 1) / kPqThreads) * unsigned(m);
    pq_encode_kernel<<<grid, kPqThreads, pq_encode_smem_bytes(dim / m), st>>>(
        static_cast<const uint16_t*>(rows) + r0 * row_stride, n, dim, row_stride, codebooks, m,
        static_cast<uint8_t*>(codes) + r0 * code_stride, code_stride);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
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

// ------------------------------------------------------------------ one-bit shards (binary.cuh, quant_kernels.cuh)
extern "C" int crag_search_topk_b1(const void* bits, const float* alpha, int64_t n_rows, int dim8, int64_t row_stride,
                                   int64_t row_offset, const void* queries_i8, const float* query_scales, int nq, int k,
                                   int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                                   size_t workspace_bytes, crag_stream_t stream) {
  const Operand c{bits, n_rows, dim8 / 8, row_stride, kS8, "bits", true}, q{queries_i8, nq, dim8, dim8, kS8, "queries_i8"};
  const SearchPlan plan = plan_search(k >= 1 && k <= 128 ? k : 1, workspace);
  int rc = check_scan_args("search_b1", nq, k, 128, c, q, workspace, workspace_bytes, plan.parts_bytes);
  if (rc != CRAG_OK) return rc;
  if ((n_rows > 0 && !alpha) || !query_scales || !out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "search_b1: null alpha, query_scales or output pointer");
  return topk_passes(c, q, k, row_offset, nullptr, B1Args{{alpha, query_scales}}, out_ids, out_scores, out_minmax,
                     nullptr, workspace_bytes, plan, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ exact top-k for large k / many queries
// Per chunk of queries the score block (score_block_chunks), then knn_select_kernel (knn_select.cuh) radix-selects each
// query's k best rows from its row.
namespace crag {
namespace {
inline int64_t knn_ld(int64_t n_rows) { return ((n_rows > 0 ? n_rows : 1) + 3) & ~int64_t(3); }

// Workspace of crag_knn_topk: the fp32 score block [q_chunk][knn_ld(n_rows)], from byte `at` on (0 for crag_knn_topk,
// the score-all pass's partials before it for crag_knn_topk_i8 / _b1: knn_code_workspace)
struct KnnWorkspace { float* block; size_t total; };
KnnWorkspace knn_workspace(int64_t n_rows, int q_chunk, void* ws = nullptr, size_t at = 0) {
  WsCursor c(ws, at);
  KnnWorkspace w;
  w.block = c.take<float>(size_t(q_chunk) * size_t(knn_ld(n_rows)));
  w.total = c.bytes;
  return w;
}

// Per chunk of queries, as many as the workspace holds score rows for after its first `at` bytes: `fill(q0, nqc, block,
// ld)` writes the chunk's fp32 score block [nqc, ld] into the workspace and returns a status, then `select(q0, nqc,
// block, ld)` launches its per-query select.
template <class Fill, class Select>
int score_block_chunks(const char* who, int64_t n_rows, int nq, void* workspace, size_t workspace_bytes, size_t at,
                       cudaStream_t stream, Fill fill, Select select) {
  const int64_t ld = knn_ld(n_rows);
  const size_t per_query = size_t(ld) * 4;
  const size_t fit = workspace_bytes > at ? (workspace_bytes - at) / per_query : 0;
  if (fit < 1) return fail(CRAG_ERR_WORKSPACE, "%s: workspace %zu < %zu bytes (one query's score row)", who, workspace_bytes, at + per_query);
  const int q_chunk = fit < size_t(nq) ? int(fit) : nq;
  float* block = knn_workspace(n_rows, q_chunk, workspace, at).block;
  for (int q0 = 0; q0 < nq; q0 += q_chunk) {
    const int nqc = (nq - q0) < q_chunk ? (nq - q0) : q_chunk;
    const int rc = fill(q0, nqc, block, ld);
    if (rc != CRAG_OK) return rc;
    select(q0, nqc, block, ld);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}

// The score block of crag_knn_topk and crag_knn_threshold: the wgmma GEMM of a chunk of bf16 queries (gemm_scores_f32)
auto gemm_fill(const Operand& corpus, const void* queries, cudaStream_t stream) {
  return [=](int q0, int nqc, float* block, int64_t ld) {
    const int dim = corpus.width;
    return gemm_scores_f32(static_cast<const uint8_t*>(queries) + size_t(q0) * dim * 2, dim, corpus.ptr, corpus.stride,
                           block, ld, nqc, int(corpus.rows), dim, stream);
  };
}

// The select of crag_knn_topk and crag_knn_topk_i8 / _b1: knn_select_kernel, one CTA per query of the chunk
auto knn_select(int64_t n_rows, int k, int64_t row_offset, int64_t* out_ids, float* out_scores, float* out_minmax,
                cudaStream_t stream) {
  return [=](int q0, int nqc, const float* block, int64_t ld) {
    knn_select_kernel<<<nqc, kKnnThreads, 0, stream>>>(block, ld, int(n_rows), k, row_offset, out_ids + size_t(q0) * k,
                                                       out_scores + size_t(q0) * k,
                                                       out_minmax ? out_minmax + size_t(q0) * 2 : nullptr);
  };
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
  return score_block_chunks("knn", n_rows, nq, workspace, workspace_bytes, 0, stream, gemm_fill(c, queries, stream),
                            knn_select(n_rows, k, row_offset, out_ids, out_scores, out_minmax, stream));
}

// Threshold join: per chunk of queries the same score block as crag_knn_topk, then knn_threshold_kernel
// (knn_threshold.cuh) keeps each query's rows scoring >= threshold among its first `limit`, skipping self_rows[q] and
// exclude_rows, at most `cap` of them.
extern "C" int crag_knn_threshold(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                  const void* queries, int nq, float threshold, int limit, int cap,
                                  const int64_t* self_rows, const int64_t* exclude_rows, int n_exclude,
                                  int* out_counts, int64_t* out_ids, float* out_scores, void* workspace,
                                  size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const Operand c{corpus, n_rows, dim, corpus_row_stride, kBf16, "corpus"}, q{queries, nq, dim, dim, kBf16, "queries"};
  int rc = check_scan_args("knn_threshold", nq, limit, 0x7FFFFFFF, c, q, workspace, workspace_bytes, 0);
  if (rc != CRAG_OK) return rc;
  if (!isfinite(threshold)) return fail(CRAG_ERR_INVALID, "knn_threshold: threshold must be finite");
  if (cap < 1 || n_exclude < 0 || n_exclude > kKnnMaxExclude || cap + n_exclude + 1 > kKnnMaxK)
    return fail(CRAG_ERR_INVALID, "knn_threshold: need cap >= 1, 0 <= n_exclude <= %d and cap + n_exclude + 1 <= %d (cap=%d n_exclude=%d)",
                kKnnMaxExclude, kKnnMaxK, cap, n_exclude);
  if (!out_counts || !out_ids || !out_scores || (n_exclude > 0 && !exclude_rows)) return fail(CRAG_ERR_INVALID, "knn_threshold: null pointer");
  return score_block_chunks("knn_threshold", n_rows, nq, workspace, workspace_bytes, 0, stream, gemm_fill(c, queries, stream),
                            [&](int q0, int nqc, const float* block, int64_t ld) {
    knn_threshold_kernel<<<nqc, kKnnThreads, 0, stream>>>(block, ld, int(n_rows), threshold, limit, cap,
                                                          self_rows ? self_rows + q0 : nullptr, exclude_rows, n_exclude,
                                                          out_counts + q0, out_ids + size_t(q0) * cap,
                                                          out_scores + size_t(q0) * cap);
  });
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

// Score-all passes (the scan with ScoreArgs, or CodeScoreArgs over int8 or one-bit rows), one per block of 32 queries.
// Block q0 stores its scores from row q0 of sa.out on, or, in assignment mode (sa.best_id set), updates every row's
// running argmax with ids counted from q0.  out_minmax (may be null) receives each query's (min, max).  Only
// plan.part_minmax is used.
template <class Args>
int score_passes(const Operand& corpus, const Operand& queries, const Args& sa, float* out_minmax,
                 const SearchPlan& plan, cudaStream_t stream) {
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
    Args pass = pass_args(sa, q0);
    if (sa.best_id) pass.base_id = q0;
    else pass.out = sa.out + int64_t(q0) * sa.ld;
    // k-blocks per row: the queries' 128-byte swizzle rows (a one-bit code row is one box, see scan_pass)
    rc = launch_scan<16, 16, 7>(tm_corpus, tm_q, int(corpus.rows), queries.num_kb(), nqc, 1, grid, nullptr, nullptr, 0u, 0, nullptr, plan.part_minmax, pass, stream);
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

// ------------------------------------------------------------------ exact top-k up to 2048 over int8 and one-bit codes
namespace crag {
namespace {
// Workspace of crag_knn_topk_i8 / _b1: the score-all pass's per-CTA (min, max) (all of a SearchPlan that score_passes
// reads), then the score block (knn_workspace from the end of these partials on)
SearchPlan plan_score_parts(const void* ws = nullptr) {
  SearchPlan p{};
  p.grid = scan_ctas();
  WsCursor c(ws);
  p.part_minmax = c.take<float>(size_t(p.grid) * kNQ * 2);
  p.parts_bytes = p.total = c.bytes;
  return p;
}

// Per chunk of queries the score-all passes over the codes write the chunk's S1 block, then crag_knn_topk's select
// keeps each query's k best rows.
template <class Codes>
int knn_code_topk(const char* who, const Operand& corpus, const Operand& queries, const Codes& codes, int64_t row_offset,
                  int k, int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace, size_t workspace_bytes,
                  cudaStream_t stream) {
  const SearchPlan parts = plan_score_parts(workspace);
  return score_block_chunks(who, corpus.rows, int(queries.rows), workspace, workspace_bytes, parts.total, stream,
                            [&](int q0, int nqc, float* block, int64_t ld) {
                              const CodeScoreArgs<Codes> sa(block, ld, codes);
                              return score_passes(corpus, queries.rows_from(q0, nqc), pass_args(sa, q0), nullptr, parts, stream);
                            },
                            knn_select(corpus.rows, k, row_offset, out_ids, out_scores, out_minmax, stream));
}
}  // namespace
}  // namespace crag

extern "C" size_t crag_knn_code_workspace_bytes(int64_t n_rows, int q_chunk) {
  if (n_rows < 0 || q_chunk < 1) return 0;
  return knn_workspace(n_rows, q_chunk, nullptr, plan_score_parts().total).total;
}

extern "C" int crag_knn_topk_i8(const void* codes, const float* row_scales, int64_t n_rows, int dim8, int64_t row_stride,
                                int64_t row_offset, const void* queries_i8, const float* query_scales, int nq, int k,
                                int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                                size_t workspace_bytes, crag_stream_t stream) {
  const Operand c{codes, n_rows, dim8, row_stride, kS8, "corpus"}, q{queries_i8, nq, dim8, dim8, kS8, "queries"};
  int rc = check_scan_args("search_i8", nq, k, kKnnMaxK, c, q, workspace, workspace_bytes, plan_score_parts().total);
  if (rc != CRAG_OK) return rc;
  if (!query_scales || !out_ids || !out_scores || (n_rows > 0 && !row_scales)) return fail(CRAG_ERR_INVALID, "search_i8: null pointer");
  return knn_code_topk("knn_i8", c, q, I8Args{row_scales, query_scales}, row_offset, k, out_ids, out_scores, out_minmax,
                       workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int crag_knn_topk_b1(const void* bits, const float* alpha, int64_t n_rows, int dim8, int64_t row_stride,
                                int64_t row_offset, const void* queries_i8, const float* query_scales, int nq, int k,
                                int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                                size_t workspace_bytes, crag_stream_t stream) {
  const Operand c{bits, n_rows, dim8 / 8, row_stride, kS8, "bits", true}, q{queries_i8, nq, dim8, dim8, kS8, "queries_i8"};
  int rc = check_scan_args("search_b1", nq, k, kKnnMaxK, c, q, workspace, workspace_bytes, plan_score_parts().total);
  if (rc != CRAG_OK) return rc;
  if ((n_rows > 0 && !alpha) || !query_scales || !out_ids || !out_scores) return fail(CRAG_ERR_INVALID, "search_b1: null alpha, query_scales or output pointer");
  return knn_code_topk("knn_b1", c, q, B1Args{{alpha, query_scales}}, row_offset, k, out_ids, out_scores, out_minmax,
                       workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
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
