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
// keeps each row's running argmax over centroid blocks (crag_ivf_assign).
// Around it in this file: the per-shard merge (merge_topk_kernel), the fused
// finalize + NVLink exchange + global merge of the row-sharded index
// (finalize_exchange_kernel), the C-ABI entry points, and crag_knn_topk -- exact
// top-k up to k = 2048 for large query batches as a score-block GEMM (gemm.cu)
// plus a per-query radix select (knn_select.cuh).
#include "common.cuh"
#include "ptx.cuh"
#include "topk.cuh"
#include "pool_floor.cuh"
#include "merge_kernels.cuh"
#include "ivf_kernels.cuh"
#include "search_types.cuh"
#include "gemm.cuh"
#include "knn_select.cuh"

namespace crag {

// the 32 scores of row `row` of a score tile (layout: score_slot) -> r[q]
__device__ __forceinline__ void ld_score_row(const float* tile, int row, uint32_t (&r)[kNQ]) {
#pragma unroll
  for (int q = 0; q < kNQ; ++q) r[q] = __float_as_uint(tile[score_slot(row, q)]);
}

template <int KLIST, int CAP, int STAGES, bool IVF = false, bool SCORES = false>
__global__ void __launch_bounds__(kSearchThreads, 1)
search_topk_kernel(const __grid_constant__ CUtensorMap tm_corpus, const __grid_constant__ CUtensorMap tm_q,
                   int n_rows, int num_kb, int nq, int k, const uint64_t* __restrict__ after_keys,
                   uint64_t* __restrict__ pool, uint32_t perm_mul, int perm_shift, uint64_t* __restrict__ part_keys,
                   float* __restrict__ part_minmax, const typename IvfParam<IVF, SCORES>::type ivf) {
  using L = SearchLayout<KLIST, CAP, STAGES>;
  static_assert(L::smem_bytes() <= 227 * 1024, "stages, score tiles and candidate lists exceed 227 KB of shared memory");
  constexpr int kAccStages = L::kAccStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  uint8_t* stage_base = smem;
  float* score_tiles = reinterpret_cast<float*>(stage_base + STAGES * kStageTotalBytes);   // [kAccStages][128 * 32]
  uint64_t* keys = reinterpret_cast<uint64_t*>(stage_base + STAGES * kStageTotalBytes + kAccStages * kScoreTileBytes);
  uint64_t* bar_full = keys + kNQ * L::kKeysPerQuery;
  uint64_t* bar_empty = bar_full + STAGES;
  uint64_t* bar_tfull = bar_empty + STAGES;            // [kAccStages]
  uint64_t* bar_tempty = bar_tfull + kAccStages;       // [kAccStages]
  uint64_t* thr_key = bar_tempty + kAccStages;         // [kNQ]
  float* thr_f = reinterpret_cast<float*>(thr_key + kNQ);  // [kNQ]
  int* cnt = reinterpret_cast<int*>(thr_f + kNQ);          // [kNQ]
  float* red = reinterpret_cast<float*>(cnt + kNQ);        // [4][kNQ][2]
  uint64_t* bnd_key = reinterpret_cast<uint64_t*>(red + 4 * kNQ * 2);  // [kNQ] admit only keys < bnd_key
  float* bnd_f = reinterpret_cast<float*>(bnd_key + kNQ);              // [kNQ] score part of the bound
  uint64_t* floor_key = reinterpret_cast<uint64_t*>(bnd_f + kNQ);      // [kNQ] pooled admission floor (see kPoolM)
  uint64_t* part_floor = floor_key + kNQ;                              // [4][kNQ] scratch of a floor refresh

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int num_tiles;
  if constexpr (IVF) num_tiles = __ldg(ivf.n_work);
  else num_tiles = (n_rows + kTileRows - 1) / kTileRows;

  // Flat scans walk GROUPS of 2^perm_shift consecutive tiles in a multiplicative permutation of the row order
  // (perm_mul coprime to the number of whole groups; a ragged tail keeps its place): at any moment the CTAs sample the
  // whole shard, so a corpus whose scores drift along the row order (rows appended in narrative order, planted
  // neighbours in the tail) looks like a random one to the selector.  Neighbouring CTAs still stream neighbouring
  // tiles of one group (2 MB at shift 3 = one page of address translation), which is what HBM and the TLBs like.
#define CRAG_SELECT_SECTION 1
#include "select_warps.inc.cuh"

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
#define CRAG_SELECT_SECTION 2
#include "select_warps.inc.cuh"
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
        const int tile = tile_of(j);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&bar_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&bar_full[stage], kStageTotalBytes);
          int tile_row0;
          if constexpr (IVF) tile_row0 = __ldg(&ivf.work[tile].x);
          else tile_row0 = tile * kTileRows;
          uint8_t* st = stage_base + stage * kStageTotalBytes;
          tma_load_2d_hint(&tm_corpus, &bar_full[stage], st, kb * kBlockK, tile_row0, pol);
          tma_load_2d(&tm_q, &bar_full[stage], st + kStageBytes, kb * kBlockK, 0);
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
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float d[2][16];
#pragma unroll
      for (int i = 0; i < 16; ++i) d[0][i] = d[1][i] = 0.f;
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&bar_full[stage], phase);
        const uint32_t a_addr = smem_u32(stage_base + stage * kStageTotalBytes);
        const uint32_t b_addr = a_addr + kStageBytes;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kBlockK / 16; ++ks) {
          const uint64_t db = wgmma_desc_sw128(b_addr + ks * 32);
          wgmma_m64n32k16_ss(d[0], wgmma_desc_sw128(a_addr + ks * 32), db, 1u);
          wgmma_m64n32k16_ss(d[1], wgmma_desc_sw128(a_addr + 64 * 128 + ks * 32), db, 1u);
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
            st[score_slot(row, 8 * j + frag_col + (i & 1))] = d[m][4 * j + i];
          }
      mbar_arrive(&bar_tfull[acc]);
      if (++acc == kAccStages) { acc = 0; acc_phase ^= 1; }
    }
  } else {
    // ================================================================== select
#define CRAG_SELECT_SECTION 3
#include "select_warps.inc.cuh"
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

// cudaFuncSetAttribute once per kernel and device instead of on every launch.  `Tag` makes the cache unique per
// kernel instantiation (the kernels share one function-pointer TYPE, so the pointer type alone would alias them).
template <class Tag, class Kern>
int ensure_smem_attr(Kern kern, size_t smem) {
  static size_t done[64] = {0};
  int dev = 0;
  CRAG_CUDA_OK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || done[dev] < smem) {
    CRAG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    if (dev >= 0 && dev < 64) done[dev] = smem;
  }
  return CRAG_OK;
}
template <int KLIST, int CAP, int STAGES, bool IVF, bool SCORES> struct KernelTag {};

template <int KLIST, int CAP, int STAGES>
int launch_search(const CUtensorMap& tm_corpus, const CUtensorMap& tm_q, int n_rows, int num_kb, int nq, int k,
                  int grid, const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul, int perm_shift,
                  uint64_t* part_keys, float* part_minmax, cudaStream_t stream) {
  using L = SearchLayout<KLIST, CAP, STAGES>;
  const size_t smem = L::smem_bytes();
  auto kern = search_topk_kernel<KLIST, CAP, STAGES>;
  int rc = ensure_smem_attr<KernelTag<KLIST, CAP, STAGES, false, false>>(kern, smem);
  if (rc != CRAG_OK) return rc;
  kern<<<grid, kSearchThreads, smem, stream>>>(tm_corpus, tm_q, n_rows, num_kb, nq, k, after_keys, pool, perm_mul,
                                               perm_shift, part_keys, part_minmax, NoIvfArgs{});
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

template <int KLIST, int CAP, int STAGES>
int launch_ivf_scan(const CUtensorMap& tm_res, const CUtensorMap& tm_q, int num_kb, int nq, int k, int grid,
                    uint64_t* pool, uint64_t* part_keys, float* part_minmax, const IvfArgs& ivf, cudaStream_t stream) {
  using L = SearchLayout<KLIST, CAP, STAGES>;
  const size_t smem = L::smem_bytes();
  auto kern = search_topk_kernel<KLIST, CAP, STAGES, true>;
  int rc = ensure_smem_attr<KernelTag<KLIST, CAP, STAGES, true, false>>(kern, smem);
  if (rc != CRAG_OK) return rc;
  kern<<<grid, kSearchThreads, smem, stream>>>(tm_res, tm_q, 0, num_kb, nq, k, nullptr, pool, 0u, 0, part_keys, part_minmax, ivf);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
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

// one corpus pass for <= 32 queries: per-CTA partial lists into the workspace
int scan_pass(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride, const void* queries, int nq,
              int k, const uint64_t* after_keys, void* workspace, size_t workspace_bytes, const SearchPlan& plan,
              cudaStream_t stream) {
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
  int rc = make_tmap_bf16_2d(&tm_corpus, corpus, uint64_t(n_rows), uint64_t(dim), uint64_t(corpus_row_stride) * 2, kTileRows);
  if (rc != CRAG_OK) return rc;
  rc = make_tmap_bf16_2d(&tm_q, queries, uint64_t(nq), uint64_t(dim), uint64_t(dim) * 2, kNQ);
  if (rc != CRAG_OK) return rc;
  const int num_kb = dim / kBlockK;
  // A/B switches for measurements (read once): CRAG_SEARCH_PERM_SHIFT = -1 (natural order) | 0..6, CRAG_SEARCH_POOL = 0
  static const int env_shift = [] { const char* e = getenv("CRAG_SEARCH_PERM_SHIFT"); return e ? atoi(e) : 3; }();
  static const bool env_pool = [] { const char* e = getenv("CRAG_SEARCH_POOL"); return e ? atoi(e) != 0 : true; }();
  if (!env_pool) pool = nullptr;
  const int shift = env_shift < 0 ? 0 : (env_shift > 6 ? 6 : env_shift);
  const uint32_t perm = env_shift < 0 ? 0u : perm_multiplier(num_tiles >> shift);
  if (k <= 64) return launch_search<64, 64, 6>(tm_corpus, tm_q, int(n_rows), num_kb, nq, k, grid, after_keys, pool, perm, shift, part_keys, part_minmax, stream);
  return launch_search<128, 128, 4>(tm_corpus, tm_q, int(n_rows), num_kb, nq, k, grid, after_keys, pool, perm, shift, part_keys, part_minmax, stream);
}

// merge the per-CTA partials of one pass into the final (ids, scores, minmax) of its <= 32 queries
int finalize_parts(const void* workspace, int grid, int nq, int k, int64_t row_offset, int64_t* out_ids,
                   float* out_scores, float* out_minmax, uint64_t* last_keys, const SearchPlan& plan, cudaStream_t stream) {
  const uint64_t* part_keys = static_cast<const uint64_t*>(workspace);
  const float* part_minmax = reinterpret_cast<const float*>(static_cast<const uint8_t*>(workspace) + plan.keys_bytes);
  const int mgrid = nq;  // one CTA per query
  if (k <= 32)
    merge_topk_kernel<32, 32, false><<<mgrid, 128, 0, stream>>>(part_keys, nullptr, nullptr, part_minmax, grid, kNQ, nq, k, row_offset, 0, 0, 0, out_ids, out_scores, out_minmax, last_keys);
  else if (k <= 64)
    merge_topk_kernel<64, 64, false><<<mgrid, 128, 0, stream>>>(part_keys, nullptr, nullptr, part_minmax, grid, kNQ, nq, k, row_offset, 0, 0, 0, out_ids, out_scores, out_minmax, last_keys);
  else
    merge_topk_kernel<128, 128, false><<<mgrid, 128, 0, stream>>>(part_keys, nullptr, nullptr, part_minmax, grid, kNQ, nq, k, row_offset, 0, 0, 0, out_ids, out_scores, out_minmax, last_keys);
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
    rc = make_tmap_bf16_2d(&tm_q, static_cast<const uint8_t*>(queries) + size_t(q0) * dim * 2, uint64_t(nqc), uint64_t(dim), uint64_t(dim) * 2, kNQ);
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
    rc = (k <= 64) ? launch_ivf_scan<64, 64, 6>(tm_res, tm_q, num_kb, nqc, k, sp.grid, pool, part_keys, part_minmax, ivf, stream)
                   : launch_ivf_scan<128, 128, 4>(tm_res, tm_q, num_kb, nqc, k, sp.grid, pool, part_keys, part_minmax, ivf, stream);
    if (rc != CRAG_OK) return rc;
    rc = finalize_parts(workspace, sp.grid, nqc, k, 0, out_ids + size_t(q0) * k, out_scores + size_t(q0) * k,
                        out_minmax ? out_minmax + size_t(q0) * 2 : nullptr, nullptr, sp, stream);
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
  return scan_pass(corpus, n_rows, dim, corpus_row_stride, queries, nq, k, nullptr, workspace, workspace_bytes, plan, static_cast<cudaStream_t>(stream));
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
    const uint8_t* qptr = static_cast<const uint8_t*>(queries) + size_t(q0) * dim * 2;
    rc = scan_pass(corpus, n_rows, dim, corpus_row_stride, qptr, nqc, k, after_keys ? after_keys + q0 : nullptr, workspace,
                   workspace_bytes, plan, stream);
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
  const int mgrid = nq;  // one CTA per query
  const float* mm = out_minmax ? minmax : nullptr;
  if (k <= 32)
    merge_topk_kernel<32, 32, true><<<mgrid, 128, 0, stream>>>(nullptr, scores, ids, mm, parts, nq, nq, k, 0, ids_stride, scores_stride, mm_stride, out_ids, out_scores, out_minmax, nullptr);
  else if (k <= 64)
    merge_topk_kernel<64, 64, true><<<mgrid, 128, 0, stream>>>(nullptr, scores, ids, mm, parts, nq, nq, k, 0, ids_stride, scores_stride, mm_stride, out_ids, out_scores, out_minmax, nullptr);
  else
    merge_topk_kernel<128, 128, true><<<mgrid, 128, 0, stream>>>(nullptr, scores, ids, mm, parts, nq, nq, k, 0, ids_stride, scores_stride, mm_stride, out_ids, out_scores, out_minmax, nullptr);
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
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a = fminf(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
  if (lane == 0) {
    out[size_t(q) * 2 + 0] = a;
    out[size_t(q) * 2 + 1] = b;
  }
}
}  // namespace
}  // namespace crag

extern "C" int crag_search_scores(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                  const void* queries, int nq, float* out_scores, int64_t out_ld, float* out_minmax,
                                  void* workspace, size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SearchPlan plan = plan_search(1);
  int rc = check_search_args(corpus, n_rows, dim, corpus_row_stride, queries, nq, 1, workspace, workspace_bytes, plan);
  if (rc != CRAG_OK) return rc;
  if (!out_scores || out_ld < n_rows) return fail(CRAG_ERR_INVALID, "crag_search_scores: need out_scores and out_ld >= n_rows");
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
  rc = make_tmap_bf16_2d(&tm_corpus, corpus, uint64_t(n_rows), uint64_t(dim), uint64_t(corpus_row_stride) * 2, kTileRows);
  if (rc != CRAG_OK) return rc;
  const int num_kb = dim / kBlockK;
  using L = SearchLayout<16, 16, 7>;
  auto kern = search_topk_kernel<16, 16, 7, false, true>;
  const size_t smem = L::smem_bytes();
  rc = ensure_smem_attr<KernelTag<16, 16, 7, false, true>>(kern, smem);
  if (rc != CRAG_OK) return rc;
  for (int q0 = 0; q0 < nq; q0 += kNQ) {
    const int nqc = (nq - q0) < kNQ ? (nq - q0) : kNQ;
    CUtensorMap tm_q;
    rc = make_tmap_bf16_2d(&tm_q, static_cast<const uint8_t*>(queries) + size_t(q0) * dim * 2, uint64_t(nqc), uint64_t(dim), uint64_t(dim) * 2, kNQ);
    if (rc != CRAG_OK) return rc;
    ScoreArgs sa{out_scores + int64_t(q0) * out_ld, out_ld, nullptr, nullptr, 0};
    kern<<<grid, kSearchThreads, smem, stream>>>(tm_corpus, tm_q, int(n_rows), num_kb, nqc, 1, nullptr, nullptr, 0u, 0, nullptr,
                                                 part_minmax, sa);
    CRAG_CUDA_OK(cudaGetLastError());
    if (out_minmax) {
      minmax_reduce_kernel<<<nqc, 32, 0, stream>>>(part_minmax, grid, nqc, out_minmax + size_t(q0) * 2);
      CRAG_CUDA_OK(cudaGetLastError());
    }
  }
  return CRAG_OK;
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
  if (k <= 32)
    finalize_exchange_kernel<32, 32><<<nq, 128, 0, stream>>>(part_keys, part_minmax, parts, nq, k, row_offset, peer_bufs, rank, world, epochs, status, out_ids, out_scores, out_minmax);
  else if (k <= 64)
    finalize_exchange_kernel<64, 64><<<nq, 128, 0, stream>>>(part_keys, part_minmax, parts, nq, k, row_offset, peer_bufs, rank, world, epochs, status, out_ids, out_scores, out_minmax);
  else
    finalize_exchange_kernel<128, 128><<<nq, 128, 0, stream>>>(part_keys, part_minmax, parts, nq, k, row_offset, peer_bufs, rank, world, epochs, status, out_ids, out_scores, out_minmax);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

// IVF build, assignment step: list of every row = argmax over the centroid table of bf16(row) . bf16(centroid) with fp32
// accumulation, ties to the smaller list id (oracle/ivf_oracle.py `assign`).  The rows are the "corpus" of the scan
// kernel and the centroids its query blocks (32 per pass): nlist / 32 passes over the rows, each row keeping its
// running best in (best_score, best_id).  Replaces a torch matmul + argmax over [rows, nlist] score blocks.
extern "C" int crag_ivf_assign(const void* rows, int64_t n_rows, int dim, int64_t row_stride, const void* centroids,
                               int nlist, float* best_score, int32_t* best_id, void* workspace, size_t workspace_bytes,
                               crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SearchPlan plan = plan_search(1);
  int rc = check_search_args(rows, n_rows, dim, row_stride, centroids, nlist, 1, workspace, workspace_bytes, plan);
  if (rc != CRAG_OK) return rc;
  if (!best_score || !best_id) return fail(CRAG_ERR_INVALID, "crag_ivf_assign: null output pointer");
  const int grid = scan_grid(n_rows, plan);
  if (grid == 0) return CRAG_OK;
  float* part_minmax = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + plan.keys_bytes);
  CUtensorMap tm_rows;
  rc = make_tmap_bf16_2d(&tm_rows, rows, uint64_t(n_rows), uint64_t(dim), uint64_t(row_stride) * 2, kTileRows);
  if (rc != CRAG_OK) return rc;
  const int num_kb = dim / kBlockK;
  using L = SearchLayout<16, 16, 7>;
  auto kern = search_topk_kernel<16, 16, 7, false, true>;
  const size_t smem = L::smem_bytes();
  rc = ensure_smem_attr<KernelTag<16, 16, 7, false, true>>(kern, smem);
  if (rc != CRAG_OK) return rc;
  // the pass over centroid block 0 initialises every row's running best (-inf, list 0); later passes update it
  for (int q0 = 0; q0 < nlist; q0 += kNQ) {
    const int nqc = (nlist - q0) < kNQ ? (nlist - q0) : kNQ;
    CUtensorMap tm_q;
    rc = make_tmap_bf16_2d(&tm_q, static_cast<const uint8_t*>(centroids) + size_t(q0) * dim * 2, uint64_t(nqc), uint64_t(dim), uint64_t(dim) * 2, kNQ);
    if (rc != CRAG_OK) return rc;
    ScoreArgs sa{nullptr, 0, best_score, best_id, q0};
    kern<<<grid, kSearchThreads, smem, stream>>>(tm_rows, tm_q, int(n_rows), num_kb, nqc, 1, nullptr, nullptr, 0u, 0, nullptr,
                                                 part_minmax, sa);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}
