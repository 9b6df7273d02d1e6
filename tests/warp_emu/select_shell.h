// search_topk_kernel's select warps inside a host function (see select_emu_test.cpp): csrc/select_warps.inc.cuh is the
// text the kernel #includes; here the same three sections are included with the score-tile read mapped to a score
// matrix the caller supplies, mbarrier waits to nothing and the named barriers to the fiber emulator.
#pragma once
#include <cuda_runtime.h>   // the stub

#include "ivf_kernels.cuh"
#include "merge_kernels.cuh"
#include "search_types.cuh"

namespace crag {

// ---- host stand-ins for the ptx.cuh operations the select warps use
static inline void mbar_wait(uint64_t*, uint32_t) {}
static inline void mbar_arrive(uint64_t*) {}
static inline void named_bar_sync(uint32_t id, uint32_t n) { warp_emu::named_barrier(int(id), int(n)); }
static inline bool named_bar_or(uint32_t id, uint32_t n, bool p) { return warp_emu::named_barrier_or(int(id), int(n), p); }

// the score tiles: scores[row * kNQ + q]; rows past the end read as 0 (TMA zero-fills out-of-bounds boxes)
struct ScoreSource {
  const float* scores = nullptr;
  int64_t rows = 0;
  const int4* work = nullptr;      // IVF: the tile index is a work-list index, the rows are work[tile].x + ...
};
static thread_local ScoreSource g_src;
static inline void emu_score_ld(int tile, int quad, int lane, uint32_t (&r)[32]) {
  const int64_t row = (g_src.work ? int64_t(g_src.work[tile].x) : int64_t(tile) * kTileRows) + quad * 32 + lane;
  for (int q = 0; q < kNQ; ++q) r[q] = row < g_src.rows ? __float_as_uint(g_src.scores[row * kNQ + q]) : 0u;
}
// the kernel's call is ld_score_row(<score tile>, <row in tile>, r); `tile`, `quad`, `lane` are locals of the included text
#define ld_score_row(buf, row_in_tile, r) emu_score_ld(tile, quad, lane, r)

// search_topk_kernel without its producer / MMA warps: same parameter names, same local names.  Launch with
// select_shell_smem_bytes<KLIST, CAP>() of dynamic shared memory.
template <int KLIST, int CAP>
constexpr size_t select_shell_smem_bytes() {
  return size_t(kNQ) * (KLIST + CAP) * 8 + 2 * SearchLayout<KLIST, CAP, 1>::kAccStages * 8 + kNQ * (8 + 4 + 4) + 4 * kNQ * 2 * 4 + kNQ * (8 + 4 + 8) + 4 * kNQ * 8 + 64;
}

template <int KLIST, int CAP, int STAGES, bool IVF = false, bool SCORES = false>
static void search_select_shell(int n_rows, int nq, int k, const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul,
                                int perm_shift, uint64_t* part_keys, float* part_minmax,
                                const typename IvfParam<IVF, SCORES>::type ivf) {
  using L = SearchLayout<KLIST, CAP, STAGES>;
  constexpr int kAccStages = L::kAccStages;
  // the selector state, carved out of the block's dynamic shared memory as the kernel carves it out of smem_raw
  uint8_t* smem = static_cast<uint8_t*>(warp_emu::dynamic_shared());
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem);
  uint64_t* bar_tfull = keys + kNQ * L::kKeysPerQuery;          // [kAccStages]  (never waited on here)
  uint64_t* bar_tempty = bar_tfull + kAccStages;                // [kAccStages]
  uint64_t* thr_key = bar_tempty + kAccStages;                  // [kNQ]
  float* thr_f = reinterpret_cast<float*>(thr_key + kNQ);       // [kNQ]
  int* cnt = reinterpret_cast<int*>(thr_f + kNQ);               // [kNQ]
  float* red = reinterpret_cast<float*>(cnt + kNQ);             // [4][kNQ][2]
  uint64_t* bnd_key = reinterpret_cast<uint64_t*>(red + 4 * kNQ * 2);
  float* bnd_f = reinterpret_cast<float*>(bnd_key + kNQ);
  uint64_t* floor_key = reinterpret_cast<uint64_t*>(bnd_f + kNQ);
  uint64_t* part_floor = floor_key + kNQ;                       // [4][kNQ]
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int num_tiles;
  if constexpr (IVF) num_tiles = __ldg(ivf.n_work);
  else num_tiles = (n_rows + kTileRows - 1) / kTileRows;
#define CRAG_SELECT_SECTION 1
#include "select_warps.inc.cuh"
#define CRAG_SELECT_SECTION 2
#include "select_warps.inc.cuh"
  __syncthreads();
  const float* score_tiles = nullptr;
  (void)score_tiles; (void)bar_tfull; (void)bar_tempty;
  if (warp >= kMmaWarp0) return;   // the wgmma warpgroup and the TMA producer: nothing to emulate
  {
#define CRAG_SELECT_SECTION 3
#include "select_warps.inc.cuh"
  }
}

}  // namespace crag
