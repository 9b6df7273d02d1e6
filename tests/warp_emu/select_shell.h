// search_topk_kernel's select warps inside a host function (see select_emu_test.cpp): the kernel's own select_warps()
// and SelectSmem from csrc/select_warps.cuh, fed by a score-tile source that reads a score matrix the caller supplies.
#pragma once
#include <cuda_runtime.h>   // the stub

#include "ivf_kernels.cuh"
#include "merge_kernels.cuh"
#include "search_types.cuh"
#include "select_warps.cuh"

namespace crag {

// the score tiles: scores[row * kNQ + q]; rows past the end read as 0 (TMA zero-fills out-of-bounds boxes)
struct MatrixScoreTiles {
  const float* scores = nullptr;
  int64_t rows = 0;
  const int4* work = nullptr;      // IVF: the tile index is a work-list index, the rows are work[tile].x + ...
  void next(int tile, int quad, int lane, uint32_t (&r)[kNQ]) const {
    const int64_t row = (work ? int64_t(work[tile].x) : int64_t(tile) * kTileRows) + quad * 32 + lane;
    for (int q = 0; q < kNQ; ++q) r[q] = row < rows ? __float_as_uint(scores[row * kNQ + q]) : 0u;
  }
};
static thread_local MatrixScoreTiles g_src;

// search_topk_kernel without its producer / MMA warps: the same parameters and the same selector calls.  Launch with
// SelectSmem<KLIST, CAP>::bytes() of dynamic shared memory.
template <int KLIST, int CAP, bool IVF = false, bool SCORES = false>
static void search_select_shell(int n_rows, int nq, int k, const uint64_t* after_keys, uint64_t* pool, uint32_t perm_mul, int perm_shift,
                                uint64_t* part_keys, float* part_minmax, const typename IvfParam<IVF, SCORES>::type args) {
  const auto sel = SelectSmem<KLIST, CAP>::carve(static_cast<uint8_t*>(warp_emu::dynamic_shared()));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int num_tiles;
  if constexpr (IVF) num_tiles = __ldg(args.n_work);
  else num_tiles = (n_rows + kTileRows - 1) / kTileRows;
  const TileOrder order(num_tiles, perm_mul, perm_shift);
  sel.init(nq, after_keys);
  __syncthreads();
  if (warp >= kMmaWarp0) return;   // the wgmma warpgroup and the TMA producer: nothing to emulate
  MatrixScoreTiles tiles = g_src;
  select_warps<KLIST, CAP, IVF, SCORES>(sel, tiles, order, num_tiles, n_rows, nq, k, after_keys, pool, part_keys, part_minmax, args, warp, lane);
}

}  // namespace crag
