// The IVF search's two integer kernels (BASELINE config 4; semantic: oracle/ivf_oracle.py): the per-pass plan -- which
// queries probe which list, their coarse terms, the work-list of probed tiles -- and the mapping of stored-row ids back
// to original ids.  Plain SIMT code, kept in a header so tests/warp_emu can run them against a direct restatement.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#include "pool_floor.cuh"   // kNQ, kTileRows

namespace crag {

// Builds one IVF pass's plan on the device (single CTA): which queries probe which list, their coarse terms, and the
// work-list of the probed lists' tiles.  probed_ids / probed_scores are the coarse top-nprobe of each query
// (crag_search_topk over the centroid table; id -1 = fewer than nprobe lists).
__global__ void __launch_bounds__(1024) ivf_plan_kernel(const int64_t* __restrict__ probed_ids,
                                                        const float* __restrict__ probed_scores, int nq, int nprobe,
                                                        int nlist, const int32_t* __restrict__ list_tile_start,
                                                        const int32_t* __restrict__ list_rows,
                                                        uint32_t* __restrict__ list_mask, float* __restrict__ coarse,
                                                        int4* __restrict__ work, int* __restrict__ n_work) {
  __shared__ int s_count;
  if (threadIdx.x == 0) s_count = 0;
  for (int l = threadIdx.x; l < nlist; l += blockDim.x) list_mask[l] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < nq * nprobe; i += blockDim.x) {
    const int64_t l = probed_ids[i];
    if (l < 0 || l >= nlist) continue;
    const int q = i / nprobe;
    atomicOr(&list_mask[l], 1u << q);
    coarse[size_t(l) * kNQ + q] = probed_scores[i];
  }
  __syncthreads();
  for (int l = threadIdx.x; l < nlist; l += blockDim.x) {
    const int rows = list_rows[l];
    if (list_mask[l] == 0u || rows <= 0) continue;
    const int tiles = (rows + kTileRows - 1) / kTileRows;
    const int at = atomicAdd(&s_count, tiles);
    const int t0 = list_tile_start[l];
    for (int j = 0; j < tiles; ++j)
      work[at + j] = make_int4((t0 + j) * kTileRows, min(kTileRows, rows - j * kTileRows), l, 0);
  }
  __syncthreads();
  if (threadIdx.x == 0) *n_work = s_count;
}

// stored-row ids of the merged answer -> the rows' original ids (-1 stays -1)
__global__ void ivf_map_ids_kernel(int64_t* __restrict__ ids, int n, const int64_t* __restrict__ row_ids) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const int64_t v = ids[i];
    ids[i] = v >= 0 ? row_ids[v] : -1;
  }
}

}  // namespace crag
