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

// ------------------------------------------------------------------ wide stage 1 (crag_ivf_search_i8_wide / _pq_wide)
// Query q's probed rows are the real rows of its distinct valid probes.  Their slot order takes the lists in ascending
// list id and the rows in stored order inside each list; lists are stored back to back in list order, so slot order is
// stored-position order.  Slot s of q holds S1 at block[q * ld + s] for s < cap (= max_probe_rows, ld = cap rounded up
// to 4); the rows of a query past cap are not scored.
constexpr int kIvfMaxProbe = 128;   // probes per query

struct IvfWidePlan {
  int32_t* slot_base;   // [nlist][kNQ]: first slot of list l for a query q that probes it
  int32_t* seg_list;    // [kNQ][kIvfMaxProbe]: q's non-empty lists whose first slot is below cap, in slot order
  int32_t* seg_slot;    // [kNQ][kIvfMaxProbe]: their first slots
  int32_t* n_seg;       // [kNQ]
  int32_t* n_rows;      // [kNQ]: n_q = min(probed rows, cap)
};

// One CTA of kIvfMaxProbe threads per query of the pass (nprobe <= kIvfMaxProbe): drops invalid and repeated probes,
// ranks the rest by list id, and lays the lists out in slot order.
__global__ void __launch_bounds__(kIvfMaxProbe) ivf_wide_plan_kernel(const int64_t* __restrict__ probed_ids, int nprobe,
                                                                    int nlist, const int32_t* __restrict__ list_rows,
                                                                    int cap, IvfWidePlan wp) {
  __shared__ int s_probe[kIvfMaxProbe];
  __shared__ int s_keep[kIvfMaxProbe];
  __shared__ int s_list[kIvfMaxProbe];
  __shared__ int s_rows[kIvfMaxProbe];
  const int q = blockIdx.x, t = threadIdx.x;
  int l = -1;
  if (t < nprobe) {
    const int64_t v = probed_ids[int64_t(q) * nprobe + t];
    if (v >= 0 && v < nlist) l = int(v);
  }
  s_probe[t] = l;
  __syncthreads();
  bool keep = l >= 0;   // the first occurrence of a list stands for all of them
  for (int u = 0; u < t; ++u) keep = keep && s_probe[u] != l;
  s_keep[t] = keep;
  __syncthreads();
  int rank = 0, n_lists = 0;
  for (int u = 0; u < kIvfMaxProbe; ++u) {
    if (!s_keep[u]) continue;
    ++n_lists;
    rank += s_probe[u] < l ? 1 : 0;
  }
  if (keep) {
    const int rows = __ldg(&list_rows[l]);
    s_list[rank] = l;
    s_rows[rank] = rows > 0 ? rows : 0;
  }
  __syncthreads();
  if (t == 0) {
    int64_t slot = 0;
    int n_seg = 0;
    for (int i = 0; i < n_lists; ++i) {
      const int li = s_list[i];
      wp.slot_base[int64_t(li) * kNQ + q] = int32_t(slot);
      if (s_rows[i] > 0 && slot < cap) {
        wp.seg_list[q * kIvfMaxProbe + n_seg] = li;
        wp.seg_slot[q * kIvfMaxProbe + n_seg] = int32_t(slot);
        ++n_seg;
      }
      slot += s_rows[i];
    }
    wp.n_seg[q] = n_seg;
    wp.n_rows[q] = int32_t(slot < cap ? slot : cap);
  }
}

// The select's slot ids -> stored positions, in place: slot s of query q lies in q's last segment whose first slot is
// <= s.  cand: [nq][n_cand], -1 stays -1.
__global__ void ivf_slot_map_kernel(int64_t* __restrict__ cand, int nq, int n_cand, const IvfWidePlan wp,
                                    const int32_t* __restrict__ list_tile_start) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq * n_cand) return;
  const int64_t s = cand[i];
  if (s < 0) return;
  const int q = i / n_cand;
  const int32_t* first = wp.seg_slot + q * kIvfMaxProbe;
  int lo = 0, hi = wp.n_seg[q] - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= s) lo = mid;
    else hi = mid - 1;
  }
  const int l = wp.seg_list[q * kIvfMaxProbe + lo];
  cand[i] = int64_t(__ldg(&list_tile_start[l])) * kTileRows + (s - first[lo]);
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
