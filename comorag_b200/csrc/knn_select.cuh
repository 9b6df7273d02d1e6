// Exact per-query top-k (k <= 2048) over a row of fp32 scores: the select half of crag_knn_topk (search.cu), which
// first writes a [q_chunk, ld] score block with the wgmma GEMM (gemm.cu, epilogue GEMM_EPI_SCORES_F32).
//
// One CTA per query row.  Ordering is make_key's (topk.cuh): score descending, then row ascending -- the order of
// crag_search_topk, so both paths rank the same rows the same way.
//   1. radix select on orderable_f32(score): three passes with 11/11/10-bit digits and a 2048-bin shared histogram,
//      each counting only rows whose higher digits match the prefix found so far, give the k-th best score word T
//      and `quota`, how many of the k rows score exactly T (k - quota rows score above it);
//   2. gather, one pass in row order: every row above T goes to the candidate list, and the FIRST `quota` rows equal
//      to T in ascending row order (a running block-wide exclusive scan per tile of rows, which stops once the quota
//      is met) -- ties then resolve to ascending row ids exactly, as make_key orders them;
//   3. bitonic sort of the <= 2048 collected keys in shared memory (16 KB, knn_sort.cuh), ids row + row_offset out.
// (min, max) over all rows is reduced in the gather pass.  n_rows <= k skips step 1 and sorts every row.
// Pure SIMT code with no wgmma / TMA / mbarrier in it, so tests/warp_emu runs this very header on emulated blocks.
// This file is also the body of the select kernels: each includes it with CRAG_KNN_SELECT_BODY defined and gets the
// text of the select (the #if branch below), which reads the names the kernel declares -- scores, ld, n_rows, k,
// row_offset, out_ids, out_scores, out_minmax -- and selects for block q = blockIdx.x.  It is text rather than a device
// function because wrapping it in one, even inlined, changes knn_select_kernel's SASS: nvcc optimises the callee
// before inlining it.
#if defined(CRAG_KNN_SELECT_BODY)
  __shared__ uint32_t s_hist[kKnnBins];
  __shared__ uint64_t s_keys[kKnnMaxK];
  __shared__ int s_warp[kKnnWarps];
  __shared__ uint32_t s_mm[2][kKnnWarps];
  __shared__ int s_sel[3];
  __shared__ int s_slot;
  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float4* row4 = reinterpret_cast<const float4*>(scores + int64_t(q) * ld);
  const int n4 = (n_rows + 3) >> 2;
  const bool take_all = n_rows <= k;

  // ---- 1. radix select: T = the k-th best score word (prefix after three digits), quota = how many of the k kept
  // rows score exactly T, n_eq = how many rows score exactly T (>= quota)
  uint32_t prefix = 0;
  int quota = k;
  int n_eq = 0;
  if (!take_all) {
    for (int pass = 0; pass < 3; ++pass) {
      const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
      const int bits = pass == 2 ? 10 : 11;
      const int nbins = 1 << bits;
      for (int i = tid; i < kKnnBins; i += kKnnThreads) s_hist[i] = 0u;
      __syncthreads();
      for (int i0 = tid; i0 < n4; i0 += kKnnLoads * kKnnThreads) {
        float4 v[kKnnLoads];   // all loads of the batch in flight before the first histogram update
#pragma unroll
        for (int t = 0; t < kKnnLoads; ++t)
          if (i0 + t * kKnnThreads < n4) v[t] = row4[i0 + t * kKnnThreads];
#pragma unroll
        for (int t = 0; t < kKnnLoads; ++t) {
          const int i = i0 + t * kKnnThreads;
          if (i >= n4) break;
          const float e[4] = {v[t].x, v[t].y, v[t].z, v[t].w};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (4 * i + c >= n_rows) break;
            const uint32_t u = orderable_f32(e[c]);
            if (pass == 0 || (u >> (shift + bits)) == prefix) atomicAdd(&s_hist[(u >> shift) & uint32_t(nbins - 1)], 1u);
          }
        }
      }
      __syncthreads();
      // thread t owns bins top, top - 1, top - 2, top - 3 (top = nbins - 1 - 4t): scanning threads in order walks
      // the bins from the highest score down, so `above` = rows of this prefix in higher bins
      const int top = nbins - 1 - 4 * tid;
      int h[4] = {0, 0, 0, 0};
      if (top >= 0) {
#pragma unroll
        for (int c = 0; c < 4; ++c) h[c] = int(s_hist[top - c]);
      }
      int total = 0;
      int above = knn_block_exclusive_scan(h[0] + h[1] + h[2] + h[3], s_warp, &total);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (above < quota && above + h[c] >= quota) {   // the quota-th row of this prefix falls in bin top - c
          s_sel[0] = top - c;
          s_sel[1] = quota - above;
          s_sel[2] = h[c];
        }
        above += h[c];
      }
      __syncthreads();
      prefix = (prefix << bits) | uint32_t(s_sel[0]);
      quota = s_sel[1];
      n_eq = s_sel[2];
      __syncthreads();   // s_sel is rewritten by the next pass
    }
  }
  const uint32_t T = prefix;
  // Only when some rows equal to T must be left out does their order matter; otherwise (distinct scores: n_eq ==
  // quota == 1) every kept row goes through the unordered path and no tile pays for a block scan.
  const bool ordered_ties = !take_all && quota < n_eq;
  const int count = take_all ? n_rows : k;               // keys kept: min(k, n_rows)
  const int c_above = ordered_ties ? k - quota : count;  // keys kept without a tie decision

  // ---- 2. gather in row order
  if (tid == 0) s_slot = 0;
  __syncthreads();
  uint32_t mn = 0xFFFFFFFFu, mx = 0u;
  int taken_ties = 0;   // block-uniform running count of rows equal to T seen so far
  for (int base = 0; base < n4; base += kKnnThreads) {
    const int i = base + tid;
    float e[4] = {0.f, 0.f, 0.f, 0.f};
    if (i < n4) {
      const float4 v = row4[i];
      e[0] = v.x; e[1] = v.y; e[2] = v.z; e[3] = v.w;
    }
    uint32_t u[4];
    bool keep[4], tie[4];
    int n_keep = 0, n_tie = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const bool live = i < n4 && 4 * i + c < n_rows;
      u[c] = orderable_f32(e[c]);
      keep[c] = live && (take_all || u[c] > T || (!ordered_ties && u[c] == T));
      tie[c] = live && ordered_ties && u[c] == T;
      if (live) {
        mn = u[c] < mn ? u[c] : mn;
        mx = u[c] > mx ? u[c] : mx;
      }
      n_keep += keep[c] ? 1 : 0;
      n_tie += tie[c] ? 1 : 0;
    }
    if (n_keep) {   // these rows may land in any order: the sort fixes it
      int slot = atomicAdd(&s_slot, n_keep);
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (keep[c]) s_keys[slot++] = make_key(e[c], uint32_t(4 * i + c));
    }
    if (ordered_ties && taken_ties < quota) {   // block-uniform: the scan stops once the first `quota` ties are in
      int total = 0;
      int r = knn_block_exclusive_scan(n_tie, s_warp, &total) + taken_ties;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (tie[c]) {
          if (r < quota) s_keys[c_above + r] = make_key(e[c], uint32_t(4 * i + c));
          ++r;
        }
      }
      taken_ties += total;
    }
  }
  mn = __reduce_min_sync(0xffffffffu, mn);
  mx = __reduce_max_sync(0xffffffffu, mx);
  if (lane == 0) {
    s_mm[0][warp] = mn;
    s_mm[1][warp] = mx;
  }

  // ---- 3. bitonic sort (descending) of the kept keys, zero-padded to a power of two
  knn_bitonic_sort(s_keys, count, tid);
  int64_t* oi = out_ids + int64_t(q) * k;
  float* os = out_scores + int64_t(q) * k;
  for (int j = tid; j < k; j += kKnnThreads) {
    if (j < count) {
      const uint64_t key = s_keys[j];
      oi[j] = int64_t(key_id(key)) + row_offset;
      os[j] = key_score(key);
    } else {
      oi[j] = -1;
      os[j] = -INFINITY;
    }
  }
  if (out_minmax && tid == 0) {
    uint32_t a = 0xFFFFFFFFu, b = 0u;
    for (int w = 0; w < kKnnWarps; ++w) {
      a = s_mm[0][w] < a ? s_mm[0][w] : a;
      b = s_mm[1][w] > b ? s_mm[1][w] : b;
    }
    out_minmax[int64_t(q) * 2 + 0] = n_rows > 0 ? unorderable_f32(a) : INFINITY;
    out_minmax[int64_t(q) * 2 + 1] = n_rows > 0 ? unorderable_f32(b) : -INFINITY;
  }
#elif !defined(CRAG_KNN_SELECT_CUH)
#define CRAG_KNN_SELECT_CUH
#include <stdint.h>
#include <cuda_runtime.h>

#include "knn_sort.cuh"
#include "topk.cuh"

namespace crag {
namespace {

constexpr int kKnnBins = 2048;
constexpr int kKnnLoads = 4;   // 16-byte loads per thread in flight in a histogram pass

// Exclusive scan of v over the block's threads in threadIdx order; *total = the sum over all threads.
__device__ __forceinline__ int knn_block_exclusive_scan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_sync(0xffffffffu, x, lane >= o ? lane - o : lane);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kKnnWarps; ++w) {
    const int c = s_warp[w];
    before += w < warp ? c : 0;
    all += c;
  }
  __syncthreads();   // s_warp is free for the next call
  *total = all;
  return before + x - v;
}

// scores: fp32 rows of `ld` floats (ld % 4 == 0, 16-byte aligned), block q reads row q; outputs [gridDim.x, k].
__global__ void __launch_bounds__(kKnnThreads)
knn_select_kernel(const float* __restrict__ scores, int64_t ld, int n_rows, int k, int64_t row_offset,
                  int64_t* __restrict__ out_ids, float* __restrict__ out_scores, float* __restrict__ out_minmax) {
#define CRAG_KNN_SELECT_BODY
#include "knn_select.cuh"
#undef CRAG_KNN_SELECT_BODY
}

// The ragged select of the wide IVF stage 1 (crag_ivf_search_i8_wide / _pq_wide): block q ranks the first n_q[q] slots
// of row q of the pass's S1 block (ivf_wide_plan_kernel's row counts) and writes slot ids, which ivf_slot_map_kernel
// turns into stored positions.
__global__ void __launch_bounds__(kKnnThreads)
ivf_wide_select_kernel(const float* __restrict__ scores, int64_t ld, const int32_t* __restrict__ n_q, int k,
                       int64_t* __restrict__ out_ids, float* __restrict__ out_scores, float* __restrict__ out_minmax) {
  const int n_rows = __ldg(&n_q[blockIdx.x]);
  const int64_t row_offset = 0;
#define CRAG_KNN_SELECT_BODY
#include "knn_select.cuh"
#undef CRAG_KNN_SELECT_BODY
}

}  // namespace
}  // namespace crag
#endif
