// Threshold join over a row of fp32 scores: the select half of crag_knn_threshold (search.cu), which first writes the
// same [q_chunk, ld] score block as crag_knn_topk (gemm_scores_f32).  For query q it returns what the synonymy-edge
// walk of the reference's add_synonymy_edges (ComoRAG.py:689-712) reads from crag_knn_topk(k = limit)'s list L:
//   walk L in make_key order (score descending, then row ascending; -0.0 below +0.0), stop at the first entry with
//   !(score >= threshold) (fp32 compare), skip self_rows[q] and every row of exclude_rows, accept the others until
//   `cap` are accepted.
// Rows with score >= threshold form a prefix of that order (a positive NaN ranks above +inf and stops the walk at
// once), so with c = #{score >= threshold} and m = #{skipped rows with score >= threshold, each counted once} the
// answer is decided by the first k_sel = min(limit, c, cap + m) keys.  cap + n_exclude + 1 <= 2048 keeps k_sel within
// the 2048 keys the select sorts in shared memory, for any limit.
//
// One CTA per query row:
//   1. one pass in row order: c, and the keys of the rows >= threshold at s_keys[0, min(c, 2048)) (block scan);
//   2. m from the <= 65 skipped rows (one warp);
//   3. c <= 2048: bitonic sort of the c gathered keys.  c > 2048 (dense near-duplicate clusters): knn_select_kernel's
//      radix select and tie-quota gather (as device functions below) of the exact top k_sel, then the same sort;
//   4. walk the first k_sel keys, compact the accepted ones with a block-wide exclusive scan.
// Columns [n_rows, ld) of the score block are never taken as rows.  Outputs per query: count in [0, cap], then ids
// (local rows) / scores [cap] with -1 / -inf past count.
// Pure SIMT code, so tests/warp_emu runs this very header on emulated blocks.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#include "knn_select.cuh"

namespace crag {
namespace {

constexpr int kKnnMaxExclude = 64;

// Phases 1 and 2 of knn_select_kernel (knn_select.cuh) as device functions: the exact top k of a row when the threshold
// admits more than 2048 rows.  knn_select_kernel keeps its own text of them: called from it, these functions reorder
// a few of its register moves, and its SASS stays byte-identical to the kernel that was measured and pinned.
// ---- 1. radix select over rows [0, n_rows) of row4 (k < n_rows): prefix = the k-th best score word T, quota = how
// many of the k kept rows score exactly T, n_eq = how many rows score exactly T (>= quota).
struct KnnCut {
  uint32_t prefix;
  int quota, n_eq;
};
__device__ __forceinline__ KnnCut knn_radix_select(const float4* row4, int n4, int n_rows, int k, int tid, uint32_t* s_hist,
                                                   int* s_warp, int* s_sel) {
  uint32_t prefix = 0;
  int quota = k;
  int n_eq = 0;
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
  return {prefix, quota, n_eq};
}

// ---- 2. gather in row order: every row above T (every row with take_all) at unordered slots from s_keys[0], and
// with ordered_ties the first `quota` rows equal to T at s_keys[c_above ..]; (mn, mx) = this thread's orderable
// (min, max) over the rows it read.
__device__ __forceinline__ void knn_gather(const float4* row4, int n4, int n_rows, int tid, bool take_all, uint32_t T,
                                           bool ordered_ties, int quota, int c_above, uint64_t* s_keys, int* s_warp,
                                           int& s_slot, uint32_t& mn, uint32_t& mx) {
  if (tid == 0) s_slot = 0;
  __syncthreads();
  mn = 0xFFFFFFFFu;
  mx = 0u;
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
}

__device__ __forceinline__ bool positive_nan(float s) { return s != s && (__float_as_uint(s) >> 31) == 0u; }

// scores: fp32 rows of `ld` floats (ld % 4 == 0, 16-byte aligned), block q reads row q.  self_rows [gridDim.x] (may
// be null), exclude_rows [n_exclude]; outputs out_count [gridDim.x], out_ids / out_scores [gridDim.x, cap].
__global__ void __launch_bounds__(kKnnThreads)
knn_threshold_kernel(const float* __restrict__ scores, int64_t ld, int n_rows, float threshold, int limit, int cap,
                     const int64_t* __restrict__ self_rows, const int64_t* __restrict__ exclude_rows, int n_exclude,
                     int* __restrict__ out_count, int64_t* __restrict__ out_ids, float* __restrict__ out_scores) {
  __shared__ uint32_t s_hist[kKnnBins];
  __shared__ uint64_t s_keys[kKnnMaxK];
  __shared__ int64_t s_skip[kKnnMaxExclude + 1];   // self row, then the excluded rows
  __shared__ int s_warp[kKnnWarps];
  __shared__ int s_sel[3];
  __shared__ int s_slot;
  __shared__ int s_m;
  __shared__ int s_nan;
  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = scores + int64_t(q) * ld;
  const float4* row4 = reinterpret_cast<const float4*>(row);
  const int n4 = (n_rows + 3) >> 2;
  const int n_skip = n_exclude + 1;
  if (tid < n_skip) s_skip[tid] = tid == 0 ? (self_rows ? self_rows[q] : -1) : exclude_rows[tid - 1];
  if (tid == 0) s_nan = 0;
  __syncthreads();

  // ---- 1. c and the keys of the rows >= threshold, in row order
  int c = 0;   // block-uniform
  for (int base = 0; base < n4; base += kKnnThreads) {
    const int i = base + tid;
    float e[4] = {0.f, 0.f, 0.f, 0.f};
    if (i < n4) {
      const float4 v = row4[i];
      e[0] = v.x; e[1] = v.y; e[2] = v.z; e[3] = v.w;
    }
    bool hit[4];
    int n_hit = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool live = i < n4 && 4 * i + j < n_rows;
      hit[j] = live && e[j] >= threshold;
      if (live && positive_nan(e[j])) s_nan = 1;
      n_hit += hit[j] ? 1 : 0;
    }
    int total = 0;
    int slot = knn_block_exclusive_scan(n_hit, s_warp, &total) + c;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (hit[j]) {
        if (slot < kKnnMaxK) s_keys[slot] = make_key(e[j], uint32_t(4 * i + j));
        ++slot;
      }
    }
    c += total;
  }

  // ---- 2. m: the skipped rows that score >= threshold, a row listed twice counted once
  __syncthreads();
  if (warp == 0) {
    int m = 0;
    for (int j = lane; j < n_skip; j += 32) {
      const int64_t r = s_skip[j];
      bool first = r >= 0 && r < n_rows;
      for (int i = 0; i < j; ++i) first = first && s_skip[i] != r;
      if (first && row[r] >= threshold) ++m;
    }
    m = __reduce_add_sync(0xffffffffu, m);
    if (lane == 0) s_m = m;
  }
  __syncthreads();
  int k_sel = limit < c ? limit : c;
  k_sel = k_sel < cap + s_m ? k_sel : cap + s_m;
  if (s_nan) k_sel = 0;   // a positive NaN is L's first entry: the walk stops there

  // ---- 3. the first k_sel keys in order at s_keys[0, k_sel)
  if (c > kKnnMaxK && k_sel > 0) {   // the buffer overflowed: select the exact top k_sel of the whole row
    const KnnCut cut = knn_radix_select(row4, n4, n_rows, k_sel, tid, s_hist, s_warp, s_sel);
    const bool ordered_ties = cut.quota < cut.n_eq;
    uint32_t mn, mx;
    knn_gather(row4, n4, n_rows, tid, false, cut.prefix, ordered_ties, cut.quota, ordered_ties ? k_sel - cut.quota : k_sel,
               s_keys, s_warp, s_slot, mn, mx);
  }
  knn_bitonic_sort(s_keys, c > kKnnMaxK ? k_sel : c, tid);

  // ---- 4. walk: thread t owns positions 4t .. 4t + 3; skipped rows are passed over, the others ranked by a scan
  uint64_t key[4];
  bool take[4];
  int n_take = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int p = 4 * tid + j;
    key[j] = p < k_sel ? s_keys[p] : 0ull;
    take[j] = p < k_sel;
    if (take[j]) {
      const int64_t r = int64_t(key_id(key[j]));
      for (int x = 0; x < n_skip; ++x) take[j] = take[j] && s_skip[x] != r;
    }
    n_take += take[j] ? 1 : 0;
  }
  int total = 0;
  int r = knn_block_exclusive_scan(n_take, s_warp, &total);
  const int count = total < cap ? total : cap;
  int64_t* oi = out_ids + int64_t(q) * cap;
  float* os = out_scores + int64_t(q) * cap;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (take[j]) {
      if (r < cap) {
        oi[r] = int64_t(key_id(key[j]));
        os[r] = key_score(key[j]);
      }
      ++r;
    }
  }
  for (int j = count + tid; j < cap; j += kKnnThreads) {
    oi[j] = -1;
    os[j] = -INFINITY;
  }
  if (tid == 0) out_count[q] = count;
}

}  // namespace
}  // namespace crag
