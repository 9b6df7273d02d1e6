// Personalized PageRank by power iteration on a CSR graph: the kernels of crag_ppr (ppr.cu), which replaces the
// prpack solve of the reference's run_ppr (ComoRAG.py:1086-1105).  DESIGN.md section 2a derives the iteration
//     y_0 = (1 - d) v,   y_{t+1} = (1 - d) v + d A y_t,   x = y_T / sum(y_T)
// with A[i][j] = coef_ij = W_ij / s_j stored in "pull" form: row i lists every neighbour j once, ascending.
//
// Load balance is merge-path: the rows and the nonzeros are merged into one list of n + nnz items (a row's end item
// follows its last nonzero) and cut into segments of kPprSegItems items, one warp per segment, so a hub row with 10^6
// neighbours is spread over thousands of warps.  Per iteration:
//   ppr_step_kernel   each warp loads 32 consecutive (col, coef) pairs at a time, gathers y_in[col], and reduces
//                     each row's products inside the warp with a fixed segmented shuffle scan; the rows the segment
//                     finishes are written, except a row that began in an earlier segment (its "head"), whose
//                     partial goes to head_val; the partial of the row still open at the segment's end to carry_val;
//   ppr_fixup_kernel  one thread per head: the row's carries from the segments before, added in segment order,
//                     plus its head partial.
// Finalize: ppr_sum_kernel (fixed-shape tree of partial sums over all n entries), then ppr_gather_kernel
// (out[p] = y[out_vertices[p]] / total).  No floating-point atomics: the same inputs give the same bits on any run
// and stream.  Pure SIMT code with no wgmma / TMA / mbarrier in it, so tests/warp_emu runs this very header on
// emulated blocks.
#pragma once
#include <limits.h>
#include <stdint.h>
#include <cuda_runtime.h>

#include "workspace.cuh"

#ifndef CRAG_EMULATED_PTX   // tests/warp_emu gives every emulated block its own dynamic shared memory
#define CRAG_DYNAMIC_SHARED(type, name) extern __shared__ type name[]
#endif

namespace crag {
namespace {

constexpr int kPprSegItems = 512;                  // merge-path items (rows + nonzeros) per warp segment
constexpr int kPprStepWarps = 4;
constexpr int kPprStepThreads = 32 * kPprStepWarps;
constexpr int kPprThreads = 256;                   // plan, init, fix-up and finalize blocks
constexpr int kPprMaxSumBlocks = 1024;             // partial sums of the finalize
// dynamic shared memory: the step kernel's per-warp row ends and row sums, the finalize's reduction tree
constexpr size_t kPprStepSmemBytes = size_t(kPprStepWarps) * (2 * kPprSegItems + 1) * 4;
constexpr size_t kPprSumSmemBytes = size_t(kPprThreads) * 4;

struct PprPlan {
  int64_t segments;                                // ceil((n + nnz) / kPprSegItems)
  int sum_blocks;
  float* y[2];                                     // the workspace's regions (null when only sized)
  int32_t *seg_row, *head_row;
  float *head_val, *carry, *partials;
  size_t total;                                    // workspace bytes
};

// Workspace `ws`: y[2][n] fp32 (double buffer), seg_row int32 [segments + 1], head_row int32, head_val and carry fp32
// [segments], partial sums fp32 [sum_blocks].
inline PprPlan plan_ppr(int64_t n, int64_t nnz, void* ws = nullptr) {
  PprPlan p;
  p.segments = (n + nnz + kPprSegItems - 1) / kPprSegItems;
  const int64_t blocks = (n + kPprThreads - 1) / kPprThreads;
  p.sum_blocks = int(blocks < 1 ? 1 : blocks > kPprMaxSumBlocks ? kPprMaxSumBlocks : blocks);
  WsCursor c(ws);
  p.y[0] = c.take<float>(size_t(n));
  p.y[1] = c.take<float>(size_t(n));
  p.seg_row = c.take<int32_t>(size_t(p.segments + 1));
  p.head_row = c.take<int32_t>(size_t(p.segments));
  p.head_val = c.take<float>(size_t(p.segments));
  p.carry = c.take<float>(size_t(p.segments));
  p.partials = c.take<float>(size_t(p.sum_blocks));
  p.total = c.bytes;
  return p;
}

__device__ __forceinline__ int64_t ppr_min64(int64_t a, int64_t b) { return a < b ? a : b; }
__device__ __forceinline__ int64_t ppr_max64(int64_t a, int64_t b) { return a > b ? a : b; }

// Rows finished before merge-path diagonal d: the largest x with row_ptr[x] <= d - x, i.e. CUB's MergePathSearch of
// the row ends row_ptr[1..n] against the nonzero indices 0..nnz-1.
__device__ __forceinline__ int64_t ppr_path_row(const int64_t* row_ptr, int64_t n, int64_t nnz, int64_t d) {
  int64_t lo = ppr_max64(d - nnz, 0), hi = ppr_min64(d, n);
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (row_ptr[mid + 1] <= d - mid - 1) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// seg_row[s] = rows finished before segment s (s = 0..segments); head_row[s] = the row segment s finishes that an
// earlier segment opened (row_ptr[x0] < y0), or -1.  Depends on the graph only.
__global__ void __launch_bounds__(kPprThreads) ppr_plan_kernel(const int64_t* __restrict__ row_ptr, int64_t n,
                                                               int64_t nnz, int64_t segments, int32_t* __restrict__ seg_row,
                                                               int32_t* __restrict__ head_row) {
  const int64_t s = int64_t(blockIdx.x) * kPprThreads + threadIdx.x;
  if (s > segments) return;
  const int64_t d0 = ppr_min64(s * kPprSegItems, n + nnz);
  const int64_t x0 = ppr_path_row(row_ptr, n, nnz, d0);
  seg_row[s] = int32_t(x0);
  if (s == segments) return;
  const int64_t x1 = ppr_path_row(row_ptr, n, nnz, ppr_min64(d0 + kPprSegItems, n + nnz));
  head_row[s] = (x1 > x0 && row_ptr[x0] < d0 - x0) ? int32_t(x0) : -1;
}

__global__ void __launch_bounds__(kPprThreads) ppr_init_kernel(const float* __restrict__ reset, float damping, int64_t n,
                                                               float* __restrict__ y) {
  const int64_t i = int64_t(blockIdx.x) * kPprThreads + threadIdx.x;
  if (i < n) y[i] = (1.f - damping) * reset[i];
}

// One warp per segment: y_out[i] = (1 - d) * reset[i] + d * sum_j coef_ij * y_in[col_ij] for the rows it finishes.
__global__ void __launch_bounds__(kPprStepThreads) ppr_step_kernel(
    const int64_t* __restrict__ row_ptr, const int32_t* __restrict__ col, const float* __restrict__ coef,
    const float* __restrict__ reset, float damping, const float* __restrict__ y_in, float* __restrict__ y_out,
    const int32_t* __restrict__ seg_row, const int32_t* __restrict__ head_row, int64_t n, int64_t nnz,
    int64_t segments, float* __restrict__ head_val, float* __restrict__ carry_val) {
  CRAG_DYNAMIC_SHARED(float, s_ppr);
  const int warp = int(threadIdx.x) >> 5, lane = int(threadIdx.x) & 31;
  const int64_t s = int64_t(blockIdx.x) * kPprStepWarps + warp;
  if (s >= segments) return;
  // row ends, relative to the segment's first nonzero; per-row partial sums (the last one: the row left open)
  int32_t* s_end = reinterpret_cast<int32_t*>(s_ppr) + warp * kPprSegItems;
  float* s_sum = s_ppr + kPprStepWarps * kPprSegItems + warp * (kPprSegItems + 1);
  const int64_t d0 = s * kPprSegItems, d1 = ppr_min64(d0 + kPprSegItems, n + nnz);
  const int64_t x0 = seg_row[s], x1 = seg_row[s + 1];
  const int64_t y0 = d0 - x0, y1 = d1 - x1;
  const int rows = int(x1 - x0);                                  // rows this segment finishes
  for (int i = lane; i < rows; i += 32) s_end[i] = int32_t(row_ptr[x0 + 1 + i] - y0);
  for (int i = lane; i <= rows; i += 32) s_sum[i] = 0.f;
  __syncwarp();
  for (int64_t c = y0; c < y1; c += 32) {
    const int64_t nz = c + lane;
    const bool valid = nz < y1;
    float x = 0.f;
    int key = INT_MAX;                                            // local row; lanes past the segment form their own run
    if (valid) {
      x = coef[nz] * y_in[col[nz]];
      const int rel = int(nz - y0);
      int lo = 0, hi = rows;                                      // local row = number of row ends <= rel
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_end[mid] <= rel) lo = mid + 1;
        else hi = mid;
      }
      key = lo;
    }
    // segmented inclusive scan over the lanes (Hillis-Steele, runs of equal key are contiguous)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int src = lane >= o ? lane - o : lane;
      const float xs = __shfl_sync(0xffffffffu, x, src);
      const int ks = __shfl_sync(0xffffffffu, key, src);
      if (lane >= o && ks == key) x = xs + x;
    }
    const int kn = __shfl_sync(0xffffffffu, key, lane < 31 ? lane + 1 : lane);
    if (valid && (lane == 31 || kn != key)) s_sum[key] += x;     // the last lane of each run: one writer per row
    __syncwarp();
  }
  const bool head = head_row[s] >= 0;
  const float omd = 1.f - damping;
  for (int i = lane; i < rows; i += 32) {
    if (i == 0 && head) head_val[s] = s_sum[0];
    else y_out[x0 + i] = omd * reset[x0 + i] + damping * s_sum[i];
  }
  if (lane == 0) carry_val[s] = s_sum[rows];
}

// One thread per segment with a head row r: the row's first nonzero lies in segment `first`, and every segment from
// there to s - 1 ended with r open.  Their carries are added in segment order, then the head partial.
__global__ void __launch_bounds__(kPprThreads) ppr_fixup_kernel(const int64_t* __restrict__ row_ptr,
                                                                const float* __restrict__ reset, float damping,
                                                                const int32_t* __restrict__ head_row,
                                                                const float* __restrict__ head_val,
                                                                const float* __restrict__ carry_val, int64_t segments,
                                                                float* __restrict__ y_out) {
  const int64_t s = int64_t(blockIdx.x) * kPprThreads + threadIdx.x;
  if (s >= segments) return;
  const int32_t r = head_row[s];
  if (r < 0) return;
  const int64_t first = (int64_t(r) + row_ptr[r]) / kPprSegItems;
  float total = carry_val[first];
#pragma unroll 8
  for (int64_t k = first + 1; k < s; ++k) total += carry_val[k];
  total += head_val[s];
  y_out[r] = (1.f - damping) * reset[r] + damping * total;
}

// Fixed pairwise tree over the kPprThreads threads of the block; every thread gets the total.
__device__ __forceinline__ float ppr_block_sum(float v, float* s_red) {
  s_red[threadIdx.x] = v;
  __syncthreads();
  for (int w = kPprThreads / 2; w > 0; w >>= 1) {
    if (int(threadIdx.x) < w) s_red[threadIdx.x] = s_red[threadIdx.x] + s_red[threadIdx.x + w];
    __syncthreads();
  }
  const float total = s_red[0];
  __syncthreads();
  return total;
}

// partials[b] = block b's sum of y over the grid-stride walk (gridDim.x = PprPlan::sum_blocks).
__global__ void __launch_bounds__(kPprThreads) ppr_sum_kernel(const float* __restrict__ y, int64_t n,
                                                              float* __restrict__ partials) {
  CRAG_DYNAMIC_SHARED(float, s_red);
  float acc = 0.f;
  for (int64_t i = int64_t(blockIdx.x) * kPprThreads + threadIdx.x; i < n; i += int64_t(gridDim.x) * kPprThreads)
    acc += y[i];
  const float t = ppr_block_sum(acc, s_red);
  if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

// out[p] = y[out_vertices[p]] / sum(y) (out_vertices NULL: p itself).  Every block sums the partials the same way.
__global__ void __launch_bounds__(kPprThreads) ppr_gather_kernel(const float* __restrict__ y,
                                                                 const float* __restrict__ partials, int n_partials,
                                                                 const int32_t* __restrict__ out_vertices, int64_t n_out,
                                                                 float* __restrict__ out) {
  CRAG_DYNAMIC_SHARED(float, s_red);
  float acc = 0.f;
  for (int i = int(threadIdx.x); i < n_partials; i += kPprThreads) acc += partials[i];
  const int64_t p = int64_t(blockIdx.x) * kPprThreads + threadIdx.x;
  const float total = ppr_block_sum(acc, s_red);
  if (p < n_out) out[p] = y[out_vertices ? out_vertices[p] : p] / total;
}

}  // namespace
}  // namespace crag
