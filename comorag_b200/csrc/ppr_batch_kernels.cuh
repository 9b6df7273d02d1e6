// Multi-source Personalized PageRank: the kernels of crag_ppr_batch (ppr.cu).  W reset vectors (W in {2, 4, 8, 16,
// 32}, the batch padded to the next width) iterate together, each column exactly as crag_ppr iterates it alone:
//     y_0 = (1 - d) V,   y_{t+1} = (1 - d) V + d A y_t,   x_b = y_T[:, b] / sum(y_T[:, b])
// with y and V stored vertex-major, [n][W]: one pass over the CSR per iteration serves all W columns, and the gather
// of a neighbour fetches its W contiguous floats (one 128-byte line at W = 32).
//
// Column b of the output is bit-identical to crag_ppr run on reset b alone.  The kernels reuse the single-source
// plan (ppr_plan_kernel's merge-path segments of kPprSegItems, chunks of 32 nonzeros from each segment's first
// nonzero) and repeat its arithmetic per column in the same order:
//   ppr_batch_step_kernel   each lane holds one nonzero and forms coef * y_in[col][b] for every column; the same
//                           segmented Hillis-Steele shuffle scan runs per column; a row that spans chunks adds its
//                           chunk partials in chunk order.  The single kernel keeps per-row sums in shared memory
//                           (0 + p1, then + p2, ...); here the row left open at a chunk's end keeps its partial in
//                           s_open and finished rows are written as they complete, which is the same sequence of
//                           additions (0 + p1 = p1 exactly for p1 >= 0).  Head partials and carries as [segment][W];
//   ppr_batch_fixup_kernel  one thread per (head segment, column): carries in segment order, then the head partial;
//   ppr_batch_sum_kernel, ppr_batch_total_kernel   the same grid-stride walk over sum_blocks blocks and the same
//                           256-thread tree (ppr_block_sum), per column; every crag_ppr gather block sums the
//                           partials identically, so one block per column computing the total gives the same bits;
//   ppr_batch_gather_kernel out[b][p] = y[v_p][b] / total_b.
// Products and row updates go through ppr_mul / ppr_row_value, pinned to the contraction ptxas chose for
// ppr_step_kernel and ppr_fixup_kernel (an unfused product; fma(1 - d, reset, d * sum)), so bit-identity does not
// rest on contraction heuristics.  Pure SIMT code like ppr_kernels.cuh: tests/warp_emu runs this header on emulated
// blocks, where the same helpers are the plain expressions of the single kernels.
#pragma once
#include "ppr_kernels.cuh"

namespace crag {
namespace {

constexpr int kPprMaxBatch = 32;
// the step's per-warp shared memory: the row ends of ppr_step_kernel, plus the open row's W partials
constexpr size_t kPprBatchStepSmemBytes = size_t(kPprStepWarps) * (kPprSegItems + kPprMaxBatch) * 4;

inline int ppr_batch_width(int batch) {
  int w = 2;
  while (w < batch) w <<= 1;
  return w;
}

struct PprBatchPlan {
  int64_t segments;                                // as plan_ppr
  int sum_blocks;
  int width;
  float* y[2];                                     // the workspace's regions (null when only sized)
  float* v;
  int32_t *seg_row, *head_row;
  float *head_val, *carry, *partials, *totals;
  size_t total;                                    // workspace bytes
};

// Workspace `ws`: y[2][n][W] fp32, the resets transposed to v[n][W], seg_row and head_row as crag_ppr, head_val and
// carry fp32 [segments][W], partial sums fp32 [sum_blocks][W], totals fp32 [W].
inline PprBatchPlan plan_ppr_batch(int64_t n, int64_t nnz, int batch, void* ws = nullptr) {
  const PprPlan single = plan_ppr(n, nnz);
  PprBatchPlan p;
  p.segments = single.segments;
  p.sum_blocks = single.sum_blocks;
  p.width = ppr_batch_width(batch);
  const size_t W = size_t(p.width);
  WsCursor c(ws);
  p.y[0] = c.take<float>(size_t(n) * W);
  p.y[1] = c.take<float>(size_t(n) * W);
  p.v = c.take<float>(size_t(n) * W);
  p.seg_row = c.take<int32_t>(size_t(p.segments + 1));
  p.head_row = c.take<int32_t>(size_t(p.segments));
  p.head_val = c.take<float>(size_t(p.segments) * W);
  p.carry = c.take<float>(size_t(p.segments) * W);
  p.partials = c.take<float>(size_t(p.sum_blocks) * W);
  p.totals = c.take<float>(W);
  p.total = c.bytes;
  return p;
}

// coef * y, never contracted into the add that follows (ppr_step_kernel: FMUL, then the scan's FADD)
__device__ __forceinline__ float ppr_mul(float a, float b) {
#ifdef CRAG_EMULATED_PTX
  return a * b;
#else
  return __fmul_rn(a, b);
#endif
}

// (1 - d) * reset + d * sum as ppr_step_kernel and ppr_fixup_kernel compute it: FMUL d * sum, FFMA with the reset
__device__ __forceinline__ float ppr_row_value(float omd, float reset, float damping, float sum) {
#ifdef CRAG_EMULATED_PTX
  return omd * reset + damping * sum;
#else
  return __fmaf_rn(omd, reset, __fmul_rn(damping, sum));
#endif
}

// the W floats of one vertex (rows are W * 4 bytes apart from a 256-B aligned base)
template <int W>
__device__ __forceinline__ void ppr_load_row(const float* __restrict__ p, float (&v)[W]) {
#ifdef CRAG_EMULATED_PTX
  for (int b = 0; b < W; ++b) v[b] = p[b];
#else
  if constexpr (W % 4 == 0) {
#pragma unroll
    for (int k = 0; k < W / 4; ++k) {
      const float4 q = reinterpret_cast<const float4*>(p)[k];
      v[4 * k] = q.x, v[4 * k + 1] = q.y, v[4 * k + 2] = q.z, v[4 * k + 3] = q.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < W / 2; ++k) {
      const float2 q = reinterpret_cast<const float2*>(p)[k];
      v[2 * k] = q.x, v[2 * k + 1] = q.y;
    }
  }
#endif
}

// v[i][b] = resets[b][i] for b < batch, 0 for the padding columns; y[i][b] = (1 - d) v[i][b].
template <int W>
__global__ void __launch_bounds__(kPprThreads) ppr_batch_init_kernel(const float* __restrict__ resets, int batch,
                                                                     float damping, int64_t n, float* __restrict__ v,
                                                                     float* __restrict__ y) {
  const int64_t t = int64_t(blockIdx.x) * kPprThreads + threadIdx.x;
  if (t >= n * W) return;
  const int64_t i = t / W;
  const int b = int(t % W);
  const float r = b < batch ? resets[int64_t(b) * n + i] : 0.f;
  v[t] = r;
  y[t] = (1.f - damping) * r;
}

// One warp per segment, as ppr_step_kernel: y_out[i][b] = (1 - d) v[i][b] + d sum_j coef_ij y_in[col_ij][b].
template <int W>
__global__ void __launch_bounds__(kPprStepThreads) ppr_batch_step_kernel(
    const int64_t* __restrict__ row_ptr, const int32_t* __restrict__ col, const float* __restrict__ coef,
    const float* __restrict__ v, float damping, const float* __restrict__ y_in, float* __restrict__ y_out,
    const int32_t* __restrict__ seg_row, const int32_t* __restrict__ head_row, int64_t n, int64_t nnz,
    int64_t segments, float* __restrict__ head_val, float* __restrict__ carry_val) {
  CRAG_DYNAMIC_SHARED(float, s_pprb);
  const int warp = int(threadIdx.x) >> 5, lane = int(threadIdx.x) & 31;
  const int64_t s = int64_t(blockIdx.x) * kPprStepWarps + warp;
  if (s >= segments) return;
  int32_t* s_end = reinterpret_cast<int32_t*>(s_pprb) + warp * kPprSegItems;      // row ends, as ppr_step_kernel
  float* s_open = s_pprb + kPprStepWarps * kPprSegItems + warp * kPprMaxBatch;      // partial of the open row
  const int64_t d0 = s * kPprSegItems, d1 = ppr_min64(d0 + kPprSegItems, n + nnz);
  const int64_t x0 = seg_row[s], x1 = seg_row[s + 1];
  const int64_t y0 = d0 - x0, y1 = d1 - x1;
  const int rows = int(x1 - x0);
  const bool head = head_row[s] >= 0;
  const float omd = 1.f - damping;
  for (int i = lane; i < rows; i += 32) s_end[i] = int32_t(row_ptr[x0 + 1 + i] - y0);
  __syncwarp();
  for (int64_t c = y0; c < y1; c += 32) {
    const int64_t nz = c + lane;
    const bool valid = nz < y1;
    float x[W];
    int key = INT_MAX;
#pragma unroll
    for (int b = 0; b < W; ++b) x[b] = 0.f;
    if (valid) {
      const float a = coef[nz];
      float yv[W];
      ppr_load_row<W>(y_in + int64_t(col[nz]) * W, yv);
#pragma unroll
      for (int b = 0; b < W; ++b) x[b] = ppr_mul(a, yv[b]);
      const int rel = int(nz - y0);
      int lo = 0, hi = rows;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_end[mid] <= rel) lo = mid + 1;
        else hi = mid;
      }
      key = lo;
    }
    // the segmented inclusive scan of ppr_step_kernel, once per column (the keys do not change between columns)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int src = lane >= o ? lane - o : lane;
      const int ks = __shfl_sync(0xffffffffu, key, src);
      const bool take = lane >= o && ks == key;
#pragma unroll
      for (int b = 0; b < W; ++b) {
        const float xs = __shfl_sync(0xffffffffu, x[b], src);
        if (take) x[b] = xs + x[b];
      }
    }
    const int kn = __shfl_sync(0xffffffffu, key, lane < 31 ? lane + 1 : lane);
    const bool run_end = valid && (lane == 31 || kn != key);
    const int rel = int(nz - y0);
    const int row_start = !valid || key == 0 ? 0 : s_end[key - 1];
    const bool finished = run_end && key < rows && s_end[key] == rel + 1;
    // a run that does not start the row continues the partial the previous chunk left open
    const bool continued = run_end && row_start < int(c - y0);
    if (run_end) {
#pragma unroll
      for (int b = 0; b < W; ++b) x[b] = (continued ? s_open[b] : 0.f) + x[b];
    }
    __syncwarp();                                                   // s_open is read before it is overwritten
    if (finished) {
      if (key == 0 && head) {
#pragma unroll
        for (int b = 0; b < W; ++b) head_val[s * W + b] = x[b];
      } else {
        const int64_t r = (x0 + key) * W;
        float vr[W];
        ppr_load_row<W>(v + r, vr);
#pragma unroll
        for (int b = 0; b < W; ++b) y_out[r + b] = ppr_row_value(omd, vr[b], damping, x[b]);
      }
    } else if (run_end) {                                           // the row goes on into the next chunk or segment
#pragma unroll
      for (int b = 0; b < W; ++b) s_open[b] = x[b];
    }
    __syncwarp();
  }
  // rows with no nonzero in this segment: sum 0, as the single kernel's zeroed s_sum
  for (int i = lane; i < rows; i += 32) {
    if (s_end[i] != (i == 0 ? 0 : s_end[i - 1])) continue;
    if (i == 0 && head) {
#pragma unroll
      for (int b = 0; b < W; ++b) head_val[s * W + b] = 0.f;
    } else {
      const int64_t r = (x0 + i) * W;
      float vr[W];
      ppr_load_row<W>(v + r, vr);
#pragma unroll
      for (int b = 0; b < W; ++b) y_out[r + b] = ppr_row_value(omd, vr[b], damping, 0.f);
    }
  }
  // the row still open at the segment's end: its partial, or 0 when it has no nonzero here
  const bool open = (rows == 0 ? 0 : s_end[rows - 1]) < int(y1 - y0);
  if (lane < W) carry_val[s * W + lane] = open ? s_open[lane] : 0.f;
}

// One thread per (segment with a head row r, column b): ppr_fixup_kernel's sum for column b.
template <int W>
__global__ void __launch_bounds__(kPprThreads) ppr_batch_fixup_kernel(const int64_t* __restrict__ row_ptr,
                                                                      const float* __restrict__ v, float damping,
                                                                      const int32_t* __restrict__ head_row,
                                                                      const float* __restrict__ head_val,
                                                                      const float* __restrict__ carry_val,
                                                                      int64_t segments, float* __restrict__ y_out) {
  const int64_t t = int64_t(blockIdx.x) * kPprThreads + threadIdx.x;
  if (t >= segments * W) return;
  const int64_t s = t / W;
  const int b = int(t % W);
  const int32_t r = head_row[s];
  if (r < 0) return;
  const int64_t first = (int64_t(r) + row_ptr[r]) / kPprSegItems;
  float total = carry_val[first * W + b];
#pragma unroll 8
  for (int64_t k = first + 1; k < s; ++k) total += carry_val[k * W + b];
  total += head_val[t];
  y_out[int64_t(r) * W + b] = ppr_row_value(1.f - damping, v[int64_t(r) * W + b], damping, total);
}

// partials[blk][b] = block blk's sum of column b over ppr_sum_kernel's grid-stride walk (gridDim.x = sum_blocks).
template <int W>
__global__ void __launch_bounds__(kPprThreads) ppr_batch_sum_kernel(const float* __restrict__ y, int64_t n,
                                                                    float* __restrict__ partials) {
  CRAG_DYNAMIC_SHARED(float, s_red);
  float acc[W];
#pragma unroll
  for (int b = 0; b < W; ++b) acc[b] = 0.f;
  for (int64_t i = int64_t(blockIdx.x) * kPprThreads + threadIdx.x; i < n; i += int64_t(gridDim.x) * kPprThreads) {
    float row[W];
    ppr_load_row<W>(y + i * W, row);
#pragma unroll
    for (int b = 0; b < W; ++b) acc[b] += row[b];
  }
#pragma unroll
  for (int b = 0; b < W; ++b) {
    const float t = ppr_block_sum(acc[b], s_red);
    if (threadIdx.x == 0) partials[int64_t(blockIdx.x) * W + b] = t;
  }
}

// totals[b]: column b's partials summed as every block of ppr_gather_kernel sums them (one block per column).
template <int W>
__global__ void __launch_bounds__(kPprThreads) ppr_batch_total_kernel(const float* __restrict__ partials,
                                                                      int n_partials, float* __restrict__ totals) {
  CRAG_DYNAMIC_SHARED(float, s_red);
  const int b = int(blockIdx.x);
  float acc = 0.f;
  for (int i = int(threadIdx.x); i < n_partials; i += kPprThreads) acc += partials[int64_t(i) * W + b];
  const float total = ppr_block_sum(acc, s_red);
  if (threadIdx.x == 0) totals[b] = total;
}

// out[b][p] = y[out_vertices[p]][b] / totals[b] for b < batch (out_vertices NULL: p itself); blocks_per_column
// blocks of kPprThreads outputs per column, column-major over the grid.
template <int W>
__global__ void __launch_bounds__(kPprThreads) ppr_batch_gather_kernel(const float* __restrict__ y,
                                                                       const float* __restrict__ totals,
                                                                       const int32_t* __restrict__ out_vertices,
                                                                       int64_t n_out, int64_t blocks_per_column,
                                                                       float* __restrict__ out) {
  const int b = int(blockIdx.x / blocks_per_column);
  const int64_t p = int64_t(blockIdx.x % blocks_per_column) * kPprThreads + threadIdx.x;
  if (p >= n_out) return;
  const int64_t vtx = out_vertices ? out_vertices[p] : p;
  out[int64_t(b) * n_out + p] = y[vtx * W + b] / totals[b];
}

}  // namespace
}  // namespace crag
