// crag_ppr: Personalized PageRank on the device, the solve behind the reference's run_ppr (ComoRAG.py:1086-1105).
// The kernels and the workspace plan live in ppr_kernels.cuh; this file checks the arguments and enqueues
//   plan, init, T x (step, fix-up), sum, gather
// on the caller's stream.  T is fixed by the caller before launch: no convergence test, no host synchronisation.
// crag_ppr_batch runs up to 32 resets through one pass per iteration (ppr_batch_kernels.cuh), each column
// bit-identical to crag_ppr on that reset alone.
#include "common.cuh"
#include "ppr_kernels.cuh"
#include "ppr_batch_kernels.cuh"

using namespace crag;

namespace {
constexpr int64_t kPprMaxRows = (int64_t(1) << 31) - 1;   // col is int32
constexpr int64_t kPprMaxNnz = int64_t(1) << 40;
constexpr int kPprMaxIterations = 1 << 20;

unsigned ppr_blocks(int64_t items, int per_block) { return unsigned((items + per_block - 1) / per_block); }
}  // namespace

extern "C" size_t crag_ppr_workspace_bytes(int64_t n_vertices, int64_t nnz) {
  if (n_vertices < 1 || n_vertices > kPprMaxRows || nnz < 0 || nnz > kPprMaxNnz) return 0;
  return plan_ppr(n_vertices, nnz).total;
}

extern "C" int crag_ppr(const int64_t* row_ptr, const int32_t* col, const float* coef, int64_t n_vertices, int64_t nnz,
                        const float* reset, float damping, int iterations, const int32_t* out_vertices, int64_t n_out,
                        float* out, void* workspace, size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int64_t n = n_vertices;
  if (n < 1 || n > kPprMaxRows) return fail(CRAG_ERR_INVALID, "crag_ppr: n_vertices out of range (%lld)", (long long)n);
  if (nnz < 0 || nnz > kPprMaxNnz) return fail(CRAG_ERR_INVALID, "crag_ppr: nnz out of range (%lld)", (long long)nnz);
  if (!(damping >= 0.f && damping < 1.f)) return fail(CRAG_ERR_INVALID, "crag_ppr: damping must be in [0, 1) (got %g)", double(damping));
  if (iterations < 0 || iterations > kPprMaxIterations)
    return fail(CRAG_ERR_INVALID, "crag_ppr: iterations out of range (%d)", iterations);
  if (n_out < 0 || n_out > kPprMaxNnz || (!out_vertices && n_out != n))
    return fail(CRAG_ERR_INVALID, "crag_ppr: n_out must be >= 0, and equal n_vertices when out_vertices is NULL (%lld)", (long long)n_out);
  if (!row_ptr || !reset || !out || !workspace || (nnz > 0 && (!col || !coef)))
    return fail(CRAG_ERR_INVALID, "crag_ppr: null pointer");
  if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail(CRAG_ERR_INVALID, "crag_ppr: workspace must be 256-byte aligned");
  const PprPlan p = plan_ppr(n, nnz);
  if (workspace_bytes < p.total) return fail(CRAG_ERR_WORKSPACE, "crag_ppr: workspace %zu < %zu bytes", workspace_bytes, p.total);
  if (n_out == 0) return CRAG_OK;

  uint8_t* ws = static_cast<uint8_t*>(workspace);
  float* y[2] = {reinterpret_cast<float*>(ws), reinterpret_cast<float*>(ws + p.y_bytes)};
  int32_t* seg_row = reinterpret_cast<int32_t*>(ws + p.seg_row_off);
  int32_t* head_row = reinterpret_cast<int32_t*>(ws + p.head_row_off);
  float* head_val = reinterpret_cast<float*>(ws + p.head_val_off);
  float* carry = reinterpret_cast<float*>(ws + p.carry_off);
  float* partials = reinterpret_cast<float*>(ws + p.partial_off);

  if (iterations > 0)
    ppr_plan_kernel<<<ppr_blocks(p.segments + 1, kPprThreads), kPprThreads, 0, stream>>>(row_ptr, n, nnz, p.segments,
                                                                                        seg_row, head_row);
  ppr_init_kernel<<<ppr_blocks(n, kPprThreads), kPprThreads, 0, stream>>>(reset, damping, n, y[0]);
  for (int t = 0; t < iterations; ++t) {
    const float* y_in = y[t & 1];
    float* y_out = y[(t + 1) & 1];
    ppr_step_kernel<<<ppr_blocks(p.segments, kPprStepWarps), kPprStepThreads, kPprStepSmemBytes, stream>>>(
        row_ptr, col, coef, reset, damping, y_in, y_out, seg_row, head_row, n, nnz, p.segments, head_val, carry);
    ppr_fixup_kernel<<<ppr_blocks(p.segments, kPprThreads), kPprThreads, 0, stream>>>(row_ptr, reset, damping, head_row,
                                                                                     head_val, carry, p.segments, y_out);
  }
  const float* y_T = y[iterations & 1];
  ppr_sum_kernel<<<p.sum_blocks, kPprThreads, kPprSumSmemBytes, stream>>>(y_T, n, partials);
  ppr_gather_kernel<<<ppr_blocks(n_out, kPprThreads), kPprThreads, kPprSumSmemBytes, stream>>>(
      y_T, partials, p.sum_blocks, out_vertices, n_out, out);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

namespace {
template <int W>
void launch_ppr_batch(const PprBatchPlan& p, const int64_t* row_ptr, const int32_t* col, const float* coef, int64_t n,
                      int64_t nnz, const float* resets, int batch, float damping, int iterations,
                      const int32_t* out_vertices, int64_t n_out, float* out, uint8_t* ws, cudaStream_t stream) {
  float* y[2] = {reinterpret_cast<float*>(ws), reinterpret_cast<float*>(ws + p.y_bytes)};
  float* v = reinterpret_cast<float*>(ws + p.v_off);
  int32_t* seg_row = reinterpret_cast<int32_t*>(ws + p.seg_row_off);
  int32_t* head_row = reinterpret_cast<int32_t*>(ws + p.head_row_off);
  float* head_val = reinterpret_cast<float*>(ws + p.head_val_off);
  float* carry = reinterpret_cast<float*>(ws + p.carry_off);
  float* partials = reinterpret_cast<float*>(ws + p.partial_off);
  float* totals = reinterpret_cast<float*>(ws + p.total_off);

  if (iterations > 0)
    ppr_plan_kernel<<<ppr_blocks(p.segments + 1, kPprThreads), kPprThreads, 0, stream>>>(row_ptr, n, nnz, p.segments,
                                                                                        seg_row, head_row);
  ppr_batch_init_kernel<W><<<ppr_blocks(n * W, kPprThreads), kPprThreads, 0, stream>>>(resets, batch, damping, n, v,
                                                                                       y[0]);
  for (int t = 0; t < iterations; ++t) {
    const float* y_in = y[t & 1];
    float* y_out = y[(t + 1) & 1];
    ppr_batch_step_kernel<W><<<ppr_blocks(p.segments, kPprStepWarps), kPprStepThreads, kPprBatchStepSmemBytes, stream>>>(
        row_ptr, col, coef, v, damping, y_in, y_out, seg_row, head_row, n, nnz, p.segments, head_val, carry);
    ppr_batch_fixup_kernel<W><<<ppr_blocks(p.segments * W, kPprThreads), kPprThreads, 0, stream>>>(
        row_ptr, v, damping, head_row, head_val, carry, p.segments, y_out);
  }
  const float* y_T = y[iterations & 1];
  ppr_batch_sum_kernel<W><<<p.sum_blocks, kPprThreads, kPprSumSmemBytes, stream>>>(y_T, n, partials);
  ppr_batch_total_kernel<W><<<W, kPprThreads, kPprSumSmemBytes, stream>>>(partials, p.sum_blocks, totals);
  const int64_t per_column = ppr_blocks(n_out, kPprThreads);
  ppr_batch_gather_kernel<W><<<unsigned(per_column * batch), kPprThreads, 0, stream>>>(y_T, totals, out_vertices, n_out,
                                                                                      per_column, out);
}
}  // namespace

extern "C" size_t crag_ppr_batch_workspace_bytes(int64_t n_vertices, int64_t nnz, int batch) {
  if (n_vertices < 1 || n_vertices > kPprMaxRows || nnz < 0 || nnz > kPprMaxNnz || batch < 1 || batch > kPprMaxBatch)
    return 0;
  return plan_ppr_batch(n_vertices, nnz, batch).total;
}

extern "C" int crag_ppr_batch(const int64_t* row_ptr, const int32_t* col, const float* coef, int64_t n_vertices,
                              int64_t nnz, const float* resets, int batch, float damping, int iterations,
                              const int32_t* out_vertices, int64_t n_out, float* out, void* workspace,
                              size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int64_t n = n_vertices;
  if (n < 1 || n > kPprMaxRows) return fail(CRAG_ERR_INVALID, "crag_ppr_batch: n_vertices out of range (%lld)", (long long)n);
  if (nnz < 0 || nnz > kPprMaxNnz) return fail(CRAG_ERR_INVALID, "crag_ppr_batch: nnz out of range (%lld)", (long long)nnz);
  if (batch < 1 || batch > kPprMaxBatch)
    return fail(CRAG_ERR_INVALID, "crag_ppr_batch: batch must be in [1, %d] (got %d)", kPprMaxBatch, batch);
  if (!(damping >= 0.f && damping < 1.f))
    return fail(CRAG_ERR_INVALID, "crag_ppr_batch: damping must be in [0, 1) (got %g)", double(damping));
  if (iterations < 0 || iterations > kPprMaxIterations)
    return fail(CRAG_ERR_INVALID, "crag_ppr_batch: iterations out of range (%d)", iterations);
  if (n_out < 0 || n_out > kPprMaxNnz || (!out_vertices && n_out != n))
    return fail(CRAG_ERR_INVALID, "crag_ppr_batch: n_out must be >= 0, and equal n_vertices when out_vertices is NULL (%lld)", (long long)n_out);
  if (!row_ptr || !resets || !out || !workspace || (nnz > 0 && (!col || !coef)))
    return fail(CRAG_ERR_INVALID, "crag_ppr_batch: null pointer");
  if (reinterpret_cast<uintptr_t>(workspace) & 255)
    return fail(CRAG_ERR_INVALID, "crag_ppr_batch: workspace must be 256-byte aligned");
  const PprBatchPlan p = plan_ppr_batch(n, nnz, batch);
  if (workspace_bytes < p.total)
    return fail(CRAG_ERR_WORKSPACE, "crag_ppr_batch: workspace %zu < %zu bytes", workspace_bytes, p.total);
  if (n_out == 0) return CRAG_OK;

  uint8_t* ws = static_cast<uint8_t*>(workspace);
  switch (p.width) {
    case 2: launch_ppr_batch<2>(p, row_ptr, col, coef, n, nnz, resets, batch, damping, iterations, out_vertices, n_out, out, ws, stream); break;
    case 4: launch_ppr_batch<4>(p, row_ptr, col, coef, n, nnz, resets, batch, damping, iterations, out_vertices, n_out, out, ws, stream); break;
    case 8: launch_ppr_batch<8>(p, row_ptr, col, coef, n, nnz, resets, batch, damping, iterations, out_vertices, n_out, out, ws, stream); break;
    case 16: launch_ppr_batch<16>(p, row_ptr, col, coef, n, nnz, resets, batch, damping, iterations, out_vertices, n_out, out, ws, stream); break;
    default: launch_ppr_batch<32>(p, row_ptr, col, coef, n, nnz, resets, batch, damping, iterations, out_vertices, n_out, out, ws, stream); break;
  }
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}
