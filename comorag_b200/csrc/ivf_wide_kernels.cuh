// The score-all fills of the wide IVF stage 1 (crag_ivf_search_i8_wide / _pq_wide; DESIGN.md section 7): every probed
// row's S1 into its slot of the pass's S1 block, which ivf_wide_select_kernel (knn_select.cuh) then ranks per query.
// They walk the IVF plan's work-list as pq_scan_kernel does: CTA b serves query q = b / slices and the items s, s +
// slices, ... (s = b % slices) of the lists q probes.  Row r of item (pos0, rows, l) goes to slot
// slot_base[l][q] + pos0 - list_tile_start[l] * 128 + r (ivf_wide_plan_kernel), and only below cap.  S1 is bit for bit
// the narrow stage 1's:
//   int8  fadd(fmul(int2float(acc), fmul(s_q, s_p)), coarse[l][q]), acc the exact int32 dot of the two int8 rows
//   PQ    fadd(pq_row_sum(codes of p, table of q), coarse[l][q])
// Pure SIMT, so tests/warp_emu runs both on emulated blocks.  On a clustered share nearly every probed list is probed
// by one query of the pass, so a 32-query wgmma tile would be mostly masked; these kernels score one query per row.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#include "ivf_kernels.cuh"
#include "pq_kernels.cuh"
#include "search_types.cuh"   // IvfArgs

namespace crag {

constexpr int kIvfFillThreads = 128;

// Where the fills write: the S1 block [kNQ][ld] of one pass and the slot layout of the wide plan
struct IvfWideBlock {
  const int32_t* list_tile_start;   // [nlist + 1]
  const int32_t* slot_base;         // [nlist][kNQ] (IvfWidePlan)
  float* block;                     // [kNQ][ld]
  int64_t ld;
  int cap;                          // max_probe_rows <= ld
};

// the slot of row 0 of work item `item` for query q
__device__ __forceinline__ int64_t ivf_item_slot(const int4& item, int q, const IvfWideBlock& out) {
  return int64_t(__ldg(&out.slot_base[int64_t(item.z) * kNQ + q])) + item.x -
         int64_t(__ldg(&out.list_tile_start[item.z])) * kTileRows;
}

// Int8 residuals: one warp per row, lanes on 16-byte chunks of the row (dim8 <= 1024), the int32 sum reduced over the
// warp (exact, so its order is free).  codes [n_rows_padded, code_stride] int8, row_scales [n_rows_padded]; queries
// [nq, dim8] int8 dense and query_scales [nq] of this pass.
__global__ void __launch_bounds__(kIvfFillThreads)
ivf_fill_i8_kernel(const int8_t* __restrict__ codes, int64_t code_stride, int dim8, const float* __restrict__ row_scales,
                   const int8_t* __restrict__ queries, const float* __restrict__ query_scales, int slices,
                   const IvfArgs plan, const IvfWideBlock out) {
  __shared__ uint4 s_q[1024 / 16];
  const int q = int(blockIdx.x / unsigned(slices)), s = int(blockIdx.x % unsigned(slices));
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n16 = dim8 / 16;
  const uint4* qrow = reinterpret_cast<const uint4*>(queries + int64_t(q) * dim8);
  for (int i = threadIdx.x; i < n16; i += kIvfFillThreads) s_q[i] = __ldg(qrow + i);
  __syncthreads();
  const float qs = __ldg(&query_scales[q]);
  const int n_work = __ldg(plan.n_work);
  for (int j = s; j < n_work; j += slices) {
    const int4 item = __ldg(&plan.work[j]);
    if (!((__ldg(&plan.list_mask[item.z]) >> q) & 1u)) continue;
    const int64_t first = ivf_item_slot(item, q, out);
    const float coarse = __ldg(plan.coarse + size_t(item.z) * kNQ + q);
    for (int r = w; r < item.y; r += kIvfFillThreads / 32) {   // warp-uniform
      const int64_t slot = first + r;
      if (slot >= out.cap) break;
      const int64_t pos = int64_t(item.x) + r;
      const uint4* row = reinterpret_cast<const uint4*>(codes + pos * code_stride);
      int acc = 0;
      for (int c = lane; c < n16; c += 32) {
        const uint4 a = __ldg(row + c), b = s_q[c];
        acc = __dp4a(int(a.x), int(b.x), acc);
        acc = __dp4a(int(a.y), int(b.y), acc);
        acc = __dp4a(int(a.z), int(b.z), acc);
        acc = __dp4a(int(a.w), int(b.w), acc);
      }
      acc = __reduce_add_sync(0xffffffffu, acc);
      if (lane == 0) {
        const float scale = __fmul_rn(qs, __ldg(&row_scales[pos]));
        out.block[int64_t(q) * out.ld + slot] = __fadd_rn(__fmul_rn(__int2float_rn(acc), scale), coarse);
      }
    }
  }
}

// PQ codes: the query's table in shared memory (m * 256 * 4 bytes of dynamic shared memory), one thread per row of an
// item.  codes [n_rows_padded, code_stride], lut [nq][m][256] of this pass (pq_table_kernel).
__global__ void __launch_bounds__(kIvfFillThreads)
ivf_fill_pq_kernel(const uint8_t* __restrict__ codes, int64_t code_stride, int m, const float* __restrict__ lut,
                   int slices, const IvfArgs plan, const IvfWideBlock out) {
  CRAG_DYNAMIC_SHARED(float, pq_smem);
  float* table = pq_smem;
  const int q = int(blockIdx.x / unsigned(slices)), s = int(blockIdx.x % unsigned(slices));
  const float4* src = reinterpret_cast<const float4*>(lut + size_t(q) * m * kPqCodewords);
  for (int i = threadIdx.x; i < m * kPqCodewords / 4; i += kIvfFillThreads) reinterpret_cast<float4*>(table)[i] = __ldg(src + i);
  __syncthreads();
  const int r = threadIdx.x;
  const int n_work = __ldg(plan.n_work);
  for (int j = s; j < n_work; j += slices) {
    const int4 item = __ldg(&plan.work[j]);
    if (!((__ldg(&plan.list_mask[item.z]) >> q) & 1u)) continue;
    const int64_t slot = ivf_item_slot(item, q, out) + r;
    if (r < item.y && slot < out.cap) {
      const int64_t pos = int64_t(item.x) + r;
      const float coarse = __ldg(plan.coarse + size_t(item.z) * kNQ + q);
      out.block[int64_t(q) * out.ld + slot] = __fadd_rn(pq_row_sum(codes + pos * code_stride, m, table), coarse);
    }
  }
}

}  // namespace crag
