// IVF over product-quantized residual lists (crag_ivf_search_pq, crag_pq_encode; semantics in DESIGN.md section 7 and
// tests/ivf_pq_oracle.py).  A stored residual r of width dim is cut into m subspaces of dsub = dim / m columns; each
// subspace has a codebook of 256 fp32 codewords and r is stored as m one-byte codes.  For inner product the table of a
// query does not depend on the list, so one table per query serves every probed list:
//   encode   code_j(r) = argmin_c sum_t (r_{j,t} - C_j[c][t])^2          (t order, no FMA, ties to the smaller c)
//   table    LUT_q[j][c] = sum_t q_{j,t} * C_j[c][t]                    (t order, no FMA)
//   stage 1  S1 = fadd(sum_j LUT_q[j][code_j], coarse[q][l])            (j order)
// Pure SIMT kernels, kept in a header so that tests/warp_emu runs them on emulated thread blocks.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

#include "pool_floor.cuh"     // kNQ, kTileRows
#include "search_types.cuh"   // IvfArgs
#include "topk.cuh"

#ifndef CRAG_EMULATED_PTX     // tests/warp_emu gives every emulated block its own dynamic shared memory
#ifndef CRAG_DYNAMIC_SHARED
#define CRAG_DYNAMIC_SHARED(type, name) extern __shared__ __align__(16) type name[]
#endif
#endif

namespace crag {

constexpr int kPqCodewords = 256;
constexpr int kPqMaxM = 192;         // one query's table, m * 256 * 4 bytes, must fit in shared memory
constexpr int kPqMaxDsub = 128;      // one subspace's codebook and a block of its residuals fit in shared memory
constexpr int kPqThreads = 128;      // encode: one row per thread; scan: four warps, one row of a tile per thread
constexpr int kPqTableThreads = 256; // one codeword per thread

__host__ __device__ constexpr int pq_code_stride(int m) { return (m + 15) / 16 * 16; }

__device__ __forceinline__ float pq_bf16(uint16_t bits) { return __uint_as_float(uint32_t(bits) << 16); }

// Dynamic shared memory of pq_encode_kernel: subspace j's codebook [256][dsub], then the block's residuals
// [dsub][kPqThreads + 1] (the pad keeps both the transposing stores and the per-thread loads conflict-free).
__host__ __device__ constexpr size_t pq_encode_smem_bytes(int dsub) {
  return (size_t(kPqCodewords) * dsub + size_t(dsub) * (kPqThreads + 1)) * 4;
}

// One CTA per (block of 128 rows, subspace j): block b covers rows (b / m) * 128 .. + 127 and subspace b % m.  rows:
// bf16 bits [n_rows, row_stride]; codebooks fp32 [m, 256, dsub]; codes [n_rows, code_stride], byte j of row r written.
__global__ void __launch_bounds__(kPqThreads) pq_encode_kernel(const uint16_t* __restrict__ rows, int64_t n_rows, int dim,
                                                               int64_t row_stride, const float* __restrict__ codebooks,
                                                               int m, uint8_t* __restrict__ codes, int64_t code_stride) {
  CRAG_DYNAMIC_SHARED(float, pq_smem);
  const int dsub = dim / m;
  const int j = int(blockIdx.x % unsigned(m));
  const int64_t r0 = int64_t(blockIdx.x / unsigned(m)) * kPqThreads;
  float* cb = pq_smem;
  float* res = pq_smem + kPqCodewords * dsub;
  const float* src = codebooks + size_t(j) * kPqCodewords * dsub;
  for (int i = threadIdx.x; i < kPqCodewords * dsub; i += kPqThreads) cb[i] = __ldg(src + i);
  for (int i = threadIdx.x; i < kPqThreads * dsub; i += kPqThreads) {
    const int rr = i / dsub, t = i - rr * dsub;
    const int64_t row = r0 + rr;
    res[t * (kPqThreads + 1) + rr] = row < n_rows ? pq_bf16(__ldg(rows + row * row_stride + j * dsub + t)) : 0.f;
  }
  __syncthreads();
  const int64_t row = r0 + threadIdx.x;
  if (row >= n_rows) return;
  float best = INFINITY;
  int best_c = 0;
  for (int c = 0; c < kPqCodewords; ++c) {
    const float* w = cb + c * dsub;
    float diff = __fsub_rn(res[threadIdx.x], w[0]);
    float d = __fmul_rn(diff, diff);
    for (int t = 1; t < dsub; ++t) {
      diff = __fsub_rn(res[t * (kPqThreads + 1) + threadIdx.x], w[t]);
      d = __fadd_rn(d, __fmul_rn(diff, diff));
    }
    if (d < best) { best = d; best_c = c; }   // strict: equal distances stay with the smaller codeword
  }
  codes[row * code_stride + j] = uint8_t(best_c);
}

// One CTA per (query q, subspace j) = block q * m + j, thread c: lut[(q * m + j) * 256 + c] = LUT_q[j][c].
// queries: bf16 bits [nq, dim] dense.
__global__ void __launch_bounds__(kPqTableThreads) pq_table_kernel(const uint16_t* __restrict__ queries, int dim,
                                                                   const float* __restrict__ codebooks, int m,
                                                                   float* __restrict__ lut) {
  const int dsub = dim / m;
  const int q = int(blockIdx.x / unsigned(m)), j = int(blockIdx.x % unsigned(m));
  const int c = threadIdx.x;
  const uint16_t* qj = queries + size_t(q) * dim + size_t(j) * dsub;
  const float* w = codebooks + (size_t(j) * kPqCodewords + c) * dsub;
  float acc = __fmul_rn(pq_bf16(__ldg(qj)), __ldg(w));
  for (int t = 1; t < dsub; ++t) acc = __fadd_rn(acc, __fmul_rn(pq_bf16(__ldg(qj + t)), __ldg(w + t)));
  lut[(size_t(q) * m + j) * kPqCodewords + c] = acc;
}

// Dynamic shared memory of pq_scan_kernel: the query's table [m][256] fp32, then four warp selectors and the merged
// one (KLIST + KLIST keys each), their thresholds and the warps' (min, max).
template <int KLIST>
struct PqScanSmem {
  static constexpr int kKeys = 2 * KLIST;
  __host__ __device__ static constexpr size_t bytes(int m) {
    return size_t(m) * kPqCodewords * 4 + 5 * size_t(kKeys) * 8 + 5 * 8 + 4 * 2 * 4;
  }
};

// sum_j table[j][code_j] in j order over one row's codes (16-byte loads; code_stride a multiple of 16)
__device__ __forceinline__ float pq_row_sum(const uint8_t* __restrict__ row_codes, int m, const float* table) {
  float acc = 0.f;
  for (int j0 = 0; j0 < m; j0 += 16) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(row_codes + j0));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      const int j = j0 + b;
      if (j < m) {
        const float x = table[j * kPqCodewords + ((w[b >> 2] >> (8 * (b & 3))) & 0xFFu)];
        acc = j == 0 ? x : __fadd_rn(acc, x);
      }
    }
  }
  return acc;
}

// The PQ scan of one 32-query pass.  CTA b serves query q = b / slices and slice s = b % slices of the plan's
// work-list (items s, s + slices, ...).  It copies the query's table into shared memory, and each warp w scores row
// w * 32 + lane of every tile of its slice that q probes, keeping its top k by (S1 desc, position asc) in a topk.cuh
// selector; warp 0 merges the four lists.  The CTA's list and (min, max) of S1 go to part (s, q) of part_keys
// [slices][kNQ][k] / part_minmax [slices][kNQ][2], which merge_topk_kernel reads as a scan's per-CTA partials.
template <int KLIST>
__global__ void __launch_bounds__(kPqThreads) pq_scan_kernel(const uint8_t* __restrict__ codes, int64_t code_stride,
                                                             int m, const float* __restrict__ lut, int slices, int k,
                                                             IvfArgs plan, uint64_t* __restrict__ part_keys,
                                                             float* __restrict__ part_minmax) {
  constexpr int KPQ = PqScanSmem<KLIST>::kKeys;
  CRAG_DYNAMIC_SHARED(float, pq_smem);
  float* table = pq_smem;
  uint64_t* keys = reinterpret_cast<uint64_t*>(pq_smem + m * kPqCodewords);   // [5][KPQ]
  uint64_t* thr = keys + 5 * KPQ;                                           // [5]
  float* red = reinterpret_cast<float*>(thr + 5);                           // [4][2]
  const int q = int(blockIdx.x / unsigned(slices)), s = int(blockIdx.x % unsigned(slices));
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const float4* src = reinterpret_cast<const float4*>(lut + size_t(q) * m * kPqCodewords);
  for (int i = threadIdx.x; i < m * kPqCodewords / 4; i += kPqThreads) reinterpret_cast<float4*>(table)[i] = __ldg(src + i);
  __syncthreads();

  const int n_work = __ldg(plan.n_work);
  const int items = n_work > s ? (n_work - s + slices - 1) / slices : 0;
  float mn = INFINITY, mx = -INFINITY;
  select_stream<KLIST, KLIST>(keys + w * KPQ, &thr[w], lane, k, items * 32, 0ull, [&](int idx) -> uint64_t {
    const int4 item = __ldg(&plan.work[s + (idx >> 5) * slices]);
    const int r = w * 32 + (idx & 31);
    if (r >= item.y || !((__ldg(&plan.list_mask[item.z]) >> q) & 1u)) return 0ull;
    const int64_t pos = int64_t(item.x) + r;
    const float s1 = __fadd_rn(pq_row_sum(codes + pos * code_stride, m, table), __ldg(plan.coarse + size_t(item.z) * kNQ + q));
    mn = fminf(mn, s1);
    mx = fmaxf(mx, s1);
    return make_key(s1, uint32_t(pos));
  });
  warp_minmax(mn, mx);
  if (lane == 0) { red[w * 2] = mn; red[w * 2 + 1] = mx; }
  __syncthreads();
  if (w != 0) return;
  select_stream<KLIST, KLIST>(keys + 4 * KPQ, &thr[4], lane, k, 4 * k, 0ull,
                              [&](int idx) -> uint64_t { return keys[(idx / k) * KPQ + idx % k]; });
  uint64_t* dst = part_keys + (size_t(s) * kNQ + q) * k;
  for (int j = lane; j < k; j += 32) dst[j] = keys[4 * KPQ + j];
  if (lane == 0) {
    float a = red[0], b = red[1];
    for (int i = 1; i < 4; ++i) { a = fminf(a, red[i * 2]); b = fmaxf(b, red[i * 2 + 1]); }
    part_minmax[(size_t(s) * kNQ + q) * 2] = a;
    part_minmax[(size_t(s) * kNQ + q) * 2 + 1] = b;
  }
}

}  // namespace crag
