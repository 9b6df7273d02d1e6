// Int8 corpus shards: the row / query quantiser and the exact bf16 rescore of the int8 scan's candidates (quant.cu).
// Pure SIMT, so tests/warp_emu can run both kernels on the CPU.  Semantics (oracle/quant_oracle.py, DESIGN.md 3e):
//
//   quantise  a bf16 row x of width dim becomes int8 [dim8 = ceil(dim / 128) * 128], zero padded, and one fp32 scale
//             s = amax / 127 (amax = max |x_i|, division rounded to nearest);  x^_i = clamp(rint(x_i / s), -127, 127)
//             with rint rounding half to even; s = 0 gives a zero row.  Queries are quantised the same way.
//   rescore   each candidate's score is recomputed as the fp32 dot of its bf16 row and the bf16 query in one pinned
//             order: lane l of a warp takes the 16-byte chunks l, l + 32, ...; inside a chunk each product (rounded)
//             is added to the lane's partial (rounded) in element order from 0.f; the partials are combined by an
//             xor-shuffle tree over 16, 8, 4, 2, 1.  The result is the top k of the candidates by (score descending,
//             row ascending), as make_key orders them: up to 128 candidates one warp sorts the keys in registers, up to
//             2048 a block sorts them in shared memory (knn_sort.cuh).
//   binarize  (one-bit shards, crag_search_topk_b1, DESIGN.md 3f) a bf16 row x of width dim becomes dim8 / 8 code bytes,
//             bit j of byte b set iff x_(8 b + j) > 0 (zeros, -0 and the padding columns dim .. dim8 - 1 give 0, read as
//             -1), and alpha = sum |x_i| / dim (division rounded to nearest), the sum taken in the rescore's order
//             below; alpha = 0 for a zero row.
//   IVF       (crag_ivf_search_i8, DESIGN.md 7) the candidates are stored positions p of an IVF shard's padded residual
//             array; p's list l is the one with list_tile_start[l] <= p / 128 < list_tile_start[l + 1], and its score
//             is fadd(dot, coarse[l][q]) with the pass's coarse table (ivf_plan_kernel).
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

#include <type_traits>

#include "knn_sort.cuh"
#include "pool_floor.cuh"   // kNQ, kTileRows
#include "topk.cuh"

namespace crag {

constexpr int kQuantThreads = 256;           // quantiser: one warp per row
constexpr int kQuantClamp = 127;             // int8 codes are symmetric: -127 .. 127
constexpr int kRescoreThreads = 256;         // rescore: one CTA per query, one warp per candidate
constexpr int kRescoreMaxCand = 128;         // candidates per query: one warp sorts them, 4 keys per lane

__device__ __forceinline__ float bf16_bits_to_f32(uint32_t bits16) { return __uint_as_float(bits16 << 16); }

// x^ of one element under scale s (s != 0)
__device__ __forceinline__ int quant_value(float x, float s) {
  int v = __float2int_rn(__fdiv_rn(x, s));
  v = v < -kQuantClamp ? -kQuantClamp : v;
  return v > kQuantClamp ? kQuantClamp : v;
}

// rows: bf16 bits [n_rows, row_stride], dim valid columns.  out: int8 [n_rows, out_stride], dim8 columns written
// (dim8 a multiple of 128, out 4-byte aligned, out_stride a multiple of 4), scales: fp32 [n_rows].
__global__ void __launch_bounds__(kQuantThreads)
quantize_rows_kernel(const uint16_t* __restrict__ rows, int64_t n_rows, int dim, int64_t row_stride, int dim8,
                     int8_t* __restrict__ out, int64_t out_stride, float* __restrict__ scales) {
  const int lane = threadIdx.x & 31;
  const int64_t row = int64_t(blockIdx.x) * (kQuantThreads / 32) + (threadIdx.x >> 5);
  if (row >= n_rows) return;   // warp-uniform
  const uint16_t* x = rows + row * row_stride;
  // |x| as bits: for non-negative finite floats the unsigned order of the bits is the order of the values
  uint32_t amax_bits = 0;
  for (int c = lane; c < dim; c += 32) {
    const uint32_t a = uint32_t(x[c] & 0x7FFFu) << 16;
    amax_bits = a > amax_bits ? a : amax_bits;
  }
  amax_bits = __reduce_max_sync(0xffffffffu, amax_bits);
  const float s = __fdiv_rn(__uint_as_float(amax_bits), 127.f);
  int8_t* o = out + row * out_stride;
  for (int c0 = lane * 4; c0 < dim8; c0 += 128) {
    uint32_t packed = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c0 + e;
      const int v = (c < dim && s != 0.f) ? quant_value(bf16_bits_to_f32(x[c]), s) : 0;
      packed |= uint32_t(uint8_t(int8_t(v))) << (8 * e);
    }
    *reinterpret_cast<uint32_t*>(o + c0) = packed;
  }
  if (lane == 0) scales[row] = s;
}

constexpr int kBinarizeThreads = 256;        // binarize: one warp per row

// rows: bf16 bits [n_rows, row_stride], dim valid columns.  bits: [n_rows, out_stride] bytes, dim8 / 8 written (dim8 a
// multiple of 128, bits 4-byte aligned, out_stride a multiple of 4); alpha: fp32 [n_rows].
__global__ void __launch_bounds__(kBinarizeThreads)
binarize_rows_kernel(const uint16_t* __restrict__ rows, int64_t n_rows, int dim, int64_t row_stride, int dim8,
                     uint8_t* __restrict__ bits, int64_t out_stride, float* __restrict__ alpha) {
  const int lane = threadIdx.x & 31;
  const int64_t row = int64_t(blockIdx.x) * (kBinarizeThreads / 32) + (threadIdx.x >> 5);
  if (row >= n_rows) return;   // warp-uniform
  const uint16_t* x = rows + row * row_stride;
  // sum |x_i|: lane l adds the 8-column chunks l, l + 32, ... in element order, then an xor tree over the lanes
  float abs_sum = 0.f;
  for (int c0 = lane * 8; c0 < dim; c0 += 32 * 8)
    for (int c = c0; c < c0 + 8 && c < dim; ++c) abs_sum = __fadd_rn(abs_sum, bf16_bits_to_f32(x[c] & 0x7FFFu));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) abs_sum = __fadd_rn(abs_sum, __shfl_xor_sync(0xffffffffu, abs_sum, o));
  // code word w: lane j's column 32 w + j in bit j; positive = sign clear and not zero
  uint32_t* out = reinterpret_cast<uint32_t*>(bits + row * out_stride);
  for (int w = 0; w < dim8 / 32; ++w) {
    const int c = 32 * w + lane;
    const uint32_t v = c < dim ? x[c] : 0u;
    const uint32_t word = __ballot_sync(0xffffffffu, v != 0u && v < 0x8000u);
    if (lane == (w & 31)) out[w] = word;
  }
  if (lane == 0) alpha[row] = __fdiv_rn(abs_sum, float(dim));
}

// partial += a_i * b_i over the 8 bf16 of one 16-byte chunk, in element order (the low half of a word comes first)
__device__ __forceinline__ float dot_chunk(float partial, const uint4& a, const uint4& b) {
  const uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    partial = __fadd_rn(partial, __fmul_rn(__uint_as_float(wa[w] << 16), __uint_as_float(wb[w] << 16)));
    partial = __fadd_rn(partial, __fmul_rn(__uint_as_float(wa[w] & 0xFFFF0000u), __uint_as_float(wb[w] & 0xFFFF0000u)));
  }
  return partial;
}

// The flat rescore passes NoListTerm; the IVF rescore passes the list layout and the coarse table of its 32-query pass.
struct NoListTerm {};
struct IvfListTerm {
  const int32_t* list_tile_start;   // [nlist + 1]
  int nlist;
  const float* coarse;              // [nlist][kNQ]: coarse[l * kNQ + q] = q . c_l for the lists query q probes
};

// the list owning stored position p: the largest l with list_tile_start[l] <= p / kTileRows, which skips empty lists
__device__ __forceinline__ int list_of_position(const int32_t* __restrict__ list_tile_start, int nlist, int64_t p) {
  const int32_t tile = int32_t(p / kTileRows);
  int lo = 0, hi = nlist - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&list_tile_start[mid]) <= tile) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// The rescore key of one candidate, by one warp (all lanes return it): make_key(S2, local) for the candidate at local
// row `local` of rows (bf16 [n_rows, row_stride], device or page-locked host memory) against the query qv (bf16 [dim],
// n_chunks = dim / 8, 16-byte aligned), S2 summed in the pinned order; 0 (no candidate) for a local row outside
// [0, n_rows), whose row is never read.  q: the query's index in the coarse table of an IVF pass.
template <class ListTerm>
__device__ __forceinline__ uint64_t rescore_key(const uint16_t* __restrict__ rows, int64_t n_rows, int n_chunks,
                                                int64_t row_stride, const uint16_t* __restrict__ qv, int64_t local,
                                                int q, int lane, const ListTerm& lists) {
  uint64_t key = 0;   // no candidate
  if (local >= 0 && local < n_rows) {   // warp-uniform
    const uint16_t* xr = rows + local * row_stride;
    float partial = 0.f;
#pragma unroll 4
    for (int ch = lane; ch < n_chunks; ch += 32)
      partial = dot_chunk(partial, *reinterpret_cast<const uint4*>(xr + ch * 8), __ldg(reinterpret_cast<const uint4*>(qv + ch * 8)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) partial = __fadd_rn(partial, __shfl_xor_sync(0xffffffffu, partial, o));
    if constexpr (std::is_same<ListTerm, IvfListTerm>::value) {
      const int l = list_of_position(lists.list_tile_start, lists.nlist, local);
      partial = __fadd_rn(partial, __ldg(&lists.coarse[int64_t(l) * kNQ + q]));
    }
    key = make_key(partial, uint32_t(local));
  }
  return key;
}

// The body of both rescore kernels; one CTA per query.  rows: bf16 [n_rows, row_stride] (device or page-locked host
// memory), queries: bf16 [nq, dim] dense, dim a multiple of 8, rows and queries 16-byte aligned.  cand_ids: int64
// [nq, n_cand] global ids; an id outside [row_offset, row_offset + n_rows) -- -1 among them -- is no candidate and its
// row is never read.  Writes the top k (k <= n_cand <= 128) to out_ids / out_scores [nq, k], -1 / -inf past the valid
// candidates.
template <class ListTerm>
__device__ __forceinline__ void rescore_topk_body(const uint16_t* __restrict__ rows, int64_t n_rows, int dim,
                                                  int64_t row_stride, int64_t row_offset,
                                                  const uint16_t* __restrict__ queries,
                                                  const int64_t* __restrict__ cand_ids, int n_cand, int k,
                                                  int64_t* __restrict__ out_ids, float* __restrict__ out_scores,
                                                  const ListTerm& lists) {
  __shared__ uint64_t keys[kRescoreMaxCand];
  const int q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint16_t* qv = queries + int64_t(q) * dim;
  const int n_chunks = dim / 8;
  for (int c = warp; c < kRescoreMaxCand; c += kRescoreThreads / 32) {
    const int64_t local = c < n_cand ? __ldg(&cand_ids[int64_t(q) * n_cand + c]) - row_offset : -1;
    const uint64_t key = rescore_key(rows, n_rows, n_chunks, row_stride, qv, local, q, lane, lists);
    if (lane == 0) keys[c] = key;
  }
  __syncthreads();
  if (warp != 0) return;
  constexpr int EPL = kRescoreMaxCand / 32;
  uint64_t v[EPL];
#pragma unroll
  for (int j = 0; j < EPL; ++j) v[j] = keys[lane * EPL + j];
  warp_sort_desc<EPL>(v, lane);
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const int g = lane * EPL + j;
    if (g < k) {
      out_ids[int64_t(q) * k + g] = v[j] ? int64_t(key_id(v[j])) + row_offset : -1;
      out_scores[int64_t(q) * k + g] = v[j] ? key_score(v[j]) : -INFINITY;
    }
  }
}

// crag_rescore_topk: candidates are global row ids
__global__ void __launch_bounds__(kRescoreThreads)
rescore_topk_kernel(const uint16_t* __restrict__ rows, int64_t n_rows, int dim, int64_t row_stride, int64_t row_offset,
                    const uint16_t* __restrict__ queries, const int64_t* __restrict__ cand_ids, int n_cand, int k,
                    int64_t* __restrict__ out_ids, float* __restrict__ out_scores) {
  rescore_topk_body(rows, n_rows, dim, row_stride, row_offset, queries, cand_ids, n_cand, k, out_ids, out_scores, NoListTerm{});
}

// crag_ivf_search_i8, one 32-query pass: candidates are stored positions of the IVF shard (row_offset 0, n_rows =
// its padded row count), each score gains its list's coarse term; out_ids are positions (ivf_map_ids_kernel follows)
__global__ void __launch_bounds__(kRescoreThreads)
ivf_rescore_topk_kernel(const uint16_t* __restrict__ rows, int64_t n_rows, int dim, int64_t row_stride,
                        const uint16_t* __restrict__ queries, const int64_t* __restrict__ cand_ids, int n_cand, int k,
                        int64_t* __restrict__ out_ids, float* __restrict__ out_scores, const IvfListTerm lists) {
  rescore_topk_body(rows, n_rows, dim, row_stride, int64_t(0), queries, cand_ids, n_cand, k, out_ids, out_scores, lists);
}

// The body of both wide rescore kernels, above 128 candidates (n_cand <= kKnnMaxK): one CTA of kKnnThreads per query,
// one warp per candidate (rescore_key, as rescore_topk_body computes it), the keys in shared memory (16 KB at 2048)
// sorted by knn_bitonic_sort, the top k out; -1 / -inf past the valid candidates.
template <class ListTerm>
__device__ __forceinline__ void rescore_wide_body(const uint16_t* __restrict__ rows, int64_t n_rows, int dim,
                                                  int64_t row_stride, int64_t row_offset,
                                                  const uint16_t* __restrict__ queries,
                                                  const int64_t* __restrict__ cand_ids, int n_cand, int k,
                                                  int64_t* __restrict__ out_ids, float* __restrict__ out_scores,
                                                  const ListTerm& lists) {
  __shared__ uint64_t s_keys[kKnnMaxK];
  const int q = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint16_t* qv = queries + int64_t(q) * dim;
  const int64_t* cand = cand_ids + int64_t(q) * n_cand;
  for (int c = warp; c < n_cand; c += kKnnWarps) {
    const uint64_t key = rescore_key(rows, n_rows, dim / 8, row_stride, qv, __ldg(&cand[c]) - row_offset, q, lane, lists);
    if (lane == 0) s_keys[c] = key;
  }
  knn_bitonic_sort(s_keys, n_cand, tid);
  for (int j = tid; j < k; j += kKnnThreads) {
    const uint64_t key = s_keys[j];
    out_ids[int64_t(q) * k + j] = key ? int64_t(key_id(key)) + row_offset : -1;
    out_scores[int64_t(q) * k + j] = key ? key_score(key) : -INFINITY;
  }
}

// crag_rescore_topk above 128 candidates
__global__ void __launch_bounds__(kKnnThreads)
rescore_wide_kernel(const uint16_t* __restrict__ rows, int64_t n_rows, int dim, int64_t row_stride, int64_t row_offset,
                    const uint16_t* __restrict__ queries, const int64_t* __restrict__ cand_ids, int n_cand, int k,
                    int64_t* __restrict__ out_ids, float* __restrict__ out_scores) {
  rescore_wide_body(rows, n_rows, dim, row_stride, row_offset, queries, cand_ids, n_cand, k, out_ids, out_scores, NoListTerm{});
}

// crag_ivf_search_i8_wide / _pq_wide, one 32-query pass: up to 2048 candidate positions per query, as
// ivf_rescore_topk_kernel scores them
__global__ void __launch_bounds__(kKnnThreads)
ivf_rescore_wide_kernel(const uint16_t* __restrict__ rows, int64_t n_rows, int dim, int64_t row_stride,
                        const uint16_t* __restrict__ queries, const int64_t* __restrict__ cand_ids, int n_cand, int k,
                        int64_t* __restrict__ out_ids, float* __restrict__ out_scores, const IvfListTerm lists) {
  rescore_wide_body(rows, n_rows, dim, row_stride, int64_t(0), queries, cand_ids, n_cand, k, out_ids, out_scores, lists);
}

}  // namespace crag
