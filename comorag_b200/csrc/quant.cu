// Int8 and one-bit corpus shards: C entries of the quantiser, the binariser and the exact bf16 rescore
// (quant_kernels.cuh).  The int8 scan
// between them, crag_search_topk_i8, is the I8 variant of the shard scan in search.cu.  The int8 IVF search
// (crag_ivf_search_i8, search.cu) launches its rescore through launch_ivf_rescore here, so that the rescore kernels
// have one translation unit.
#include "common.cuh"
#include "quant_kernels.cuh"

namespace crag {

// The rows may be device memory or page-locked host memory reached through unified addressing.  A kernel that
// dereferences pageable host memory faults, so anything else is refused here, before a launch.
int device_readable(const void* p, const void** out, const char* who) {
  cudaPointerAttributes attr;
  const cudaError_t e = cudaPointerGetAttributes(&attr, p);
  if (e != cudaSuccess) {
    cudaGetLastError();   // the failed query must not surface at the caller's next cudaGetLastError
    return fail(CRAG_ERR_INVALID, "%s: rows are not memory the device can read (%s)", who, cudaGetErrorString(e));
  }
  if (attr.type == cudaMemoryTypeHost) {
    if (!attr.devicePointer) return fail(CRAG_ERR_INVALID, "%s: page-locked rows are not mapped into the device's address space", who);
    *out = attr.devicePointer;
  } else if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged) {
    return fail(CRAG_ERR_INVALID, "%s: rows must be device memory or page-locked host memory (pageable host memory given)", who);
  } else {
    *out = p;
  }
  return CRAG_OK;
}

int launch_ivf_rescore(const void* rows, int64_t n_rows, int dim, int64_t row_stride, const void* queries, int nq,
                       const int64_t* cand, int n_cand, int k, const int32_t* list_tile_start, int nlist,
                       const float* coarse, int64_t* out_ids, float* out_scores, cudaStream_t stream) {
  const IvfListTerm lists{list_tile_start, nlist, coarse};
  const uint16_t* r = static_cast<const uint16_t*>(rows);
  const uint16_t* qb = static_cast<const uint16_t*>(queries);
  if (n_cand <= kRescoreMaxCand)   // one warp sorts the keys in registers
    ivf_rescore_topk_kernel<<<nq, kRescoreThreads, 0, stream>>>(r, n_rows, dim, row_stride, qb, cand, n_cand, k, out_ids, out_scores, lists);
  else                             // a block sorts them in shared memory (crag_ivf_search_i8_wide / _pq_wide)
    ivf_rescore_wide_kernel<<<nq, kKnnThreads, 0, stream>>>(r, n_rows, dim, row_stride, qb, cand, n_cand, k, out_ids, out_scores, lists);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

}  // namespace crag

using namespace crag;

extern "C" int crag_quantize_rows_i8(const void* rows_bf16, int64_t n_rows, int dim, int64_t row_stride, void* out_i8,
                                     int64_t out_stride, float* out_scales, crag_stream_t stream) {
  if (dim < 1 || dim > 1024) return fail(CRAG_ERR_INVALID, "quantize_i8: dim must be in [1, 1024] (dim=%d)", dim);
  const int dim8 = (dim + 127) / 128 * 128;
  if (n_rows < 0 || n_rows >= (int64_t(1) << 31)) return fail(CRAG_ERR_INVALID, "quantize_i8: n_rows out of range (%lld)", (long long)n_rows);
  if (row_stride < dim) return fail(CRAG_ERR_INVALID, "quantize_i8: row_stride must be >= dim");
  if (out_stride < dim8 || out_stride % 16 != 0) return fail(CRAG_ERR_INVALID, "quantize_i8: out_stride must be >= %d and a multiple of 16", dim8);
  if (n_rows == 0) return CRAG_OK;
  if (!rows_bf16 || !out_i8 || !out_scales) return fail(CRAG_ERR_INVALID, "quantize_i8: null pointer");
  if ((reinterpret_cast<uintptr_t>(rows_bf16) & 1) || (reinterpret_cast<uintptr_t>(out_i8) & 15)) return fail(CRAG_ERR_INVALID, "quantize_i8: rows must be 2-byte and out 16-byte aligned");
  const int64_t grid = (n_rows + kQuantThreads / 32 - 1) / (kQuantThreads / 32);
  quantize_rows_kernel<<<unsigned(grid), kQuantThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(rows_bf16), n_rows, dim, row_stride, dim8, static_cast<int8_t*>(out_i8), out_stride, out_scales);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

extern "C" int crag_binarize_rows(const void* rows_bf16, int64_t n_rows, int dim, int64_t row_stride, void* out_bits,
                                  int64_t out_stride, float* out_alpha, crag_stream_t stream) {
  if (dim < 1 || dim > 1024) return fail(CRAG_ERR_INVALID, "binarize: dim must be in [1, 1024] (dim=%d)", dim);
  const int dim8 = (dim + 127) / 128 * 128;
  if (n_rows < 0 || n_rows >= (int64_t(1) << 31)) return fail(CRAG_ERR_INVALID, "binarize: n_rows out of range (%lld)", (long long)n_rows);
  if (row_stride < dim) return fail(CRAG_ERR_INVALID, "binarize: row_stride must be >= dim");
  if (out_stride < dim8 / 8 || out_stride % 16 != 0) return fail(CRAG_ERR_INVALID, "binarize: out_stride must be >= %d bytes and a multiple of 16", dim8 / 8);
  if (n_rows == 0) return CRAG_OK;
  if (!rows_bf16 || !out_bits || !out_alpha) return fail(CRAG_ERR_INVALID, "binarize: null rows, out_bits or out_alpha pointer");
  if ((reinterpret_cast<uintptr_t>(rows_bf16) & 1) || (reinterpret_cast<uintptr_t>(out_bits) & 15)) return fail(CRAG_ERR_INVALID, "binarize: rows must be 2-byte and out_bits 16-byte aligned");
  const int64_t grid = (n_rows + kBinarizeThreads / 32 - 1) / (kBinarizeThreads / 32);
  binarize_rows_kernel<<<unsigned(grid), kBinarizeThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(rows_bf16), n_rows, dim, row_stride, dim8, static_cast<uint8_t*>(out_bits), out_stride, out_alpha);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

extern "C" int crag_rescore_topk(const void* rows_bf16, int64_t n_rows, int dim, int64_t row_stride, int64_t row_offset,
                                 const void* queries_bf16, int nq, const int64_t* cand_ids, int n_cand, int k,
                                 int64_t* out_ids, float* out_scores, crag_stream_t stream) {
  if (nq < 1 || n_cand < 1 || n_cand > kKnnMaxK || k < 1 || k > n_cand) return fail(CRAG_ERR_INVALID, "rescore: need nq >= 1 and 1 <= k <= n_cand <= %d (nq=%d n_cand=%d k=%d)", kKnnMaxK, nq, n_cand, k);
  if (dim < 8 || dim > 1024 || dim % 8 != 0) return fail(CRAG_ERR_INVALID, "rescore: dim must be a multiple of 8 in [8, 1024] (dim=%d)", dim);
  if (n_rows < 0 || n_rows >= (int64_t(1) << 31) || row_offset < 0) return fail(CRAG_ERR_INVALID, "rescore: need 0 <= n_rows < 2^31 and row_offset >= 0");
  if (row_stride < dim || row_stride % 8 != 0) return fail(CRAG_ERR_INVALID, "rescore: row_stride must be >= dim and a multiple of 8");
  if (!queries_bf16 || !cand_ids || !out_ids || !out_scores || (n_rows > 0 && !rows_bf16)) return fail(CRAG_ERR_INVALID, "rescore: null pointer");
  if ((reinterpret_cast<uintptr_t>(rows_bf16) | reinterpret_cast<uintptr_t>(queries_bf16)) & 15) return fail(CRAG_ERR_INVALID, "rescore: rows/queries must be 16-byte aligned");
  const void* rows = rows_bf16;
  if (n_rows > 0) {
    const int rc = device_readable(rows_bf16, &rows, "rescore");
    if (rc != CRAG_OK) return rc;
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint16_t* r = static_cast<const uint16_t*>(rows);
  const uint16_t* qb = static_cast<const uint16_t*>(queries_bf16);
  if (n_cand <= kRescoreMaxCand)   // one warp sorts the keys in registers
    rescore_topk_kernel<<<nq, kRescoreThreads, 0, st>>>(r, n_rows, dim, row_stride, row_offset, qb, cand_ids, n_cand, k, out_ids, out_scores);
  else                             // a block sorts them in shared memory
    rescore_wide_kernel<<<nq, kKnnThreads, 0, st>>>(r, n_rows, dim, row_stride, row_offset, qb, cand_ids, n_cand, k, out_ids, out_scores);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}
