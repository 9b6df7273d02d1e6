// Full descending ranking of one query's score array on the device: the
//   sorted_doc_ids = np.argsort(query_doc_scores)[::-1]; sorted_doc_scores = query_doc_scores[sorted_doc_ids]
// step of the reference's dense_passage_retrieval (ComoRAG.py:965-966), whose whole permutation feeds the PPR reset
// weights (ComoRAG.py:1034-1042).  Equal scores rank by ascending row (the engine's deterministic tie rule; numpy's
// argsort[::-1] leaves ties unspecified).
//
// Stable LSD radix sort, 4 passes of 8 bits over key = ~orderable(score) (ascending key == descending score) with
// the row index as payload.  HBM-bound integer work: per pass every element is read twice (histogram, scatter) and
// written once; nothing here is GEMM-shaped.
//   pass p:  hist_kernel    each warp owns a contiguous run of elements and counts its 256 digit bins
//            scan_kernel    block d turns hist[d][*] into exclusive global offsets (digit base + running sum)
//            scatter_kernel each warp replays its run in order, 32 elements a round; equal digits inside a round
//                           are ranked with match.any so the scatter stays stable
// Pass 0 builds the keys from the fp32 scores on the fly, the last pass writes int64 ids + fp32 scores.
#include "common.cuh"
#include "topk.cuh"
#include "rank_kernels.cuh"

using namespace crag;

extern "C" size_t crag_rank_workspace_bytes(int64_t n) {
  if (n < 0 || n >= (int64_t(1) << 31)) return 0;
  return plan_sort(n).total;
}

extern "C" int crag_rank_scores(const float* scores, int64_t n, int64_t* out_ids, float* out_scores, void* workspace,
                                size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n < 0 || n >= (int64_t(1) << 31)) return fail(CRAG_ERR_INVALID, "crag_rank_scores: n out of range (%lld)", (long long)n);
  if (n == 0) return CRAG_OK;
  if (!scores || !out_ids || !out_scores || !workspace) return fail(CRAG_ERR_INVALID, "crag_rank_scores: null pointer");
  const SortPlan p = plan_sort(n, workspace);
  const int rc = check_workspace("crag_rank_scores", workspace, workspace_bytes, p.total);
  if (rc != CRAG_OK) return rc;
  uint32_t* hist = p.hist;
  uint32_t* totals = hist + size_t(256) * p.n_warps;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = pass * 8;
    const uint32_t* kin = pass ? p.keys[(pass - 1) & 1] : nullptr;
    const uint32_t* vin = pass ? p.vals[(pass - 1) & 1] : nullptr;
    uint32_t* kout = p.keys[pass & 1];
    uint32_t* vout = p.vals[pass & 1];
    CRAG_CUDA_OK(cudaMemsetAsync(totals, 0, 256 * 4, stream));
    if (pass == 0) hist_kernel<true><<<p.grid, kSortThreads, 0, stream>>>(scores, nullptr, n, p.run, p.n_warps, shift, hist, totals);
    else hist_kernel<false><<<p.grid, kSortThreads, 0, stream>>>(nullptr, kin, n, p.run, p.n_warps, shift, hist, totals);
    scan_kernel<<<256, 256, 0, stream>>>(hist, totals, p.n_warps);
    if (pass == 0) scatter_kernel<true, false><<<p.grid, kSortThreads, 0, stream>>>(scores, nullptr, nullptr, n, p.run, p.n_warps, shift, hist, kout, vout, nullptr, nullptr);
    else if (pass < 3) scatter_kernel<false, false><<<p.grid, kSortThreads, 0, stream>>>(nullptr, kin, vin, n, p.run, p.n_warps, shift, hist, kout, vout, nullptr, nullptr);
    else scatter_kernel<false, true><<<p.grid, kSortThreads, 0, stream>>>(nullptr, kin, vin, n, p.run, p.n_warps, shift, hist, nullptr, nullptr, out_ids, out_scores);
    CRAG_CUDA_OK(cudaGetLastError());
  }
  return CRAG_OK;
}
