// crag_umap_fuzzy_graph, crag_umap_spectral_init, crag_umap_optimize: the three device stages of UMAP for
// ChunkSoftClustering._reduce_dimensions (cluster_utils.py:191-211).  The kernels and workspace plans live in
// umap_kernels.cuh; this file checks the arguments and enqueues on the caller's stream
//   fuzzy graph     knn lists, mean, smooth                                                   (3 launches)
//   spectral start  degree, basis, iters x (spmm, gram, cholqr, apply), spmm, gram, ritz,
//                   ritz vectors, post                                                        (4 iters + 7 launches)
//   optimize        one epoch kernel per epoch, double-buffered                               (epochs launches)
// The launch counts depend on the shapes and the host's arguments only; nothing waits for the host.
#include "common.cuh"
#include "umap_kernels.cuh"

using namespace crag;

namespace {
constexpr int64_t kUmapMaxRows = int64_t(1) << 30;

unsigned umap_blocks(int64_t items, int per_block) { return unsigned((items + per_block - 1) / per_block); }
}  // namespace

extern "C" size_t crag_umap_fuzzy_graph_workspace_bytes(int64_t n, int k) {
  if (n < 2 || n > kUmapMaxRows || k < 1 || k > kUmapMaxK || k > n) return 0;
  return umap_fuzzy_workspace(n).total;
}

extern "C" int crag_umap_fuzzy_graph(const int64_t* knn_ids, const float* knn_scores, int64_t n, int k,
                                     int32_t* out_nbr, float* out_dist, float* out_rho, float* out_sigma,
                                     float* out_memb, void* workspace, size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n < 2 || n > kUmapMaxRows)
    return fail(CRAG_ERR_INVALID, "crag_umap_fuzzy_graph: n out of range (%lld)", (long long)n);
  if (k < 1 || k > kUmapMaxK || k > n)
    return fail(CRAG_ERR_INVALID, "crag_umap_fuzzy_graph: k must be in [1, min(%d, n)] (got %d, n = %lld)", kUmapMaxK,
                k, (long long)n);
  if (!knn_ids || !knn_scores || !out_nbr || !out_dist || !out_rho || !out_sigma || !out_memb || !workspace)
    return fail(CRAG_ERR_INVALID, "crag_umap_fuzzy_graph: null pointer");
  const UmapFuzzyWorkspace w = umap_fuzzy_workspace(n, workspace);
  const int rc = check_workspace("crag_umap_fuzzy_graph", workspace, workspace_bytes, w.total);
  if (rc != CRAG_OK) return rc;
  const unsigned rows_grid = umap_blocks(n, kUmapThreads / 32);
  umap_knn_lists_kernel<<<rows_grid, kUmapThreads, 0, stream>>>(knn_ids, knn_scores, n, k, out_nbr, out_dist, w.rowsum);
  umap_mean_kernel<<<1, 1024, sizeof(double) * 1024, stream>>>(w.rowsum, n, k, w.mean);
  umap_smooth_kernel<<<rows_grid, kUmapThreads, 0, stream>>>(out_nbr, out_dist, w.rowsum, w.mean, n, k, out_rho,
                                                             out_sigma, out_memb);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

extern "C" size_t crag_umap_spectral_init_workspace_bytes(int64_t n, int d) {
  if (n < 2 || n > kUmapMaxRows || d < 1 || d > kUmapMaxD || d + 1 > n) return 0;
  return plan_umap_spectral(n, d).total;
}

extern "C" int crag_umap_spectral_init(const int64_t* indptr, const int32_t* indices, const float* weights, int64_t n,
                                       int d, int iters, uint64_t seed, float* out_y, double* out_vectors,
                                       double* out_eigenvalues, void* workspace, size_t workspace_bytes,
                                       crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n < 2 || n > kUmapMaxRows)
    return fail(CRAG_ERR_INVALID, "crag_umap_spectral_init: n out of range (%lld)", (long long)n);
  if (d < 1 || d > kUmapMaxD || d + 1 > n)
    return fail(CRAG_ERR_INVALID, "crag_umap_spectral_init: d must be in [1, min(%d, n - 1)] (got %d, n = %lld)",
                kUmapMaxD, d, (long long)n);
  if (iters < 0 || (n > 16 && iters < 1))
    return fail(CRAG_ERR_INVALID, "crag_umap_spectral_init: iters must be >= 1 for n > 16 (got %d)", iters);
  if (!indptr || !indices || !weights || !out_y || !workspace)
    return fail(CRAG_ERR_INVALID, "crag_umap_spectral_init: null pointer");
  const UmapSpectralPlan s = plan_umap_spectral(n, d, workspace);
  const int rc = check_workspace("crag_umap_spectral_init", workspace, workspace_bytes, s.total);
  if (rc != CRAG_OK) return rc;
  double* yr = out_vectors ? out_vectors : s.yr;
  const int p = s.p;
  const unsigned np_grid = umap_blocks(n * p, kUmapThreads);
  const int loops = n <= 16 ? 0 : iters;       // n <= 16: p = n, Rayleigh-Ritz on the whole space is exact

  umap_degree_kernel<<<umap_blocks(n, kUmapThreads), kUmapThreads, 0, stream>>>(indptr, weights, n, s.deg, s.dis);
  umap_basis_kernel<<<np_grid, kUmapThreads, 0, stream>>>(s.deg, n, p, seed, s.v);
  for (int it = 0; it < loops; ++it) {
    umap_spmm_kernel<<<np_grid, kUmapThreads, 0, stream>>>(indptr, indices, weights, s.dis, n, p, s.v, s.w);
    umap_gram_kernel<<<s.chunks, kUmapGramThreads, 0, stream>>>(s.w, s.w, n, p, s.chunk_rows, s.part);
    umap_cholqr_kernel<<<1, 32, 0, stream>>>(s.part, s.chunks, p, s.rinv);
    umap_apply_r_kernel<<<np_grid, kUmapThreads, 0, stream>>>(s.w, s.rinv, n, p, s.v);
  }
  umap_spmm_kernel<<<np_grid, kUmapThreads, 0, stream>>>(indptr, indices, weights, s.dis, n, p, s.v, s.w);
  umap_gram_kernel<<<s.chunks, kUmapGramThreads, 0, stream>>>(s.v, s.w, n, p, s.chunk_rows, s.part);
  umap_ritz_kernel<<<1, 32, 0, stream>>>(s.part, s.chunks, p, s.q);
  umap_ritz_vectors_kernel<<<umap_blocks(n * d, kUmapThreads), kUmapThreads, 0, stream>>>(s.v, s.q, n, p, d, yr);
  umap_post_kernel<<<1, 1024, 0, stream>>>(yr, n, d, seed, out_y);
  if (out_eigenvalues)
    CRAG_CUDA_OK(cudaMemcpyAsync(out_eigenvalues, s.q + p * p, sizeof(double) * p, cudaMemcpyDeviceToDevice, stream));
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

extern "C" size_t crag_umap_optimize_workspace_bytes(int64_t n, int d) {
  if (n < 2 || n > kUmapMaxRows || d < 1 || d > kUmapMaxD) return 0;
  return umap_optimize_workspace(n, d).total;
}

extern "C" int crag_umap_optimize(const int64_t* indptr, const int32_t* indices, const double* epochs_per_sample,
                                  int64_t n, int64_t nnz, int d, float a, float b, int n_epochs, int epoch_begin,
                                  int epoch_end, uint64_t seed, double* next_sample, double* next_neg,
                                  const float* y0, float* out_y, void* workspace, size_t workspace_bytes,
                                  crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n < 2 || n > kUmapMaxRows)
    return fail(CRAG_ERR_INVALID, "crag_umap_optimize: n out of range (%lld)", (long long)n);
  if (d < 1 || d > kUmapMaxD) return fail(CRAG_ERR_INVALID, "crag_umap_optimize: d must be in [1, %d] (got %d)", kUmapMaxD, d);
  if (nnz < 0) return fail(CRAG_ERR_INVALID, "crag_umap_optimize: nnz must be >= 0");
  if (n_epochs < 1 || epoch_begin < 0 || epoch_end < epoch_begin || epoch_end > n_epochs)
    return fail(CRAG_ERR_INVALID, "crag_umap_optimize: need 0 <= epoch_begin <= epoch_end <= n_epochs (got %d, %d, %d)",
                epoch_begin, epoch_end, n_epochs);
  if (!(a > 0.0f) || !(b > 0.0f)) return fail(CRAG_ERR_INVALID, "crag_umap_optimize: a and b must be positive");
  if (!indptr || (nnz > 0 && (!indices || !epochs_per_sample || !next_sample || !next_neg)) || !y0 || !out_y ||
      !workspace)
    return fail(CRAG_ERR_INVALID, "crag_umap_optimize: null pointer");
  const UmapOptimizeWorkspace w = umap_optimize_workspace(n, d, workspace);
  const int rc = check_workspace("crag_umap_optimize", workspace, workspace_bytes, w.total);
  if (rc != CRAG_OK) return rc;
  const int epochs = epoch_end - epoch_begin;
  // the last epoch writes out_y: start in out_y after an even number of epochs, in the other buffer after an odd one
  float* cur = (epochs % 2 == 0) ? out_y : w.other;
  float* nxt = (epochs % 2 == 0) ? w.other : out_y;
  const size_t bytes = sizeof(float) * size_t(n) * size_t(d);
  if (cur != y0) CRAG_CUDA_OK(cudaMemcpyAsync(cur, y0, bytes, cudaMemcpyDeviceToDevice, stream));
  for (int e = epoch_begin; e < epoch_end; ++e) {
    const float alpha = float(1.0 - double(e > 1 ? e - 1 : 0) / double(n_epochs));
    umap_epoch_kernel<<<umap_blocks(n, kUmapThreads), kUmapThreads, 0, stream>>>(
        indptr, indices, epochs_per_sample, n, d, a, b, e, alpha, seed, next_sample, next_neg, cur, nxt);
    float* t = cur;
    cur = nxt;
    nxt = t;
  }
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}
