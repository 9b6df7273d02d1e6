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

bool misaligned(const void* ws) { return (reinterpret_cast<uintptr_t>(ws) & 255) != 0; }
}  // namespace

extern "C" size_t crag_umap_fuzzy_graph_workspace_bytes(int64_t n, int k) {
  if (n < 2 || n > kUmapMaxRows || k < 1 || k > kUmapMaxK || k > n) return 0;
  return umap_fuzzy_ws(n);
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
  if (misaligned(workspace)) return fail(CRAG_ERR_INVALID, "crag_umap_fuzzy_graph: workspace must be 256-byte aligned");
  if (workspace_bytes < umap_fuzzy_ws(n))
    return fail(CRAG_ERR_WORKSPACE, "crag_umap_fuzzy_graph: workspace %zu < %zu bytes", workspace_bytes,
                umap_fuzzy_ws(n));
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  double* rowsum = reinterpret_cast<double*>(ws);
  double* mean = reinterpret_cast<double*>(ws + umap_align(sizeof(double) * size_t(n)));
  const unsigned rows_grid = umap_blocks(n, kUmapThreads / 32);
  umap_knn_lists_kernel<<<rows_grid, kUmapThreads, 0, stream>>>(knn_ids, knn_scores, n, k, out_nbr, out_dist, rowsum);
  umap_mean_kernel<<<1, 1024, sizeof(double) * 1024, stream>>>(rowsum, n, k, mean);
  umap_smooth_kernel<<<rows_grid, kUmapThreads, 0, stream>>>(out_nbr, out_dist, rowsum, mean, n, k, out_rho, out_sigma,
                                                             out_memb);
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
  if (misaligned(workspace))
    return fail(CRAG_ERR_INVALID, "crag_umap_spectral_init: workspace must be 256-byte aligned");
  const UmapSpectralPlan s = plan_umap_spectral(n, d);
  if (workspace_bytes < s.total)
    return fail(CRAG_ERR_WORKSPACE, "crag_umap_spectral_init: workspace %zu < %zu bytes", workspace_bytes, s.total);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  double* deg = reinterpret_cast<double*>(ws + s.deg_off);
  double* dis = reinterpret_cast<double*>(ws + s.dis_off);
  double* v = reinterpret_cast<double*>(ws + s.v_off);
  double* w = reinterpret_cast<double*>(ws + s.w_off);
  double* part = reinterpret_cast<double*>(ws + s.part_off);
  double* rinv = reinterpret_cast<double*>(ws + s.rinv_off);
  double* q = reinterpret_cast<double*>(ws + s.q_off);
  double* yr = out_vectors ? out_vectors : reinterpret_cast<double*>(ws + s.yr_off);
  const int p = s.p;
  const unsigned np_grid = umap_blocks(n * p, kUmapThreads);
  const int loops = n <= 16 ? 0 : iters;       // n <= 16: p = n, Rayleigh-Ritz on the whole space is exact

  umap_degree_kernel<<<umap_blocks(n, kUmapThreads), kUmapThreads, 0, stream>>>(indptr, weights, n, deg, dis);
  umap_basis_kernel<<<np_grid, kUmapThreads, 0, stream>>>(deg, n, p, seed, v);
  for (int it = 0; it < loops; ++it) {
    umap_spmm_kernel<<<np_grid, kUmapThreads, 0, stream>>>(indptr, indices, weights, dis, n, p, v, w);
    umap_gram_kernel<<<s.chunks, kUmapGramThreads, 0, stream>>>(w, w, n, p, s.chunk_rows, part);
    umap_cholqr_kernel<<<1, 32, 0, stream>>>(part, s.chunks, p, rinv);
    umap_apply_r_kernel<<<np_grid, kUmapThreads, 0, stream>>>(w, rinv, n, p, v);
  }
  umap_spmm_kernel<<<np_grid, kUmapThreads, 0, stream>>>(indptr, indices, weights, dis, n, p, v, w);
  umap_gram_kernel<<<s.chunks, kUmapGramThreads, 0, stream>>>(v, w, n, p, s.chunk_rows, part);
  umap_ritz_kernel<<<1, 32, 0, stream>>>(part, s.chunks, p, q);
  umap_ritz_vectors_kernel<<<umap_blocks(n * d, kUmapThreads), kUmapThreads, 0, stream>>>(v, q, n, p, d, yr);
  umap_post_kernel<<<1, 1024, 0, stream>>>(yr, n, d, seed, out_y);
  if (out_eigenvalues)
    CRAG_CUDA_OK(cudaMemcpyAsync(out_eigenvalues, q + p * p, sizeof(double) * p, cudaMemcpyDeviceToDevice, stream));
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

extern "C" size_t crag_umap_optimize_workspace_bytes(int64_t n, int d) {
  if (n < 2 || n > kUmapMaxRows || d < 1 || d > kUmapMaxD) return 0;
  return umap_optimize_ws(n, d);
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
  if (misaligned(workspace)) return fail(CRAG_ERR_INVALID, "crag_umap_optimize: workspace must be 256-byte aligned");
  if (workspace_bytes < umap_optimize_ws(n, d))
    return fail(CRAG_ERR_WORKSPACE, "crag_umap_optimize: workspace %zu < %zu bytes", workspace_bytes,
                umap_optimize_ws(n, d));
  float* other = static_cast<float*>(workspace);
  const int epochs = epoch_end - epoch_begin;
  // the last epoch writes out_y: start in out_y after an even number of epochs, in the other buffer after an odd one
  float* cur = (epochs % 2 == 0) ? out_y : other;
  float* nxt = (epochs % 2 == 0) ? other : out_y;
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
