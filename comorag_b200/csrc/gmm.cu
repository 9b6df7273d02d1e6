// crag_gmm_sweep: the BIC sweep of ComoRAG's soft clustering (cluster_utils.py:175-189, then the refit and
// predict_proba of :252-260 / :315-323) on the device.  The kernels and the workspace plan live in gmm_kernels.cuh;
// this file checks the arguments and enqueues
//   moments, centre, seed, 300 x (Lloyd assign, Lloyd update), final assign, EM setup, init stats, init M-step,
//   100 x (EM stats, M-step), score, select, memberships
// on the caller's stream.  The launch count depends on M only: a model that has finished keeps a done flag on the
// device and the later launches skip it, so nothing waits for the host.
#include "common.cuh"
#include "gmm_kernels.cuh"

using namespace crag;

namespace {
constexpr int64_t kGmmMaxRows = int64_t(1) << 31;

unsigned gmm_blocks(int64_t items, int per_block) { return unsigned((items + per_block - 1) / per_block); }

size_t em_stats_smem(int m, int d) { return sizeof(double) * size_t(kGmmTile) * (m + d); }
size_t lloyd_assign_smem(int m, int d) {
  return sizeof(double) * size_t(m * d + kGmmThreads * d) + sizeof(int32_t) * 2 * kGmmThreads;
}
size_t lloyd_update_smem(int m, int d) {
  return sizeof(double) * size_t(m * (d + 1) + kGmmThreads) + sizeof(int64_t) * (kGmmMaxM + kGmmThreads) +
         sizeof(int) * (kGmmMaxM + 1);
}
size_t mstep_smem(int d) { return sizeof(double) * size_t((kGmmThreads / 32) * (1 + d + gmm_tri(d)) + 2 * kGmmMaxM) + 16; }
constexpr size_t kSeedSmem = sizeof(double) * (2 * kGmmSeedThreads + 1 + kGmmMaxTrials * (1 + kGmmMaxD)) +
                             sizeof(int64_t) * kGmmMaxTrials;
}  // namespace

extern "C" size_t crag_gmm_sweep_workspace_bytes(int64_t n, int d, int max_components) {
  if (n < 2 || n > kGmmMaxRows || d < 1 || d > kGmmMaxD || max_components < 1 || max_components > kGmmMaxM ||
      max_components > n - 1)
    return 0;
  return plan_gmm(n, d, max_components).total;
}

extern "C" int crag_gmm_sweep(const double* x, int64_t n, int d, int max_components, const int64_t* first_centre,
                              const double* seed_draws, double* out_bic, int32_t* out_iters, int32_t* out_converged,
                              int32_t* out_best, double* out_weights, double* out_means, double* out_memberships,
                              int32_t* out_seeds, int32_t* out_labels, void* workspace, size_t workspace_bytes,
                              crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int M = max_components;
  if (n < 2 || n > kGmmMaxRows) return fail(CRAG_ERR_INVALID, "crag_gmm_sweep: n out of range (%lld)", (long long)n);
  if (d < 1 || d > kGmmMaxD) return fail(CRAG_ERR_INVALID, "crag_gmm_sweep: d must be in [1, %d] (got %d)", kGmmMaxD, d);
  if (M < 1 || M > kGmmMaxM || M > n - 1)
    return fail(CRAG_ERR_INVALID, "crag_gmm_sweep: max_components must be in [1, min(%d, n - 1)] (got %d, n = %lld)",
                kGmmMaxM, M, (long long)n);
  if (!x || !first_centre || (M > 1 && !seed_draws) || !out_bic || !out_iters || !out_converged || !out_best ||
      !out_weights || !out_means || !out_memberships || !workspace)
    return fail(CRAG_ERR_INVALID, "crag_gmm_sweep: null pointer");
  if (reinterpret_cast<uintptr_t>(workspace) & 255)
    return fail(CRAG_ERR_INVALID, "crag_gmm_sweep: workspace must be 256-byte aligned");
  const GmmPlan p = plan_gmm(n, d, M);
  if (workspace_bytes < p.total)
    return fail(CRAG_ERR_WORKSPACE, "crag_gmm_sweep: workspace %zu < %zu bytes", workspace_bytes, p.total);

  uint8_t* ws = static_cast<uint8_t*>(workspace);
  double* glob = reinterpret_cast<double*>(ws + p.glob_off);
  GmmState* state = reinterpret_cast<GmmState*>(ws + p.state_off);
  double* xc = reinterpret_cast<double*>(ws + p.xc_off);
  int32_t* labels = out_labels ? out_labels : reinterpret_cast<int32_t*>(ws + p.labels_off);
  double* dist = reinterpret_cast<double*>(ws + p.dist_off);
  double* centres = reinterpret_cast<double*>(ws + p.centre_off);
  double* lsum = reinterpret_cast<double*>(ws + p.lsum_off);
  int32_t* lchg = reinterpret_cast<int32_t*>(ws + p.lchg_off);
  double* mu = reinterpret_cast<double*>(ws + p.mu_off);
  double* prec = reinterpret_cast<double*>(ws + p.prec_off);
  double* cst = reinterpret_cast<double*>(ws + p.cst_off);
  double* wt = reinterpret_cast<double*>(ws + p.wt_off);
  double* esum = reinterpret_cast<double*>(ws + p.esum_off);
  double* lse = reinterpret_cast<double*>(ws + p.lse_off);
  int32_t* seeds = out_seeds ? out_seeds : reinterpret_cast<int32_t*>(ws + p.seeds_off);
  const int R = p.chunks, C = p.components;
  const unsigned grid = unsigned(R) * unsigned(M);

  gmm_moments_kernel<<<1, 1024, sizeof(double) * 1024, stream>>>(x, n, d, M, glob, state);
  gmm_centre_kernel<<<gmm_blocks(n * (d > M ? d : M), kGmmThreads * 8), kGmmThreads, 0, stream>>>(x, n, d, M, glob, xc,
                                                                                                  labels);
  gmm_seed_kernel<<<M, kGmmSeedThreads, kSeedSmem, stream>>>(xc, n, d, first_centre, seed_draws, dist, centres, seeds);
  const size_t assign_smem = lloyd_assign_smem(M, d), update_smem = lloyd_update_smem(M, d);
  for (int it = 0; it < kGmmLloydIters; ++it) {
    gmm_lloyd_assign_kernel<<<grid, kGmmThreads, assign_smem, stream>>>(xc, n, d, M, R, p.chunk_rows, 1, state, centres,
                                                                       labels, dist, lsum, lchg);
    gmm_lloyd_update_kernel<<<M, kGmmThreads, update_smem, stream>>>(xc, n, d, M, R, it, glob, state, centres, labels,
                                                                    dist, lsum, lchg);
  }
  gmm_lloyd_assign_kernel<<<grid, kGmmThreads, assign_smem, stream>>>(xc, n, d, M, R, p.chunk_rows, 0, state, centres,
                                                                     labels, dist, lsum, lchg);
  gmm_em_setup_kernel<<<gmm_blocks(int64_t(C) * d, kGmmThreads), kGmmThreads, 0, stream>>>(d, C, glob, centres, mu);
  const size_t stats_smem = em_stats_smem(M, d), m_smem = mstep_smem(d);
  gmm_em_stats_kernel<<<grid, kGmmThreads, stats_smem, stream>>>(x, n, d, M, R, p.chunk_rows, kGmmInit, state, nullptr,
                                                                 labels, mu, prec, cst, esum, lse, nullptr);
  gmm_mstep_kernel<<<M, kGmmThreads, m_smem, stream>>>(n, d, M, R, kGmmInit, 0, state, mu, prec, cst, wt, esum, lse);
  for (int it = 1; it <= kGmmEmIters; ++it) {
    gmm_em_stats_kernel<<<grid, kGmmThreads, stats_smem, stream>>>(x, n, d, M, R, p.chunk_rows, kGmmStep, state,
                                                                   nullptr, labels, mu, prec, cst, esum, lse, nullptr);
    gmm_mstep_kernel<<<M, kGmmThreads, m_smem, stream>>>(n, d, M, R, kGmmStep, it, state, mu, prec, cst, wt, esum, lse);
  }
  gmm_em_stats_kernel<<<grid, kGmmThreads, stats_smem, stream>>>(x, n, d, M, R, p.chunk_rows, kGmmScore, state, nullptr,
                                                                 labels, mu, prec, cst, esum, lse, nullptr);
  gmm_select_kernel<<<1, kGmmMaxM, sizeof(double) * (kGmmMaxM + 1), stream>>>(
      n, d, M, R, state, mu, wt, lse, out_bic, out_iters, out_converged, out_best, out_weights, out_means);
  gmm_em_stats_kernel<<<unsigned(R), kGmmThreads, stats_smem, stream>>>(x, n, d, M, R, p.chunk_rows, kGmmResp, state,
                                                                        out_best, labels, mu, prec, cst, esum, lse,
                                                                        out_memberships);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}
