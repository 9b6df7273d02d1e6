// The BIC sweep of ComoRAG's soft clustering (ChunkSoftClustering._get_optimal_clusters, cluster_utils.py:175-189):
// the kernels of crag_gmm_sweep (gmm.cu).  Model m (m = 1..M) is scikit-learn's
//     GaussianMixture(n_components=m, covariance_type="full", random_state=RandomState(224))
// in float64: k-means++ seeding on the column-centred rows (the random draws come from the host, they do not depend
// on the data), Lloyd, then EM from the one-hot k-means labels; BIC on the final parameters, and the memberships of
// the first BIC argmin.  DESIGN.md section 2b restates the algorithm.  All M models advance together:
//   gmm_moments_kernel        column means and the k-means tolerance 1e-4 * mean(var(X, axis=0)); per-model state
//   gmm_centre_kernel         Xc = X - mean; k-means labels := -1
//   gmm_seed_kernel           one block per model: the whole k-means++ seeding
//   gmm_lloyd_assign_kernel   (row chunk, model) blocks: labels, distances, per-chunk cluster sums
//   gmm_lloyd_update_kernel   one block per model: chunk sums reduced in chunk order, empty-cluster relocation,
//                             new centres, convergence (labels unchanged, or squared centre shift <= tol)
//   gmm_em_stats_kernel       (row chunk, model) blocks: E-step fused with the sufficient statistics
//                             sum r, sum r (x - s), sum r (x - s)(x - s)^T  (s = the component's current mean)
//   gmm_mstep_kernel          one block per model, one warp per component: statistics reduced in chunk order,
//                             means, covariances + reg_covar, Cholesky and triangular inverse in registers, weights,
//                             lower bound and the per-model convergence test |delta| < 1e-3
//   gmm_select_kernel         BIC per model, the first argmin, the winner's weights and means
// A model that has converged keeps its done flag on the device; every later launch skips it.  No floating-point
// atomics, and every sum runs in an order fixed by the shapes alone: the same input gives the same bits on any run
// and stream.  Pure SIMT code (no wgmma / TMA / mbarrier), so tests/warp_emu runs this very header on emulated blocks.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

#ifndef CRAG_EMULATED_PTX   // tests/warp_emu gives every emulated block its own dynamic shared memory
#define CRAG_DYNAMIC_SHARED(type, name) extern __shared__ type name[]
#endif

namespace crag {
namespace {

constexpr int kGmmMaxD = 16;
constexpr int kGmmMaxM = 64;
constexpr int kGmmMaxTrials = 8;                   // 2 + int(log m) <= 6 for m <= 64
constexpr int kGmmThreads = 256;                   // every kernel but the seeding
constexpr int kGmmSeedThreads = 512;
constexpr int kGmmTile = 32;                       // rows per E-step tile: one per lane
constexpr int kGmmChunkRows = 256;                 // rows per chunk, until there are kGmmMaxChunks chunks
constexpr int kGmmMaxChunks = 32;
constexpr int kGmmLloydIters = 300;                // KMeans(max_iter=300)
constexpr int kGmmEmIters = 100;                   // GaussianMixture(max_iter=100)
constexpr double kGmmEmTol = 1e-3;
constexpr double kGmmRegCovar = 1e-6;
constexpr double kGmmKmeansTol = 1e-4;
constexpr double kGmmEps10 = 10 * 2.220446049250313e-16;   // 10 * finfo(float64).eps, added to every nk
constexpr double kGmmLog2Pi = 1.8378770664093453;

enum GmmStatsMode { kGmmInit = 0, kGmmStep = 1, kGmmScore = 2, kGmmResp = 3 };

struct GmmState {
  double lower_bound;                              // the last E-step's mean log-likelihood (-inf before the first)
  int32_t lloyd_done, lloyd_strict, lloyd_iters;
  int32_t em_done, em_iters, em_converged;         // em_converged -1: a covariance was not positive definite
};

struct GmmPlan {
  int chunks, stats, components;                   // row chunks R, statistics per component S, sum of m for m <= M
  int64_t chunk_rows;
  size_t glob_off, state_off, seeds_off, xc_off, labels_off, dist_off, centre_off, lsum_off, lchg_off, mu_off, prec_off,
      cst_off, wt_off, esum_off, lse_off, total;
};

inline size_t gmm_align(size_t b) { return (b + 255) & ~size_t(255); }
__host__ __device__ inline int64_t gmm_min64(int64_t a, int64_t b) { return a < b ? a : b; }
__host__ __device__ inline int gmm_tri(int d) { return d * (d + 1) / 2; }
__host__ __device__ inline int gmm_comp_off(int m) { return m * (m - 1) / 2; }   // model m's first component
__host__ __device__ inline int gmm_trials(int m) { return 2 + int(log(double(m))); }
__host__ __device__ inline int64_t gmm_draw_off(int m) {                         // model m's first k-means++ draw
  int64_t off = 0;
  for (int j = 1; j < m; ++j) off += int64_t(j - 1) * gmm_trials(j);
  return off;
}

// Workspace: globals (mean[16], tol), per-model state, k-means++ rows int32 [C], Xc [n][d], labels int32 [M][n], distances [M][n], k-means
// centres [C][d], Lloyd chunk sums [R][C][d + 1] and label-change counts int32 [R][M], means [C][d], packed precision
// Cholesky factors [C][d(d+1)/2], log weight + log det constants [C], weights [C], EM chunk statistics [R][C][S], log-likelihood
// chunk sums [R][M]; C = M(M+1)/2 components, S = 1 + d + d(d+1)/2.  Nothing scales with n * C.
inline GmmPlan plan_gmm(int64_t n, int d, int M) {
  GmmPlan p;
  const int64_t want = (n + kGmmChunkRows - 1) / kGmmChunkRows;
  p.chunks = int(want < 1 ? 1 : want > kGmmMaxChunks ? kGmmMaxChunks : want);
  p.chunk_rows = (n + p.chunks - 1) / p.chunks;
  p.stats = 1 + d + gmm_tri(d);
  p.components = M * (M + 1) / 2;
  const size_t C = size_t(p.components), R = size_t(p.chunks);
  size_t o = 0;
  p.glob_off = o;    o += gmm_align(sizeof(double) * (kGmmMaxD + 1));
  p.state_off = o;   o += gmm_align(sizeof(GmmState) * M);
  p.seeds_off = o;   o += gmm_align(sizeof(int32_t) * C);
  p.xc_off = o;      o += gmm_align(sizeof(double) * size_t(n) * d);
  p.labels_off = o;  o += gmm_align(sizeof(int32_t) * size_t(n) * M);
  p.dist_off = o;    o += gmm_align(sizeof(double) * size_t(n) * M);
  p.centre_off = o;  o += gmm_align(sizeof(double) * C * d);
  p.lsum_off = o;    o += gmm_align(sizeof(double) * R * C * (d + 1));
  p.lchg_off = o;    o += gmm_align(sizeof(int32_t) * R * M);
  p.mu_off = o;      o += gmm_align(sizeof(double) * C * d);
  p.prec_off = o;    o += gmm_align(sizeof(double) * C * gmm_tri(d));
  p.cst_off = o;     o += gmm_align(sizeof(double) * C);
  p.wt_off = o;      o += gmm_align(sizeof(double) * C);
  p.esum_off = o;    o += gmm_align(sizeof(double) * R * C * p.stats);
  p.lse_off = o;     o += gmm_align(sizeof(double) * R * M);
  p.total = o;
  return p;
}

// Fixed pairwise tree over the block's threads (blockDim.x a power of two); every thread gets the total.
__device__ __forceinline__ double gmm_block_sum(double v, double* s_red) {
  s_red[threadIdx.x] = v;
  __syncthreads();
  for (int w = int(blockDim.x) / 2; w > 0; w >>= 1) {
    if (int(threadIdx.x) < w) s_red[threadIdx.x] = s_red[threadIdx.x] + s_red[threadIdx.x + w];
    __syncthreads();
  }
  const double total = s_red[0];
  __syncthreads();
  return total;
}

__device__ __forceinline__ double gmm_warp_sum(double v) {          // fixed butterfly: every lane gets the total
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One block of 1024 threads: mean[j] = column mean, glob[kGmmMaxD] = 1e-4 * mean_j var_j; per-model state reset.
__global__ void __launch_bounds__(1024) gmm_moments_kernel(const double* __restrict__ x, int64_t n, int d, int M,
                                                           double* __restrict__ glob, GmmState* __restrict__ state) {
  CRAG_DYNAMIC_SHARED(double, s_red);
  double var_sum = 0.0;
  for (int j = 0; j < d; ++j) {
    double acc = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) acc += x[i * d + j];
    const double mean = gmm_block_sum(acc, s_red) / double(n);
    double sq = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const double c = x[i * d + j] - mean;
      sq += c * c;
    }
    var_sum += gmm_block_sum(sq, s_red) / double(n);
    if (threadIdx.x == 0) glob[j] = mean;
  }
  if (threadIdx.x == 0) glob[kGmmMaxD] = var_sum / double(d) * kGmmKmeansTol;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    GmmState s;
    s.lower_bound = -INFINITY;
    s.lloyd_done = s.lloyd_strict = s.lloyd_iters = 0;
    s.em_done = s.em_iters = s.em_converged = 0;
    state[m] = s;
  }
}

__global__ void __launch_bounds__(kGmmThreads) gmm_centre_kernel(const double* __restrict__ x, int64_t n, int d, int M,
                                                                 const double* __restrict__ glob,
                                                                 double* __restrict__ xc, int32_t* __restrict__ labels) {
  const int64_t stride = int64_t(gridDim.x) * kGmmThreads;
  for (int64_t e = int64_t(blockIdx.x) * kGmmThreads + threadIdx.x; e < n * d; e += stride) xc[e] = x[e] - glob[e % d];
  for (int64_t e = int64_t(blockIdx.x) * kGmmThreads + threadIdx.x; e < n * M; e += stride) labels[e] = -1;
}

__device__ __forceinline__ double gmm_d2(const double* __restrict__ a, const double* __restrict__ b, int d) {
  double s = 0.0;
  for (int j = 0; j < d; ++j) {
    const double t = a[j] - b[j];
    s += t * t;
  }
  return s;
}

// k-means++ for model m = blockIdx.x + 1 (scikit-learn's _kmeans_plusplus with unit sample weights): the first centre
// is first_centre[m - 1]; centre c >= 1 takes trials = 2 + int(log m) draws u, looks each value u * pot up in the
// running sum of the closest squared distances (the first row whose running sum reaches it, clipped to n - 1), and
// keeps the candidate whose potential sum_i min(closest_i, |x_i - x_cand|^2) is smallest (the first on a tie).
// Each thread owns a contiguous run of rows; the runs' totals are scanned in order by one thread, so the running sum
// never decreases and the row a value falls on is well defined.
__global__ void __launch_bounds__(kGmmSeedThreads) gmm_seed_kernel(const double* __restrict__ xc, int64_t n, int d,
                                                                   const int64_t* __restrict__ first_centre,
                                                                   const double* __restrict__ draws,
                                                                   double* __restrict__ dist_all,
                                                                   double* __restrict__ centres,
                                                                   int32_t* __restrict__ seeds) {
  CRAG_DYNAMIC_SHARED(double, s_mem);
  double* s_red = s_mem;                               // [kGmmSeedThreads]
  double* s_excl = s_mem + kGmmSeedThreads;            // [kGmmSeedThreads + 1] running sum before each run
  double* s_pot = s_excl + kGmmSeedThreads + 1;        // [kGmmMaxTrials]
  double* s_cand_x = s_pot + kGmmMaxTrials;            // [kGmmMaxTrials][kGmmMaxD]
  int64_t* s_cand = reinterpret_cast<int64_t*>(s_cand_x + kGmmMaxTrials * kGmmMaxD);   // [kGmmMaxTrials]
  const int m = int(blockIdx.x) + 1;
  const int T = int(blockDim.x), tid = int(threadIdx.x);
  const int trials = gmm_trials(m);
  double* closest = dist_all + int64_t(m - 1) * n;
  const int64_t run = (n + T - 1) / T, lo = gmm_min64(int64_t(tid) * run, n), hi = gmm_min64(lo + run, n);
  const double* dr = draws + gmm_draw_off(m);
  double cx[kGmmMaxD];

  int64_t best_id = first_centre[m - 1];
  for (int j = 0; j < d; ++j) cx[j] = xc[best_id * d + j];
  double acc = 0.0;
  for (int64_t i = lo; i < hi; ++i) {
    closest[i] = gmm_d2(xc + i * d, cx, d);
    acc += closest[i];
  }
  double pot = gmm_block_sum(acc, s_red);
  if (tid == 0) seeds[gmm_comp_off(m)] = int32_t(best_id);
  if (tid < d) centres[int64_t(gmm_comp_off(m)) * d + tid] = cx[tid];

  for (int c = 1; c < m; ++c) {
    double mine = 0.0;                                 // this run's total, summed in row order
    for (int64_t i = lo; i < hi; ++i) mine += closest[i];
    s_red[tid] = mine;
    __syncthreads();
    if (tid == 0) {
      double r = 0.0;
      for (int t = 0; t < T; ++t) {
        s_excl[t] = r;
        r = r + s_red[t];
      }
      s_excl[T] = r;
    }
    __syncthreads();
    if (tid < trials) {
      const double v = dr[int64_t(c - 1) * trials + tid] * pot;
      int a = 0, b = T;                                // the first run whose end reaches v
      while (a < b) {
        const int mid = (a + b) >> 1;
        if (s_excl[mid + 1] >= v) b = mid;
        else a = mid + 1;
      }
      int64_t id = n - 1;
      if (a < T) {
        const int64_t r_lo = gmm_min64(int64_t(a) * run, n), r_hi = gmm_min64(r_lo + run, n);
        double s = 0.0;
        for (int64_t i = r_lo; i < r_hi; ++i) {
          s += closest[i];
          if (s_excl[a] + s >= v) { id = i; break; }
        }
      }
      s_cand[tid] = id;
      for (int j = 0; j < d; ++j) s_cand_x[tid * kGmmMaxD + j] = xc[id * d + j];
    }
    __syncthreads();
    for (int t = 0; t < trials; ++t) {
      double part = 0.0;
      for (int64_t i = lo; i < hi; ++i) part += fmin(closest[i], gmm_d2(xc + i * d, s_cand_x + t * kGmmMaxD, d));
      const double total = gmm_block_sum(part, s_red);
      if (tid == 0) s_pot[t] = total;
    }
    __syncthreads();
    int best = 0;
    for (int t = 1; t < trials; ++t)
      if (s_pot[t] < s_pot[best]) best = t;
    pot = s_pot[best];
    best_id = s_cand[best];
    for (int j = 0; j < d; ++j) cx[j] = s_cand_x[best * kGmmMaxD + j];
    for (int64_t i = lo; i < hi; ++i) closest[i] = fmin(closest[i], gmm_d2(xc + i * d, cx, d));
    if (tid == 0) seeds[gmm_comp_off(m) + c] = int32_t(best_id);
    if (tid < d) centres[int64_t(gmm_comp_off(m) + c) * d + tid] = cx[tid];
    __syncthreads();
  }
}

// Block b: model m = b / R + 1, rows [r * chunk_rows, (r + 1) * chunk_rows) with r = b % R, one row per thread and
// tile.  Each row gets the nearest centre (the first on a tie) and its squared distance; update == 1 also writes the
// chunk's per-cluster sums of Xc and counts ([R][C][d + 1], summed over the tile's rows in row order) and its
// number of changed labels.  update == 0 is the final assignment of a model whose Lloyd loop did not end on
// unchanged labels.
__global__ void __launch_bounds__(kGmmThreads) gmm_lloyd_assign_kernel(
    const double* __restrict__ xc, int64_t n, int d, int M, int R, int64_t chunk_rows, int update,
    const GmmState* __restrict__ state, const double* __restrict__ centres, int32_t* __restrict__ labels_all,
    double* __restrict__ dist_all, double* __restrict__ lsum, int32_t* __restrict__ lchg) {
  CRAG_DYNAMIC_SHARED(double, s_mem);
  const int m = int(blockIdx.x) / R + 1, r = int(blockIdx.x) % R, tid = int(threadIdx.x);
  const GmmState st = state[m - 1];
  if (update ? st.lloyd_done : st.lloyd_strict) return;
  double* s_c = s_mem;                                 // [m][d]
  double* s_x = s_mem + m * d;                         // [kGmmThreads][d]
  int32_t* s_lab = reinterpret_cast<int32_t*>(s_x + kGmmThreads * d);
  int* s_cnt = s_lab + kGmmThreads;                    // [kGmmThreads] changed-label counts
  const int off = gmm_comp_off(m);
  for (int e = tid; e < m * d; e += kGmmThreads) s_c[e] = centres[int64_t(off) * d + e];
  const int tasks = m * (d + 1);
  const int comps = gmm_comp_off(M + 1);
  double* part = lsum + int64_t(r) * comps * (d + 1) + int64_t(off) * (d + 1);
  if (update)
    for (int t = tid; t < tasks; t += kGmmThreads) part[t] = 0.0;
  __syncthreads();
  int32_t* labels = labels_all + int64_t(m - 1) * n;
  double* dist = dist_all + int64_t(m - 1) * n;
  const int64_t row0 = int64_t(r) * chunk_rows, row1 = gmm_min64(row0 + chunk_rows, n);
  int changed = 0;
  for (int64_t t0 = row0; t0 < row1; t0 += kGmmThreads) {
    const int64_t i = t0 + tid;
    int lab = -1;
    if (i < row1) {
      for (int j = 0; j < d; ++j) s_x[tid * d + j] = xc[i * d + j];
      double best = INFINITY;
      for (int k = 0; k < m; ++k) {
        const double dk = gmm_d2(s_x + tid * d, s_c + k * d, d);
        if (dk < best) { best = dk; lab = k; }
      }
      changed += labels[i] != lab;
      labels[i] = lab;
      dist[i] = best;
    }
    s_lab[tid] = lab;
    __syncthreads();
    if (update) {
      const int rows = int(gmm_min64(kGmmThreads, row1 - t0));
      for (int t = tid; t < tasks; t += kGmmThreads) {
        const int k = t / (d + 1), j = t % (d + 1);
        double s = 0.0;
        for (int p = 0; p < rows; ++p)
          if (s_lab[p] == k) s += j < d ? s_x[p * d + j] : 1.0;
        part[t] += s;
      }
    }
    __syncthreads();
  }
  if (!update) return;
  s_cnt[tid] = changed;
  __syncthreads();
  if (tid == 0) {
    int total = 0;
    for (int t = 0; t < kGmmThreads; ++t) total += s_cnt[t];
    lchg[int64_t(r) * M + (m - 1)] = total;
  }
}

// One block per model, iteration `iter` of the Lloyd loop (scikit-learn 1.9's lloyd_iter_chunked_dense): chunk sums
// reduced in chunk order; unless every row sits on its centre, every empty cluster takes one of the rows farthest
// from their centres (descending distance, the higher row first on a tie), which leaves its old cluster
// (_relocate_empty_clusters_dense); centres = sums * (1 / weight), and a cluster still empty takes the heaviest
// cluster's row as it stands at that point of the pass (_average_centers); then the loop ends on unchanged labels
// (strict), on a squared centre shift <= tol, or after kGmmLloydIters iterations.
__global__ void __launch_bounds__(kGmmThreads) gmm_lloyd_update_kernel(
    const double* __restrict__ xc, int64_t n, int d, int M, int R, int iter, const double* __restrict__ glob,
    GmmState* __restrict__ state, double* __restrict__ centres, const int32_t* __restrict__ labels_all,
    const double* __restrict__ dist_all, const double* __restrict__ lsum, const int32_t* __restrict__ lchg) {
  CRAG_DYNAMIC_SHARED(double, s_mem);
  const int m = int(blockIdx.x) + 1, tid = int(threadIdx.x);
  GmmState* st = state + (m - 1);
  if (st->lloyd_done) return;
  double* s_sum = s_mem;                               // [m][d + 1]
  double* s_red = s_sum + m * (d + 1);                 // [kGmmThreads]
  int64_t* s_far = reinterpret_cast<int64_t*>(s_red + kGmmThreads);   // [kGmmMaxM] relocated rows
  int64_t* s_idx = s_far + kGmmMaxM;                   // [kGmmThreads]
  int* s_empty = reinterpret_cast<int*>(s_idx + kGmmThreads);         // [kGmmMaxM + 1]
  const int off = gmm_comp_off(m), comps = gmm_comp_off(M + 1), tasks = m * (d + 1);
  for (int t = tid; t < tasks; t += kGmmThreads) {
    double s = 0.0;
    for (int r = 0; r < R; ++r) s += lsum[int64_t(r) * comps * (d + 1) + int64_t(off) * (d + 1) + t];
    s_sum[t] = s;
  }
  __syncthreads();
  if (tid == 0) {
    int e = 0;
    for (int k = 0; k < m; ++k)
      if (s_sum[k * (d + 1) + d] == 0.0) s_empty[1 + e++] = k;
    s_empty[0] = e;
  }
  __syncthreads();
  const int n_empty = s_empty[0];
  const double* dist = dist_all + int64_t(m - 1) * n;
  // the n_empty farthest rows, one block argmax each: the largest (distance, row) below the previous pick
  double prev_d = INFINITY;
  int64_t prev_i = 0;
  for (int e = 0; e < n_empty; ++e) {
    double bd = -1.0;
    int64_t bi = -1;
    for (int64_t i = tid; i < n; i += kGmmThreads) {
      const double di = dist[i];
      const bool below = di < prev_d || (di == prev_d && i < prev_i);
      if (below && (di > bd || (di == bd && i > bi))) { bd = di; bi = i; }
    }
    s_red[tid] = bd;
    s_idx[tid] = bi;
    __syncthreads();
    if (tid == 0) {
      for (int t = 1; t < kGmmThreads; ++t)
        if (s_red[t] > s_red[0] || (s_red[t] == s_red[0] && s_idx[t] > s_idx[0])) {
          s_red[0] = s_red[t];
          s_idx[0] = s_idx[t];
        }
      s_far[e] = s_idx[0];
    }
    __syncthreads();
    prev_d = s_red[0];
    prev_i = s_idx[0];
    __syncthreads();
  }
  if (tid == 0) {
    const int32_t* labels = labels_all + int64_t(m - 1) * n;
    const int relocate = n_empty > 0 && dist[s_far[0]] > 0.0 ? n_empty : 0;   // all rows on their centres: none
    for (int e = 0; e < relocate; ++e) {
      const int knew = s_empty[1 + e];
      const int64_t i = s_far[e];
      const int kold = labels[i];
      for (int j = 0; j < d; ++j) {
        s_sum[kold * (d + 1) + j] -= xc[i * d + j];
        s_sum[knew * (d + 1) + j] = xc[i * d + j];
      }
      s_sum[knew * (d + 1) + d] = 1.0;
      s_sum[kold * (d + 1) + d] -= 1.0;
    }
    int big = 0;                                       // the heaviest cluster, the first on a tie
    for (int k = 1; k < m; ++k)
      if (s_sum[k * (d + 1) + d] > s_sum[big * (d + 1) + d]) big = k;
    for (int k = 0; k < m; ++k) {                      // in cluster order: an empty cluster before `big` copies its sum
      const double w = s_sum[k * (d + 1) + d];
      for (int j = 0; j < d; ++j)
        s_sum[k * (d + 1) + j] = w > 0.0 ? s_sum[k * (d + 1) + j] * (1.0 / w) : s_sum[big * (d + 1) + j];
    }
    double shift = 0.0;
    double* c = centres + int64_t(off) * d;
    for (int k = 0; k < m; ++k) {
      double sk = 0.0;
      for (int j = 0; j < d; ++j) {
        const double t = s_sum[k * (d + 1) + j] - c[k * d + j];
        sk += t * t;
        c[k * d + j] = s_sum[k * (d + 1) + j];
      }
      const double norm = sqrt(sk);
      shift += norm * norm;
    }
    int changed = 0;
    for (int r = 0; r < R; ++r) changed += lchg[int64_t(r) * M + (m - 1)];
    if (changed == 0) st->lloyd_strict = 1;
    if (changed == 0 || shift <= glob[kGmmMaxD] || iter + 1 == kGmmLloydIters) {
      st->lloyd_done = 1;
      st->lloyd_iters = iter + 1;
    }
  }
}

// mu = k-means centre + column mean: the first shift of the EM statistics
__global__ void __launch_bounds__(kGmmThreads) gmm_em_setup_kernel(int d, int comps, const double* __restrict__ glob,
                                                                   const double* __restrict__ centres,
                                                                   double* __restrict__ mu) {
  const int e = int(blockIdx.x) * kGmmThreads + int(threadIdx.x);
  if (e < comps * d) mu[e] = centres[e] + glob[e % d];
}

// log N(x | mu_k, Sigma_k) + log w_k with W_k = L_k^-1 (lower, packed by rows): y = W_k (x - mu_k),
// value = cst_k - |y|^2 / 2, cst_k = log w_k + sum_j log W_jj - d log(2 pi) / 2.
__device__ __forceinline__ double gmm_log_prob(const double* xr, const double* __restrict__ mu,
                                               const double* __restrict__ w, double cst, int d) {
  double diff[kGmmMaxD];
#pragma unroll
  for (int i = 0; i < kGmmMaxD; ++i) diff[i] = i < d ? xr[i] - __ldg(mu + i) : 0.0;
  double sq = 0.0;
  int e = 0;
#pragma unroll
  for (int j = 0; j < kGmmMaxD; ++j) {
    if (j < d) {
      double y = 0.0;
#pragma unroll
      for (int i = 0; i <= j; ++i) y += __ldg(w + e + i) * diff[i];
      e += j + 1;
      sq += y * y;
    }
  }
  return cst - 0.5 * sq;
}

// Block b: model m = b / R + 1 and row chunk r = b % R (kGmmResp: m = *best, r = b), tiles of kGmmTile rows.
//   kGmmInit   r = one-hot k-means labels, shift = mu (the k-means centres) -> statistics
//   kGmmStep   r = responsibilities of the current parameters -> statistics and the chunk's sum of log-likelihoods
//   kGmmScore  the chunk's sum of log-likelihoods only, for every model (the BIC)
//   kGmmResp   out[i][k] = r_ik for the winner
// Statistics [R][C][S]: for component k, S = 1 + d + d(d+1)/2 sums over the chunk's rows (row order within a tile,
// tile order within the chunk): r, r (x - s), r (x - s)_i (x - s)_j for i <= j.
__global__ void __launch_bounds__(kGmmThreads) gmm_em_stats_kernel(
    const double* __restrict__ x, int64_t n, int d, int M, int R, int64_t chunk_rows, int mode,
    const GmmState* __restrict__ state, const int32_t* __restrict__ best, const int32_t* __restrict__ labels_all,
    const double* __restrict__ mu_all, const double* __restrict__ prec_all, const double* __restrict__ cst_all,
    double* __restrict__ esum, double* __restrict__ lse_part, double* __restrict__ out_resp) {
  CRAG_DYNAMIC_SHARED(double, s_mem);
  int m, r;
  if (mode == kGmmResp) { m = *best; r = int(blockIdx.x); }
  else { m = int(blockIdx.x) / R + 1; r = int(blockIdx.x) % R; }
  if (mode == kGmmStep && state[m - 1].em_done) return;
  const int tid = int(threadIdx.x), warp = tid >> 5, lane = tid & 31;
  const int S = 1 + d + gmm_tri(d), off = gmm_comp_off(m), comps = gmm_comp_off(M + 1);
  double* s_r = s_mem;                                 // [kGmmTile][m]: log-probabilities, then responsibilities
  double* s_x = s_r + kGmmTile * m;                    // [kGmmTile][d]
  const bool stats = mode == kGmmInit || mode == kGmmStep;
  double* part = esum + (int64_t(r) * comps + off) * S;
  const int tasks = m * S;
  if (stats)
    for (int t = tid; t < tasks; t += kGmmThreads) part[t] = 0.0;
  const int32_t* labels = labels_all + int64_t(m - 1) * n;
  const int64_t row0 = int64_t(r) * chunk_rows, row1 = gmm_min64(row0 + chunk_rows, n);
  double lse_acc = 0.0;                                // warp 0, lane p: the log-likelihoods of its rows
  for (int64_t t0 = row0; t0 < row1; t0 += kGmmTile) {
    const int rows = int(gmm_min64(kGmmTile, row1 - t0));
    for (int e = tid; e < rows * d; e += kGmmThreads) s_x[e] = x[t0 * d + e];
    __syncthreads();
    if (mode == kGmmInit) {
      for (int e = tid; e < rows * m; e += kGmmThreads) s_r[e] = labels[t0 + e / m] == e % m ? 1.0 : 0.0;
    } else if (lane < rows) {
      double xr[kGmmMaxD];
#pragma unroll
      for (int i = 0; i < kGmmMaxD; ++i) xr[i] = i < d ? s_x[lane * d + i] : 0.0;
      for (int k = warp; k < m; k += kGmmThreads / 32) {
        const int c = off + k;
        s_r[lane * m + k] = gmm_log_prob(xr, mu_all + int64_t(c) * d, prec_all + int64_t(c) * gmm_tri(d),
                                         __ldg(cst_all + c), d);
      }
    }
    __syncthreads();
    if (mode != kGmmInit && warp == 0 && lane < rows) {
      double* lp = s_r + lane * m;
      double mx = lp[0];
      for (int k = 1; k < m; ++k) mx = fmax(mx, lp[k]);
      double s = 0.0;
      for (int k = 0; k < m; ++k) s += exp(lp[k] - mx);
      const double lse = mx + log(s);
      lse_acc += lse;
      for (int k = 0; k < m; ++k) lp[k] = exp(lp[k] - lse);
      if (mode == kGmmResp)
        for (int k = 0; k < m; ++k) out_resp[(t0 + lane) * m + k] = lp[k];
    }
    __syncthreads();
    if (stats) {
      for (int t = tid; t < tasks; t += kGmmThreads) {
        const int k = t / S, s = t % S;
        const double* sh = mu_all + int64_t(off + k) * d;
        double acc = 0.0;
        if (s == 0) {
          for (int p = 0; p < rows; ++p) acc += s_r[p * m + k];
        } else if (s <= d) {
          const int i = s - 1;
          const double si = sh[i];
          for (int p = 0; p < rows; ++p) acc += s_r[p * m + k] * (s_x[p * d + i] - si);
        } else {
          int q = s - 1 - d, i = 0;                    // (i, j), i <= j, packed by rows of the upper triangle
          while (q >= d - i) { q -= d - i; ++i; }
          const int j = i + q;
          const double si = sh[i], sj = sh[j];
          for (int p = 0; p < rows; ++p) acc += s_r[p * m + k] * ((s_x[p * d + i] - si) * (s_x[p * d + j] - sj));
        }
        part[t] += acc;
      }
    }
    __syncthreads();
  }
  if (mode == kGmmInit || mode == kGmmResp) return;
  if (warp == 0) {
    const double total = gmm_warp_sum(lse_acc);
    if (lane == 0) lse_part[int64_t(r) * M + (m - 1)] = total;
  }
}

// Cholesky A = L L^T of the d x d matrix whose row i lane i holds in a[] (lanes >= d hold nothing), then W = L^-1;
// lane i returns row i of W in w[].  false if a pivot is not positive (A not positive definite).
__device__ __forceinline__ bool gmm_warp_chol_inverse(double (&a)[kGmmMaxD], double (&w)[kGmmMaxD], int d, int lane) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j < kGmmMaxD; ++j) {
    if (j < d) {
      const double pivot = __shfl_sync(0xffffffffu, a[j], j);
      ok = ok && pivot > 0.0;
      const double ljj = sqrt(pivot);
      if (lane == j) a[j] = ljj;
      else if (lane > j) a[j] = a[j] / ljj;
#pragma unroll
      for (int k = j + 1; k < kGmmMaxD; ++k) {
        const double lkj = __shfl_sync(0xffffffffu, a[j], k);
        if (k < d && lane >= k && lane > j) a[k] -= a[j] * lkj;
      }
    }
  }
  // forward substitution, row by row: W[i][c] = (delta_ic - sum_{k<i} L[i][k] W[k][c]) / L[i][i]
  double acc[kGmmMaxD];
#pragma unroll
  for (int c = 0; c < kGmmMaxD; ++c) acc[c] = 0.0, w[c] = 0.0;
#pragma unroll
  for (int k = 0; k < kGmmMaxD; ++k) {
    if (k < d) {
      if (lane == k) {
#pragma unroll
        for (int c = 0; c <= k; ++c) w[c] = ((c == k ? 1.0 : 0.0) - acc[c]) / a[k];
      }
#pragma unroll
      for (int c = 0; c <= k; ++c) {
        const double wkc = __shfl_sync(0xffffffffu, w[c], k);
        if (lane > k && lane < d) acc[c] += a[k] * wkc;
      }
    }
  }
  return ok;
}

// One block per model.  kGmmInit: the M-step of the one-hot k-means responsibilities (weights nk / n).  kGmmStep,
// iteration `iter`: lower bound = (sum of the chunks' log-likelihood sums) / n, then the M-step (weights nk / sum nk),
// then done when |lower bound - previous| < tol or iter == kGmmEmIters.  Warp w handles components w, w + 8, ...
//   nk = sum r + 10 eps,  delta = sum r (x - s) / nk,  mu' = s + delta,
//   Sigma = (sum r (x - s)(x - s)^T - (sum r + 20 eps) delta delta^T) / nk + reg_covar I
// (= sum r (x - mu')(x - mu')^T / nk + reg_covar I, with s = the old mean, so nothing cancels near convergence).
__global__ void __launch_bounds__(kGmmThreads) gmm_mstep_kernel(
    int64_t n, int d, int M, int R, int mode, int iter, GmmState* __restrict__ state, double* __restrict__ mu_all,
    double* __restrict__ prec_all, double* __restrict__ cst_all, double* __restrict__ wt_all,
    const double* __restrict__ esum,
    const double* __restrict__ lse_part) {
  CRAG_DYNAMIC_SHARED(double, s_mem);
  const int m = int(blockIdx.x) + 1, tid = int(threadIdx.x), warp = tid >> 5, lane = tid & 31;
  GmmState* st = state + (m - 1);
  if (mode == kGmmStep && st->em_done) return;
  const int S = 1 + d + gmm_tri(d), off = gmm_comp_off(m), comps = gmm_comp_off(M + 1), T = gmm_tri(d);
  double* s_st = s_mem + warp * S;                     // [8][S] the warp's component statistics
  double* s_nk = s_mem + (kGmmThreads / 32) * S;       // [m]
  double* s_logdet = s_nk + kGmmMaxM;                  // [m]
  int* s_bad = reinterpret_cast<int*>(s_logdet + kGmmMaxM);
  if (tid == 0) *s_bad = 0;
  __syncthreads();
  for (int k = warp; k < m; k += kGmmThreads / 32) {
    const int c = off + k;
    for (int s = lane; s < S; s += 32) {
      double acc = 0.0;
      for (int r = 0; r < R; ++r) acc += esum[(int64_t(r) * comps + c) * S + s];
      s_st[s] = acc;
    }
    __syncwarp();
    const double a = s_st[0], nk = a + kGmmEps10;
    double* mu = mu_all + int64_t(c) * d;
    double delta_i = 0.0, a_row[kGmmMaxD], w_row[kGmmMaxD];
    if (lane < d) delta_i = s_st[1 + lane] / nk;
#pragma unroll
    for (int j = 0; j < kGmmMaxD; ++j) {
      const double delta_j = __shfl_sync(0xffffffffu, delta_i, j);
      double v = 0.0;
      if (lane < d && j < d) {
        const int i0 = lane < j ? lane : j, j0 = lane < j ? j : lane;
        const int q = i0 * d - i0 * (i0 - 1) / 2 + (j0 - i0);
        v = (s_st[1 + d + q] - (a + 2 * kGmmEps10) * delta_i * delta_j) / nk;
        if (j == lane) v += kGmmRegCovar;
      }
      a_row[j] = v;
    }
    __syncwarp();
    const bool ok = gmm_warp_chol_inverse(a_row, w_row, d, lane);
    double logdet = 0.0;
#pragma unroll
    for (int j = 0; j < kGmmMaxD; ++j) {
      const double wjj = __shfl_sync(0xffffffffu, w_row[j], j);
      if (j < d) logdet += log(wjj);
    }
    if (lane < d) {
      mu[lane] = mu[lane] + delta_i;
      double* wp = prec_all + int64_t(c) * T + lane * (lane + 1) / 2;
      for (int i = 0; i <= lane; ++i) wp[i] = w_row[i];
    }
    if (lane == 0) {
      s_nk[k] = nk;
      s_logdet[k] = logdet;
      if (!ok) *s_bad = 1;
    }
    __syncwarp();
  }
  __syncthreads();
  if (tid == 0) {
    double norm = double(n);
    if (mode == kGmmStep) {
      norm = 0.0;
      for (int k = 0; k < m; ++k) norm += s_nk[k];
    }
    for (int k = 0; k < m; ++k) {
      const double w = s_nk[k] / norm;
      wt_all[off + k] = w;
      cst_all[off + k] = log(w) + s_logdet[k] - 0.5 * d * kGmmLog2Pi;
    }
    if (*s_bad) {
      st->em_done = 1;
      st->em_converged = -1;
      st->em_iters = iter;
    } else if (mode == kGmmStep) {
      double ll = 0.0;
      for (int r = 0; r < R; ++r) ll += lse_part[int64_t(r) * M + (m - 1)];
      const double lb = ll / double(n);
      const bool conv = fabs(lb - st->lower_bound) < kGmmEmTol;
      st->lower_bound = lb;
      if (conv || iter == kGmmEmIters) {
        st->em_done = 1;
        st->em_iters = iter;
        st->em_converged = conv ? 1 : 0;
      }
    }
  }
}

// One block, one thread per model: BIC_m = -2 n mean(log-likelihood) + p_m ln n on the final parameters
// (p_m = m d(d+1)/2 + m d + m - 1); best = the first argmin (1-based); the winner's weights and means.
__global__ void __launch_bounds__(kGmmMaxM) gmm_select_kernel(
    int64_t n, int d, int M, int R, const GmmState* __restrict__ state, const double* __restrict__ mu_all,
    const double* __restrict__ wt_all, const double* __restrict__ lse_part,
    double* __restrict__ out_bic, int32_t* __restrict__ out_iters, int32_t* __restrict__ out_converged,
    int32_t* __restrict__ best, double* __restrict__ out_weights, double* __restrict__ out_means) {
  CRAG_DYNAMIC_SHARED(double, s_bic);
  const int tid = int(threadIdx.x);
  if (tid < M) {
    const int m = tid + 1;
    double ll = 0.0;
    for (int r = 0; r < R; ++r) ll += lse_part[int64_t(r) * M + tid];
    const double p = double(m) * d * (d + 1) / 2.0 + double(m) * d + m - 1;
    const double bic = -2.0 * (ll / double(n)) * double(n) + p * log(double(n));
    s_bic[tid] = bic;
    out_bic[tid] = bic;
    out_iters[tid] = state[tid].em_iters;
    out_converged[tid] = state[tid].em_converged;
  }
  __syncthreads();
  if (tid == 0) {
    int b = 0;
    for (int k = 1; k < M; ++k)
      if (s_bic[k] < s_bic[b]) b = k;
    *best = b + 1;
    s_bic[kGmmMaxM] = double(b + 1);
  }
  __syncthreads();
  const int m = int(s_bic[kGmmMaxM]), off = gmm_comp_off(m);
  if (tid < m) {
    out_weights[tid] = wt_all[off + tid];
    for (int j = 0; j < d; ++j) out_means[tid * d + j] = mu_all[int64_t(off + tid) * d + j];
  }
}

}  // namespace
}  // namespace crag
