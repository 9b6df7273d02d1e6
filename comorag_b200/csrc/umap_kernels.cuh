// UMAP on the device for ComoRAG's soft clustering (ChunkSoftClustering._reduce_dimensions, cluster_utils.py:191-211):
// the kernels of crag_umap_fuzzy_graph, crag_umap_spectral_init and crag_umap_optimize (umap.cu).  DESIGN.md section 2c
// states the semantics; in short, umap-learn 0.5's defaults with three named departures (a subspace-iteration spectral
// start, no multi-component meta-layout, and layout epochs in which every vertex moves from its own current position
// against a snapshot of the others):
//   umap_knn_lists_kernel     one warp per row: the self rule on crag_knn_topk's lists, distances 1 - score, row sums
//   umap_mean_kernel          one block: the mean of all distances, a fixed tree
//   umap_smooth_kernel        one warp per row: rho, the 64-step sigma bisection, memberships
//   umap_degree_kernel        degrees and D^-1/2 of the symmetric CSR graph
//   umap_basis_kernel         the start block: D^1/2 1 and counter-hash columns (the identity for n <= 16)
//   umap_spmm_kernel          W = S' V,  S' = (I + D^-1/2 G D^-1/2) / 2,  one thread per (row, column)
//   umap_gram_kernel          per-chunk partial A^T B (p x p), one thread per entry, rows in order
//   umap_cholqr_kernel        one block: partials summed in chunk order, Cholesky, R^-1
//   umap_apply_r_kernel       V = W R^-1
//   umap_ritz_kernel          one block: H = V^T S' V, cyclic Jacobi, eigenpairs by descending eigenvalue
//   umap_ritz_vectors_kernel  Ritz vectors 2..d+1
//   umap_post_kernel          one block: sign fix, scale to 10 / max|Y|, noise 1e-4, min-max rescale to [0, 10]
//   umap_epoch_kernel         one thread per vertex: one layout epoch, read from the snapshot, write the other buffer
// Every sum runs in an order fixed by the shapes, and nothing uses atomics, so the same input gives the same bits on
// any run and stream.  Pure SIMT code, so tests/warp_emu runs this very header on emulated blocks.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

#include "workspace.cuh"

#ifndef CRAG_EMULATED_PTX
#define CRAG_DYNAMIC_SHARED(type, name) extern __shared__ type name[]
#endif

namespace crag {
namespace {

constexpr int kUmapMaxD = 16;
constexpr int kUmapMaxK = 256;                 // n_neighbors
constexpr int kUmapMaxP = 17;                  // subspace columns: max(16, d + 1), at most n
constexpr int kUmapThreads = 128;
constexpr int kUmapGramThreads = 320;          // >= kUmapMaxP^2, a whole number of warps
constexpr int kUmapChunkRows = 1024;           // rows per Gram chunk, until there are kUmapMaxChunks chunks
constexpr int kUmapMaxChunks = 64;
constexpr int kUmapBisect = 64;
constexpr int kUmapJacobiSweeps = 30;
constexpr double kUmapSmoothTol = 1e-5;
constexpr double kUmapMinScale = 1e-3;
constexpr double kUmapNegRate = 5.0;
constexpr float kUmapGamma = 1.0f;
// counter-hash streams besides the epochs (which use the epoch number): start columns and start noise
constexpr uint64_t kUmapStreamBasis = 0xFFFFFFFF00000001ull;
constexpr uint64_t kUmapStreamNoise = 0xFFFFFFFF00000002ull;

__host__ __device__ __forceinline__ uint64_t umap_mix(uint64_t z) {      // splitmix64's finaliser
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// the stateless counter hash of (seed, stream, a, b)
__host__ __device__ __forceinline__ uint64_t umap_hash(uint64_t seed, uint64_t stream, uint64_t a, uint64_t b) {
  return umap_mix(umap_mix(umap_mix(umap_mix(seed) ^ stream) ^ a) ^ b);
}
__host__ __device__ __forceinline__ double umap_unit(uint64_t h) {       // (0, 1]
  return double((h >> 11) + 1) * (1.0 / 9007199254740992.0);
}

__host__ __device__ inline int umap_p(int64_t n, int d) {
  const int p = d + 1 > 16 ? d + 1 : 16;
  return int(n < p ? n : p);
}

// Workspace of the fuzzy graph: the rows' distance sums [n] and their mean (fp64).
struct UmapFuzzyWorkspace { double *rowsum, *mean; size_t total; };
inline UmapFuzzyWorkspace umap_fuzzy_workspace(int64_t n, void* ws = nullptr) {
  WsCursor c(ws);
  UmapFuzzyWorkspace w;
  w.rowsum = c.take<double>(size_t(n));
  w.mean = c.take<double>(1);
  w.total = c.bytes;
  return w;
}

// The spectral start.  Workspace `ws`: degrees and D^-1/2 [n], V and W [n][p], Gram partials [chunks][p][p], R^-1
// [p][p], eigenvectors + eigenvalues [p][p] + [p], Ritz vectors [n][d] (fp64 throughout).
struct UmapSpectralPlan {
  int p, chunks;
  int64_t chunk_rows;
  double *deg, *dis, *v, *w, *part, *rinv, *q, *yr;   // the workspace's regions (null when only sized)
  size_t total;                                        // workspace bytes
};
inline UmapSpectralPlan plan_umap_spectral(int64_t n, int d, void* ws = nullptr) {
  UmapSpectralPlan s;
  s.p = umap_p(n, d);
  const int64_t want = (n + kUmapChunkRows - 1) / kUmapChunkRows;
  s.chunks = int(want < 1 ? 1 : want > kUmapMaxChunks ? kUmapMaxChunks : want);
  s.chunk_rows = (n + s.chunks - 1) / s.chunks;
  const size_t P = size_t(s.p), N = size_t(n);
  WsCursor c(ws);
  s.deg = c.take<double>(N);
  s.dis = c.take<double>(N);
  s.v = c.take<double>(N * P);
  s.w = c.take<double>(N * P);
  s.part = c.take<double>(size_t(s.chunks) * P * P);
  s.rinv = c.take<double>(P * P);
  s.q = c.take<double>(P * P + P);
  s.yr = c.take<double>(N * size_t(d));
  s.total = c.bytes;
  return s;
}

// Workspace of the layout: the second layout buffer [n][d].
struct UmapOptimizeWorkspace { float* other; size_t total; };
inline UmapOptimizeWorkspace umap_optimize_workspace(int64_t n, int d, void* ws = nullptr) {
  WsCursor c(ws);
  UmapOptimizeWorkspace w;
  w.other = c.take<float>(size_t(n) * size_t(d));
  w.total = c.bytes;
  return w;
}

// The schedule counters advance as umap-learn's do, a product then a sum, never contracted into one fma.
#ifdef CRAG_EMULATED_PTX
inline double umap_mul_rn(double x, double y) { return x * y; }
#else
__device__ __forceinline__ double umap_mul_rn(double x, double y) { return __dmul_rn(x, y); }
#endif

__device__ __forceinline__ double umap_warp_sum(double v) {          // fixed butterfly: every lane gets the same bits
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------- fuzzy simplicial set
// One warp per row i.  The search returned k entries (score desc, row asc); the list is i itself at distance 0, then
// the k - 1 best other rows: i's own entry is removed where the search returned it, otherwise the last is dropped.
__global__ void __launch_bounds__(kUmapThreads) umap_knn_lists_kernel(const int64_t* __restrict__ ids,
                                                                      const float* __restrict__ scores, int64_t n,
                                                                      int k, int32_t* __restrict__ nbr,
                                                                      float* __restrict__ dist,
                                                                      double* __restrict__ rowsum) {
  const int lane = int(threadIdx.x) & 31;
  const int64_t i = int64_t(blockIdx.x) * (kUmapThreads / 32) + int64_t(threadIdx.x) / 32;
  if (i >= n) return;
  const int64_t* id = ids + i * k;
  const float* sc = scores + i * k;
  int q = k;                                   // position of i in the search's list (k: absent)
  float self_d = 0.0f;
  for (int t = 0; t < k; t += 32) {
    const int j = t + lane;
    const unsigned hit = __ballot_sync(0xffffffffu, j < k && id[j] == i);
    if (hit) {
      q = t + __ffs(hit) - 1;
      break;
    }
  }
  if (q < k) self_d = 0.0f;                    // pinned: bf16 rounding leaves a row's self-score below 1
  double part = 0.0;
  for (int j = lane; j < k; j += 32) {
    int32_t col;
    float dj;
    if (j == 0) {
      col = int32_t(i);
      dj = self_d;
    } else {
      const int src = j - 1 < q ? j - 1 : j;
      col = int32_t(id[src]);
      dj = fmaxf(0.0f, 1.0f - sc[src]);
    }
    nbr[i * k + j] = col;
    dist[i * k + j] = dj;
    part += double(dj);
  }
  part = umap_warp_sum(part);
  if (lane == 0) rowsum[i] = part;
}

// One block of 1024 threads: mean of all n * k distances; strided partials, then a fixed tree.
__global__ void __launch_bounds__(1024) umap_mean_kernel(const double* __restrict__ rowsum, int64_t n, int k,
                                                         double* __restrict__ mean) {
  CRAG_DYNAMIC_SHARED(double, s_red);
  double v = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) v += rowsum[i];
  s_red[threadIdx.x] = v;
  __syncthreads();
  for (int w = int(blockDim.x) / 2; w > 0; w >>= 1) {
    if (int(threadIdx.x) < w) s_red[threadIdx.x] = s_red[threadIdx.x] + s_red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) mean[0] = s_red[0] / (double(n) * double(k));
}

// One warp per row: rho = the first nonzero distance; sigma by bisection toward sum_{j>=1} f(d_j - rho) = log2(k);
// the floor; memberships mu_ij (0 on i itself, 1 within rho, exp(-(d - rho) / sigma) beyond).
__global__ void __launch_bounds__(kUmapThreads) umap_smooth_kernel(const int32_t* __restrict__ nbr,
                                                                   const float* __restrict__ dist,
                                                                   const double* __restrict__ rowsum,
                                                                   const double* __restrict__ mean, int64_t n, int k,
                                                                   float* __restrict__ rho_out,
                                                                   float* __restrict__ sigma_out,
                                                                   float* __restrict__ memb) {
  const int lane = int(threadIdx.x) & 31;
  const int64_t i = int64_t(blockIdx.x) * (kUmapThreads / 32) + int64_t(threadIdx.x) / 32;
  if (i >= n) return;
  const float* di = dist + i * k;
  float rho = 0.0f;
  for (int t = 0; t < k; t += 32) {
    const int j = t + lane;
    const unsigned nz = __ballot_sync(0xffffffffu, j < k && di[j] > 0.0f);
    if (nz) {
      rho = di[t + __ffs(nz) - 1];
      break;
    }
  }
  const double target = log2(double(k));
  double lo = 0.0, hi = INFINITY, mid = 1.0;
  for (int it = 0; it < kUmapBisect; ++it) {
    double part = 0.0;
    for (int j = 1 + lane; j < k; j += 32) {
      const double x = double(di[j]) - double(rho);
      part += x > 0.0 ? exp(-(x / mid)) : 1.0;
    }
    const double psum = umap_warp_sum(part);
    if (fabs(psum - target) < kUmapSmoothTol) break;
    if (psum > target) {
      hi = mid;
      mid = (lo + hi) / 2.0;
    } else {
      lo = mid;
      if (hi == INFINITY) mid *= 2.0;
      else mid = (lo + hi) / 2.0;
    }
  }
  double sigma = mid;
  const double floor_ = kUmapMinScale * (rho > 0.0f ? rowsum[i] / double(k) : mean[0]);
  if (sigma < floor_) sigma = floor_;
  for (int j = lane; j < k; j += 32) {
    const double x = double(di[j]) - double(rho);
    float mu;
    if (nbr[i * k + j] == int32_t(i)) mu = 0.0f;
    else if (x <= 0.0 || sigma == 0.0) mu = 1.0f;
    else mu = float(exp(-(x / sigma)));
    memb[i * k + j] = mu;
  }
  if (lane == 0) {
    rho_out[i] = rho;
    sigma_out[i] = float(sigma);
  }
}

// ----------------------------------------------------------------------------------------------- spectral start
__global__ void __launch_bounds__(kUmapThreads) umap_degree_kernel(const int64_t* __restrict__ indptr,
                                                                   const float* __restrict__ w, int64_t n,
                                                                   double* __restrict__ deg, double* __restrict__ dis) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int64_t e = indptr[i]; e < indptr[i + 1]; ++e) s += double(w[e]);
  deg[i] = s;
  dis[i] = s > 0.0 ? 1.0 / sqrt(s) : 0.0;
}

// V [n][p]: column 0 = D^1/2 1, the others uniform in [-1, 1) from the counter hash; the identity when n <= 16 (p = n:
// Rayleigh-Ritz on the whole space).
__global__ void __launch_bounds__(kUmapThreads) umap_basis_kernel(const double* __restrict__ deg, int64_t n, int p,
                                                                  uint64_t seed, double* __restrict__ v) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n * p) return;
  const int64_t i = t / p;
  const int c = int(t % p);
  double x;
  if (n <= 16) x = (i == c) ? 1.0 : 0.0;
  else if (c == 0) x = sqrt(deg[i]);
  else x = 2.0 * umap_unit(umap_hash(seed, kUmapStreamBasis, uint64_t(i), uint64_t(c))) - 1.0;
  v[t] = x;
}

// W = S' V, one thread per (row, column), the row's edges in column order.
__global__ void __launch_bounds__(kUmapThreads) umap_spmm_kernel(const int64_t* __restrict__ indptr,
                                                                 const int32_t* __restrict__ col,
                                                                 const float* __restrict__ w,
                                                                 const double* __restrict__ dis, int64_t n, int p,
                                                                 const double* __restrict__ v, double* __restrict__ out) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n * p) return;
  const int64_t i = t / p;
  const int c = int(t % p);
  double s = 0.0;
  for (int64_t e = indptr[i]; e < indptr[i + 1]; ++e) {
    const int64_t j = col[e];
    s += double(w[e]) * dis[j] * v[j * p + c];
  }
  out[t] = 0.5 * (v[t] + dis[i] * s);
}

// Block r: part[r][a][b] = sum over the chunk's rows, in order, of A[i][a] * B[i][b].
__global__ void __launch_bounds__(kUmapGramThreads) umap_gram_kernel(const double* __restrict__ A,
                                                                     const double* __restrict__ B, int64_t n, int p,
                                                                     int64_t chunk_rows, double* __restrict__ part) {
  const int r = int(blockIdx.x);
  const int t = int(threadIdx.x);
  if (t >= p * p) return;
  const int a = t / p, b = t % p;
  const int64_t lo = int64_t(r) * chunk_rows;
  const int64_t hi = lo + chunk_rows < n ? lo + chunk_rows : n;
  double s = 0.0;
  for (int64_t i = lo; i < hi; ++i) s += A[i * p + a] * B[i * p + b];
  part[int64_t(r) * p * p + t] = s;
}

// One block: G = sum of the chunk partials in chunk order; G = L L^T; rinv = L^-T (upper).  A pivot that is not
// positive (a column dependent on the earlier ones) drops its column.
__global__ void __launch_bounds__(32) umap_cholqr_kernel(const double* __restrict__ part, int chunks, int p,
                                                         double* __restrict__ rinv) {
  __shared__ double g[kUmapMaxP * kUmapMaxP];
  __shared__ double li[kUmapMaxP * kUmapMaxP];
  for (int t = int(threadIdx.x); t < p * p; t += 32) {
    double s = 0.0;
    for (int r = 0; r < chunks; ++r) s += part[int64_t(r) * p * p + t];
    g[t] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double dmax = 0.0;
    for (int c = 0; c < p; ++c) dmax = g[c * p + c] > dmax ? g[c * p + c] : dmax;
    for (int c = 0; c < p; ++c) {                 // in place: g's lower triangle becomes L
      double s = g[c * p + c];
      for (int m = 0; m < c; ++m) s -= g[c * p + m] * g[c * p + m];
      const bool ok = s > 1e-28 * dmax;
      const double l = ok ? sqrt(s) : 0.0;
      g[c * p + c] = l;
      for (int r = c + 1; r < p; ++r) {
        double x = g[r * p + c];
        for (int m = 0; m < c; ++m) x -= g[r * p + m] * g[c * p + m];
        g[r * p + c] = ok ? x / l : 0.0;
      }
    }
    for (int c = 0; c < p; ++c) {                 // L^-1 by forward substitution, column c
      for (int r = 0; r < p; ++r) {
        double x;
        if (r < c) x = 0.0;
        else {
          x = (r == c) ? 1.0 : 0.0;
          for (int m = c; m < r; ++m) x -= g[r * p + m] * li[m * p + c];
          x = g[r * p + r] > 0.0 ? x / g[r * p + r] : 0.0;
        }
        li[r * p + c] = x;
      }
    }
    for (int r = 0; r < p; ++r)
      for (int c = 0; c < p; ++c) rinv[r * p + c] = li[c * p + r];
  }
}

// V = W R^-1 (R^-1 upper triangular), one thread per (row, column).
__global__ void __launch_bounds__(kUmapThreads) umap_apply_r_kernel(const double* __restrict__ w,
                                                                    const double* __restrict__ rinv, int64_t n, int p,
                                                                    double* __restrict__ v) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n * p) return;
  const int64_t i = t / p;
  const int c = int(t % p);
  double s = 0.0;
  for (int m = 0; m <= c; ++m) s += w[i * p + m] * rinv[m * p + c];
  v[t] = s;
}

// One block: H = sum of the chunk partials of V^T (S' V), symmetrised; cyclic Jacobi with a fixed sweep count; q =
// eigenvectors (columns) by descending eigenvalue (ties by index), q[p * p + c] = the eigenvalues.
__global__ void __launch_bounds__(32) umap_ritz_kernel(const double* __restrict__ part, int chunks, int p,
                                                       double* __restrict__ q) {
  __shared__ double h[kUmapMaxP * kUmapMaxP];
  __shared__ double z[kUmapMaxP * kUmapMaxP];
  for (int t = int(threadIdx.x); t < p * p; t += 32) {
    double s = 0.0;
    for (int r = 0; r < chunks; ++r) s += part[int64_t(r) * p * p + t];
    h[t] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int a = 0; a < p; ++a)
    for (int b = a + 1; b < p; ++b) {
      const double m = 0.5 * (h[a * p + b] + h[b * p + a]);
      h[a * p + b] = m;
      h[b * p + a] = m;
    }
  for (int t = 0; t < p * p; ++t) z[t] = (t / p == t % p) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < kUmapJacobiSweeps; ++sweep)
    for (int a = 0; a < p - 1; ++a)
      for (int b = a + 1; b < p; ++b) {
        const double apq = h[a * p + b];
        if (apq == 0.0) continue;
        const double theta = (h[b * p + b] - h[a * p + a]) / (2.0 * apq);
        const double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double cs = 1.0 / sqrt(tt * tt + 1.0), sn = tt * cs;
        for (int m = 0; m < p; ++m) {            // H = J^T H J, columns a and b
          const double ha = h[m * p + a], hb = h[m * p + b];
          h[m * p + a] = cs * ha - sn * hb;
          h[m * p + b] = sn * ha + cs * hb;
        }
        for (int m = 0; m < p; ++m) {            // rows a and b
          const double ha = h[a * p + m], hb = h[b * p + m];
          h[a * p + m] = cs * ha - sn * hb;
          h[b * p + m] = sn * ha + cs * hb;
        }
        h[a * p + b] = 0.0;
        h[b * p + a] = 0.0;
        for (int m = 0; m < p; ++m) {            // Z = Z J
          const double za = z[m * p + a], zb = z[m * p + b];
          z[m * p + a] = cs * za - sn * zb;
          z[m * p + b] = sn * za + cs * zb;
        }
      }
  int order[kUmapMaxP];
  for (int c = 0; c < p; ++c) order[c] = c;
  for (int c = 1; c < p; ++c) {                  // insertion sort: descending eigenvalue, ties by index
    const int x = order[c];
    int m = c;
    while (m > 0 && h[order[m - 1] * p + order[m - 1]] < h[x * p + x]) {
      order[m] = order[m - 1];
      --m;
    }
    order[m] = x;
  }
  for (int c = 0; c < p; ++c) {
    for (int m = 0; m < p; ++m) q[m * p + c] = z[m * p + order[c]];
    q[p * p + c] = h[order[c] * p + order[c]];
  }
}

// yr[i][c] = sum_m V[i][m] q[m][c + 1]: the Ritz vectors of the 2nd .. (d+1)th eigenvalues.
__global__ void __launch_bounds__(kUmapThreads) umap_ritz_vectors_kernel(const double* __restrict__ v,
                                                                         const double* __restrict__ q, int64_t n, int p,
                                                                         int d, double* __restrict__ yr) {
  const int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n * d) return;
  const int64_t i = t / d;
  const int c = int(t % d);
  double s = 0.0;
  for (int m = 0; m < p; ++m) s += v[i * p + m] * q[m * p + c + 1];
  yr[t] = s;
}

// One block of 1024 threads (min / max are exact in any order; ties of |.| go to the lower row):
//   the sign of each column makes its largest-magnitude entry positive (written back to yr);
//   E = fp32(yr * 10 / max|yr|) + fp32(1e-4 * N(0, 1) from the counter hash);
//   y = 10 * (E - min_col E) / (max_col E - min_col E), in fp32.
__global__ void __launch_bounds__(1024) umap_post_kernel(double* __restrict__ yr, int64_t n, int d, uint64_t seed,
                                                         float* __restrict__ y) {
  __shared__ double s_v[1024];
  __shared__ int64_t s_i[1024];
  __shared__ float s_lo[1024], s_hi[1024];
  __shared__ double s_sign[kUmapMaxD];
  __shared__ float s_min[kUmapMaxD], s_max[kUmapMaxD];
  __shared__ double s_expand, s_absmax;
  const int tid = int(threadIdx.x);
  for (int c = 0; c < d; ++c) {
    double best = -1.0;
    int64_t at = n;
    for (int64_t i = tid; i < n; i += 1024) {
      const double a = fabs(yr[i * d + c]);
      if (a > best) { best = a; at = i; }
    }
    s_v[tid] = best;
    s_i[tid] = at;
    __syncthreads();
    if (tid == 0) {
      for (int t = 1; t < 1024; ++t)
        if (s_v[t] > s_v[0] || (s_v[t] == s_v[0] && s_i[t] < s_i[0])) { s_v[0] = s_v[t]; s_i[0] = s_i[t]; }
      s_sign[c] = yr[s_i[0] * d + c] < 0.0 ? -1.0 : 1.0;
      s_absmax = (c == 0 || s_v[0] > s_absmax) ? s_v[0] : s_absmax;
    }
    __syncthreads();
  }
  if (tid == 0) s_expand = 10.0 / s_absmax;
  __syncthreads();
  for (int64_t t = tid; t < n * d; t += 1024) {
    const int64_t i = t / d;
    const int c = int(t % d);
    const double s = yr[t] * s_sign[c];
    yr[t] = s;
    const double u1 = umap_unit(umap_hash(seed, kUmapStreamNoise, uint64_t(i), uint64_t(2 * c)));
    const double u2 = umap_unit(umap_hash(seed, kUmapStreamNoise, uint64_t(i), uint64_t(2 * c + 1)));
    const double g = sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
    y[t] = float(s * s_expand) + float(1e-4 * g);
  }
  __syncthreads();
  for (int c = 0; c < d; ++c) {
    float lo = INFINITY, hi = -INFINITY;
    for (int64_t i = tid; i < n; i += 1024) {
      const float e = y[i * d + c];
      lo = e < lo ? e : lo;
      hi = e > hi ? e : hi;
    }
    s_lo[tid] = lo;
    s_hi[tid] = hi;
    __syncthreads();
    if (tid == 0) {
      for (int t = 1; t < 1024; ++t) {
        s_lo[0] = s_lo[t] < s_lo[0] ? s_lo[t] : s_lo[0];
        s_hi[0] = s_hi[t] > s_hi[0] ? s_hi[t] : s_hi[0];
      }
      s_min[c] = s_lo[0];
      s_max[c] = s_hi[0];
    }
    __syncthreads();
  }
  for (int64_t t = tid; t < n * d; t += 1024) {
    const int c = int(t % d);
    y[t] = 10.0f * (y[t] - s_min[c]) / (s_max[c] - s_min[c]);
  }
}

// ---------------------------------------------------------------------------------------------- layout epochs
__device__ __forceinline__ float umap_clip(float x) { return x > 4.0f ? 4.0f : (x < -4.0f ? -4.0f : x); }

// Epoch e, one thread per vertex i: y_i moves from its own current position; every other vertex is read from the
// snapshot `prev` (the previous epoch's output), and the result goes to `next`.  For each edge of row i (columns
// ascending) whose next sample is due, the attraction is applied twice (edge (i, j) with i as head, then edge (j, i)
// with i as the moved tail), then the edge's negative samples; the schedule counters advance in fp64.
__global__ void __launch_bounds__(kUmapThreads) umap_epoch_kernel(const int64_t* __restrict__ indptr,
                                                                  const int32_t* __restrict__ col,
                                                                  const double* __restrict__ eps, int64_t n, int d,
                                                                  float a, float b, int e, float alpha, uint64_t seed,
                                                                  double* __restrict__ next_sample,
                                                                  double* __restrict__ next_neg,
                                                                  const float* __restrict__ prev,
                                                                  float* __restrict__ next) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* snap = prev;
  float y[kUmapMaxD];
#pragma unroll
  for (int c = 0; c < kUmapMaxD; ++c) y[c] = c < d ? prev[i * d + c] : 0.0f;
  const double ed = double(e);
  for (int64_t p = indptr[i]; p < indptr[i + 1]; ++p) {
    if (next_sample[p] > ed) continue;
    const float* o = snap + int64_t(col[p]) * d;
    for (int rep = 0; rep < 2; ++rep) {
      float d2 = 0.0f;
#pragma unroll
      for (int c = 0; c < kUmapMaxD; ++c)
        if (c < d) d2 += (y[c] - o[c]) * (y[c] - o[c]);
      float g = 0.0f;
      if (d2 > 0.0f) g = -2.0f * a * b * powf(d2, b - 1.0f) / (a * powf(d2, b) + 1.0f);
#pragma unroll
      for (int c = 0; c < kUmapMaxD; ++c)
        if (c < d) y[c] += umap_clip(g * (y[c] - o[c])) * alpha;
    }
    const double epn = eps[p] / kUmapNegRate;
    next_sample[p] += eps[p];
    const int n_neg = int((ed - next_neg[p]) / epn);
    for (int s = 0; s < n_neg; ++s) {
      const int64_t kk = int64_t(umap_hash(seed, uint64_t(e), uint64_t(p), uint64_t(s)) % uint64_t(n));
      if (kk == i) continue;
      const float* r = snap + kk * d;
      float d2 = 0.0f;
#pragma unroll
      for (int c = 0; c < kUmapMaxD; ++c)
        if (c < d) d2 += (y[c] - r[c]) * (y[c] - r[c]);
      if (!(d2 > 0.0f)) continue;
      const float g = 2.0f * kUmapGamma * b / ((0.001f + d2) * (a * powf(d2, b) + 1.0f));
#pragma unroll
      for (int c = 0; c < kUmapMaxD; ++c)
        if (c < d) y[c] += umap_clip(g * (y[c] - r[c])) * alpha;
    }
    next_neg[p] += umap_mul_rn(double(n_neg), epn);
  }
#pragma unroll
  for (int c = 0; c < kUmapMaxD; ++c)
    if (c < d) next[i * d + c] = y[c];
}

}  // namespace
}  // namespace crag
