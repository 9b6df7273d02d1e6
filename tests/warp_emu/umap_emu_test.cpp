// The kernels of crag_umap_* (csrc/umap_kernels.cuh, the header umap.cu includes) on emulated thread blocks
// (warp_emu.h), enqueued as umap.cu enqueues them.  Each stage runs twice: blocks one after the other, then with all
// blocks of each launch resident and advancing in a random interleaving.  The two outputs must be bit-identical; the
// first is written for tests/test_umap_emulated.py, which checks it against the float64 oracle (tests/umap_oracle.py).
//
//   --fuzzy in out     in:  int64 n; int32 k; int64 ids[n][k]; float scores[n][k]
//                      out: int32 nbr[n][k]; float dist[n][k], rho[n], sigma[n], memb[n][k]
//   --spectral in out  in:  int64 n, nnz; int32 d, iters; uint64 seed; int64 indptr[n+1]; int32 idx[nnz]; float w[nnz]
//                      out: float y[n][d]; double vectors[n][d], eigenvalues[p]
//   --epochs in out    in:  int64 n, nnz; int32 d, n_epochs, e0, e1; uint64 seed; float a, b; int64 indptr[n+1];
//                           int32 idx[nnz]; double eps[nnz], next_sample[nnz], next_neg[nnz]; float y[n][d]
//                      out: float y[n][d]; double next_sample[nnz], next_neg[nnz]
// The epoch kernel runs in 32-thread blocks here (128 on the GPU; it does not depend on the block size) so that a
// small graph spans several blocks.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>   // the stub

#include "umap_kernels.cuh"

using namespace crag;

#define REQUIRE(cond, ...)                                                \
  do {                                                                    \
    if (!(cond)) {                                                        \
      fprintf(stderr, "FAILED %s:%d: %s\n  ", __FILE__, __LINE__, #cond); \
      fprintf(stderr, __VA_ARGS__);                                       \
      fprintf(stderr, "\n");                                              \
      exit(1);                                                            \
    }                                                                     \
  } while (0)

template <class T>
static void get(FILE* f, T* p, size_t count) {
  REQUIRE(fread(p, sizeof(T), count, f) == count, "short case file");
}
template <class T>
static std::vector<T> getv(FILE* f, size_t count) {
  std::vector<T> v(count);
  get(f, v.data(), count);
  return v;
}
template <class T>
static void put(FILE* f, const std::vector<T>& v) {
  REQUIRE(fwrite(v.data(), sizeof(T), v.size(), f) == v.size(), "short write");
}
template <class T>
static bool same(const std::vector<T>& a, const std::vector<T>& b) {
  return a.size() == b.size() && memcmp(a.data(), b.data(), a.size() * sizeof(T)) == 0;
}

static void launch(uint64_t seed, unsigned grid, int block, size_t smem, const std::function<void()>& body) {
  if (grid == 0) return;
  if (seed == 0) warp_emu::launch(grid, block, body, smem);
  else warp_emu::launch_concurrent(grid, block, body, smem, seed, 96 << 10);
}
static unsigned blocks(int64_t items, int per) { return unsigned((items + per - 1) / per); }

// ------------------------------------------------------------------------------------------------- fuzzy graph
struct Fuzzy {
  std::vector<int32_t> nbr;
  std::vector<float> dist, rho, sigma, memb;
};
static Fuzzy run_fuzzy(int64_t n, int k, const std::vector<int64_t>& ids, const std::vector<float>& sc, uint64_t seed) {
  Fuzzy o;
  o.nbr.assign(size_t(n) * k, -7);
  o.dist.assign(size_t(n) * k, -7.0f);
  o.memb.assign(size_t(n) * k, -7.0f);
  o.rho.assign(size_t(n), -7.0f);
  o.sigma.assign(size_t(n), -7.0f);
  std::vector<double> rowsum(size_t(n), -7.0), mean(1, -7.0);
  uint64_t s = seed;
  auto next = [&]() { return seed ? ++s : 0; };
  const unsigned g = blocks(n, kUmapThreads / 32);
  launch(next(), g, kUmapThreads, 0,
         [&] { umap_knn_lists_kernel(ids.data(), sc.data(), n, k, o.nbr.data(), o.dist.data(), rowsum.data()); });
  launch(next(), 1, 1024, sizeof(double) * 1024, [&] { umap_mean_kernel(rowsum.data(), n, k, mean.data()); });
  launch(next(), g, kUmapThreads, 0, [&] {
    umap_smooth_kernel(o.nbr.data(), o.dist.data(), rowsum.data(), mean.data(), n, k, o.rho.data(), o.sigma.data(),
                       o.memb.data());
  });
  return o;
}

// ---------------------------------------------------------------------------------------------- spectral start
struct Spectral {
  std::vector<float> y;
  std::vector<double> vec, vals;
};
static Spectral run_spectral(int64_t n, int d, int iters, uint64_t hseed, const std::vector<int64_t>& ip,
                             const std::vector<int32_t>& ix, const std::vector<float>& w, uint64_t seed) {
  const UmapSpectralPlan pl = plan_umap_spectral(n, d);
  const int p = pl.p;
  std::vector<double> deg(n, -7), dis(n, -7), v(size_t(n) * p, -7), wk(size_t(n) * p, -7),
      part(size_t(pl.chunks) * p * p, -7), rinv(size_t(p) * p, -7), q(size_t(p) * p + p, -7);
  Spectral o;
  o.y.assign(size_t(n) * d, -7.0f);
  o.vec.assign(size_t(n) * d, -7.0);
  uint64_t s = seed;
  auto next = [&]() { return seed ? ++s : 0; };
  const unsigned npg = blocks(n * p, kUmapThreads);
  launch(next(), blocks(n, kUmapThreads), kUmapThreads, 0,
         [&] { umap_degree_kernel(ip.data(), w.data(), n, deg.data(), dis.data()); });
  launch(next(), npg, kUmapThreads, 0, [&] { umap_basis_kernel(deg.data(), n, p, hseed, v.data()); });
  for (int it = 0; it < (n <= 16 ? 0 : iters); ++it) {
    launch(next(), npg, kUmapThreads, 0,
           [&] { umap_spmm_kernel(ip.data(), ix.data(), w.data(), dis.data(), n, p, v.data(), wk.data()); });
    launch(next(), pl.chunks, kUmapGramThreads, 0,
           [&] { umap_gram_kernel(wk.data(), wk.data(), n, p, pl.chunk_rows, part.data()); });
    launch(next(), 1, 32, 0, [&] { umap_cholqr_kernel(part.data(), pl.chunks, p, rinv.data()); });
    launch(next(), npg, kUmapThreads, 0, [&] { umap_apply_r_kernel(wk.data(), rinv.data(), n, p, v.data()); });
  }
  launch(next(), npg, kUmapThreads, 0,
         [&] { umap_spmm_kernel(ip.data(), ix.data(), w.data(), dis.data(), n, p, v.data(), wk.data()); });
  launch(next(), pl.chunks, kUmapGramThreads, 0,
         [&] { umap_gram_kernel(v.data(), wk.data(), n, p, pl.chunk_rows, part.data()); });
  launch(next(), 1, 32, 0, [&] { umap_ritz_kernel(part.data(), pl.chunks, p, q.data()); });
  launch(next(), blocks(n * d, kUmapThreads), kUmapThreads, 0,
         [&] { umap_ritz_vectors_kernel(v.data(), q.data(), n, p, d, o.vec.data()); });
  launch(next(), 1, 1024, 0, [&] { umap_post_kernel(o.vec.data(), n, d, hseed, o.y.data()); });
  o.vals.assign(q.begin() + size_t(p) * p, q.end());
  return o;
}

// ------------------------------------------------------------------------------------------------------ epochs
struct Layout {
  std::vector<float> y;
  std::vector<double> ns, nn;
};
static Layout run_epochs(int64_t n, int d, int n_epochs, int e0, int e1, uint64_t hseed, float a, float b,
                         const std::vector<int64_t>& ip, const std::vector<int32_t>& ix, const std::vector<double>& eps,
                         Layout o, uint64_t seed) {
  std::vector<float> other(size_t(n) * d, -7.0f);
  float* cur = o.y.data();
  float* nxt = other.data();
  uint64_t s = seed;
  auto next = [&]() { return seed ? ++s : 0; };
  for (int e = e0; e < e1; ++e) {
    const float alpha = float(1.0 - double(e > 1 ? e - 1 : 0) / double(n_epochs));
    launch(next(), blocks(n, 32), 32, 0, [&] {
      umap_epoch_kernel(ip.data(), ix.data(), eps.data(), n, d, a, b, e, alpha, hseed, o.ns.data(), o.nn.data(), cur,
                        nxt);
    });
    std::swap(cur, nxt);
  }
  if (cur != o.y.data()) memcpy(o.y.data(), cur, sizeof(float) * size_t(n) * d);
  return o;
}

int main(int argc, char** argv) {
  REQUIRE(argc == 4, "usage: umap_emu_test --fuzzy|--spectral|--epochs case.bin out.bin");
  FILE* f = fopen(argv[2], "rb");
  REQUIRE(f != nullptr, "cannot open %s", argv[2]);
  FILE* out = nullptr;
  const uint64_t shuffle = 20261017ull;
  if (strcmp(argv[1], "--fuzzy") == 0) {
    int64_t n;
    int32_t k;
    get(f, &n, 1);
    get(f, &k, 1);
    const auto ids = getv<int64_t>(f, size_t(n) * k);
    const auto sc = getv<float>(f, size_t(n) * k);
    const Fuzzy base = run_fuzzy(n, k, ids, sc, 0), again = run_fuzzy(n, k, ids, sc, shuffle);
    REQUIRE(same(base.nbr, again.nbr) && same(base.dist, again.dist) && same(base.rho, again.rho) &&
                same(base.sigma, again.sigma) && same(base.memb, again.memb),
            "fuzzy graph differs between block interleavings");
    out = fopen(argv[3], "wb");
    REQUIRE(out != nullptr, "cannot write %s", argv[3]);
    put(out, base.nbr); put(out, base.dist); put(out, base.rho); put(out, base.sigma); put(out, base.memb);
    printf("ok  fuzzy n=%lld k=%d, 2 interleavings bit-identical\n", (long long)n, k);
  } else if (strcmp(argv[1], "--spectral") == 0) {
    int64_t n, nnz;
    int32_t d, iters;
    uint64_t hseed;
    get(f, &n, 1); get(f, &nnz, 1); get(f, &d, 1); get(f, &iters, 1); get(f, &hseed, 1);
    const auto ip = getv<int64_t>(f, size_t(n) + 1);
    const auto ix = getv<int32_t>(f, size_t(nnz));
    const auto w = getv<float>(f, size_t(nnz));
    const Spectral base = run_spectral(n, d, iters, hseed, ip, ix, w, 0);
    const Spectral again = run_spectral(n, d, iters, hseed, ip, ix, w, shuffle);
    REQUIRE(same(base.y, again.y) && same(base.vec, again.vec) && same(base.vals, again.vals),
            "spectral start differs between block interleavings");
    out = fopen(argv[3], "wb");
    REQUIRE(out != nullptr, "cannot write %s", argv[3]);
    put(out, base.y); put(out, base.vec); put(out, base.vals);
    printf("ok  spectral n=%lld d=%d iters=%d, 2 interleavings bit-identical\n", (long long)n, d, iters);
  } else if (strcmp(argv[1], "--epochs") == 0) {
    int64_t n, nnz;
    int32_t d, n_epochs, e0, e1;
    uint64_t hseed;
    float a, b;
    get(f, &n, 1); get(f, &nnz, 1); get(f, &d, 1); get(f, &n_epochs, 1); get(f, &e0, 1); get(f, &e1, 1);
    get(f, &hseed, 1); get(f, &a, 1); get(f, &b, 1);
    const auto ip = getv<int64_t>(f, size_t(n) + 1);
    const auto ix = getv<int32_t>(f, size_t(nnz));
    const auto eps = getv<double>(f, size_t(nnz));
    Layout in;
    in.ns = getv<double>(f, size_t(nnz));
    in.nn = getv<double>(f, size_t(nnz));
    in.y = getv<float>(f, size_t(n) * d);
    const Layout base = run_epochs(n, d, n_epochs, e0, e1, hseed, a, b, ip, ix, eps, in, 0);
    const Layout again = run_epochs(n, d, n_epochs, e0, e1, hseed, a, b, ip, ix, eps, in, shuffle);
    REQUIRE(same(base.y, again.y) && same(base.ns, again.ns) && same(base.nn, again.nn),
            "layout differs between block interleavings");
    out = fopen(argv[3], "wb");
    REQUIRE(out != nullptr, "cannot write %s", argv[3]);
    put(out, base.y); put(out, base.ns); put(out, base.nn);
    printf("ok  epochs n=%lld d=%d [%d, %d), 2 interleavings bit-identical\n", (long long)n, d, e0, e1);
  } else {
    REQUIRE(false, "unknown mode %s", argv[1]);
  }
  fclose(f);
  fclose(out);
  printf("ALL OK\n");
  return 0;
}
