// The kernels of crag_gmm_sweep (csrc/gmm_kernels.cuh, the header gmm.cu includes) on emulated thread blocks
// (warp_emu.h), enqueued as gmm.cu enqueues them.  Each case runs twice: blocks one after the other, then with all
// blocks of each launch resident and advancing in a random interleaving.  The two outputs must be bit-identical; the
// first is written for tests/test_gmm_emulated.py, which checks it against the float64 oracle.
//
// Case file (little endian): int64 n; int32 d, M; double x[n][d]; int64 first_centre[M]; int64 n_draws;
// double draws[n_draws].
// Output file: double bic[M]; int32 iters[M], converged[M], best; double weights[M], means[M][d],
// memberships[n][best]; int32 seeds[M(M+1)/2], labels[M][n], Lloyd iterations[M] (from the workspace's state).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>   // the stub

#include "gmm_kernels.cuh"

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

struct Case {
  int64_t n = 0;
  int32_t d = 0, M = 0;
  std::vector<double> x, draws;
  std::vector<int64_t> first;
};

template <class T>
static void read_into(FILE* f, std::vector<T>& v, int64_t count) {
  v.resize(size_t(count));
  REQUIRE(fread(v.data(), sizeof(T), size_t(count), f) == size_t(count), "short case file");
}

static Case read_case(const char* path) {
  FILE* f = fopen(path, "rb");
  REQUIRE(f != nullptr, "cannot open %s", path);
  Case c;
  int64_t n_draws = 0;
  REQUIRE(fread(&c.n, 8, 1, f) == 1 && fread(&c.d, 4, 1, f) == 1 && fread(&c.M, 4, 1, f) == 1, "short header");
  read_into(f, c.x, c.n * c.d);
  read_into(f, c.first, c.M);
  REQUIRE(fread(&n_draws, 8, 1, f) == 1, "short case file");
  read_into(f, c.draws, n_draws);
  fclose(f);
  return c;
}

static void launch(uint64_t seed, unsigned grid, int block, size_t smem, const std::function<void()>& body) {
  if (grid == 0) return;
  if (seed == 0) warp_emu::launch(grid, block, body, smem);
  else warp_emu::launch_concurrent(grid, block, body, smem, seed, 96 << 10);
}

struct Out {
  std::vector<double> bic, weights, means, memb;
  std::vector<int32_t> iters, conv, best, seeds, labels, lloyd_iters;
};

// gmm.cu's sequence for one call
static Out run(const Case& c, uint64_t seed) {
  const int64_t n = c.n;
  const int d = c.d, M = c.M;
  warp_emu::Workspace ws(plan_gmm(n, d, M).total, kWsAlign, 0xFF);   // NaN everywhere
  const GmmPlan p = plan_gmm(n, d, M, ws.base);
  const int R = p.chunks, C = p.components;
  const unsigned grid = unsigned(R * M);
  Out o;
  o.bic.assign(M, -7.0); o.weights.assign(M, -7.0); o.means.assign(size_t(M) * d, -7.0);
  o.memb.assign(size_t(n) * M, -7.0);
  o.iters.assign(M, -7); o.conv.assign(M, -7); o.best.assign(1, -7); o.seeds.assign(C, -7);
  o.labels.assign(size_t(M) * n, -7);
  const double* x = c.x.data();
  int32_t* labels = o.labels.data();
  const size_t assign_smem = sizeof(double) * size_t(M * d + kGmmThreads * d) + sizeof(int32_t) * 2 * kGmmThreads;
  const size_t update_smem = sizeof(double) * size_t(M * (d + 1) + kGmmThreads) +
                             sizeof(int64_t) * (kGmmMaxM + kGmmThreads) + sizeof(int) * (kGmmMaxM + 1);
  const size_t stats_smem = sizeof(double) * size_t(kGmmTile) * (M + d);
  const size_t m_smem = sizeof(double) * size_t((kGmmThreads / 32) * (1 + d + gmm_tri(d)) + 2 * kGmmMaxM) + 16;
  const size_t seed_smem = sizeof(double) * (2 * kGmmSeedThreads + 1 + kGmmMaxTrials * (1 + kGmmMaxD)) +
                           sizeof(int64_t) * kGmmMaxTrials;
  uint64_t s = seed;
  auto next = [&]() { return seed ? ++s : 0; };

  launch(next(), 1, 1024, sizeof(double) * 1024, [&] { gmm_moments_kernel(x, n, d, M, p.glob, p.state); });
  launch(next(), 4, kGmmThreads, 0, [&] { gmm_centre_kernel(x, n, d, M, p.glob, p.xc, labels); });
  launch(next(), M, kGmmSeedThreads, seed_smem,
         [&] { gmm_seed_kernel(p.xc, n, d, c.first.data(), c.draws.data(), p.dist, p.centres, o.seeds.data()); });
  for (int it = 0; it < kGmmLloydIters; ++it) {
    launch(next(), grid, kGmmThreads, assign_smem, [&] {
      gmm_lloyd_assign_kernel(p.xc, n, d, M, R, p.chunk_rows, 1, p.state, p.centres, labels, p.dist, p.lsum, p.lchg);
    });
    launch(next(), M, kGmmThreads, update_smem, [&] {
      gmm_lloyd_update_kernel(p.xc, n, d, M, R, it, p.glob, p.state, p.centres, labels, p.dist, p.lsum, p.lchg);
    });
  }
  launch(next(), grid, kGmmThreads, assign_smem, [&] {
    gmm_lloyd_assign_kernel(p.xc, n, d, M, R, p.chunk_rows, 0, p.state, p.centres, labels, p.dist, p.lsum, p.lchg);
  });
  launch(next(), unsigned((C * d + kGmmThreads - 1) / kGmmThreads), kGmmThreads, 0,
         [&] { gmm_em_setup_kernel(d, C, p.glob, p.centres, p.mu); });
  launch(next(), grid, kGmmThreads, stats_smem, [&] {
    gmm_em_stats_kernel(x, n, d, M, R, p.chunk_rows, kGmmInit, p.state, nullptr, labels, p.mu, p.prec, p.cst, p.esum, p.lse, nullptr);
  });
  launch(next(), M, kGmmThreads, m_smem,
         [&] { gmm_mstep_kernel(n, d, M, R, kGmmInit, 0, p.state, p.mu, p.prec, p.cst, p.wt, p.esum, p.lse); });
  for (int it = 1; it <= kGmmEmIters; ++it) {
    launch(next(), grid, kGmmThreads, stats_smem, [&] {
      gmm_em_stats_kernel(x, n, d, M, R, p.chunk_rows, kGmmStep, p.state, nullptr, labels, p.mu, p.prec, p.cst, p.esum, p.lse,
                          nullptr);
    });
    launch(next(), M, kGmmThreads, m_smem,
           [&] { gmm_mstep_kernel(n, d, M, R, kGmmStep, it, p.state, p.mu, p.prec, p.cst, p.wt, p.esum, p.lse); });
  }
  launch(next(), grid, kGmmThreads, stats_smem, [&] {
    gmm_em_stats_kernel(x, n, d, M, R, p.chunk_rows, kGmmScore, p.state, nullptr, labels, p.mu, p.prec, p.cst, p.esum, p.lse, nullptr);
  });
  launch(next(), 1, kGmmMaxM, sizeof(double) * (kGmmMaxM + 1), [&] {
    gmm_select_kernel(n, d, M, R, p.state, p.mu, p.wt, p.lse, o.bic.data(), o.iters.data(), o.conv.data(), o.best.data(),
                      o.weights.data(), o.means.data());
  });
  launch(next(), unsigned(R), kGmmThreads, stats_smem, [&] {
    gmm_em_stats_kernel(x, n, d, M, R, p.chunk_rows, kGmmResp, p.state, o.best.data(), labels, p.mu, p.prec, p.cst, p.esum, p.lse,
                        o.memb.data());
  });
  o.memb.resize(size_t(n) * o.best[0]);
  for (int m = 0; m < M; ++m) o.lloyd_iters.push_back(p.state[m].lloyd_iters);
  return o;
}

// --lloyd: the Lloyd loop alone, from given centres (Xc coordinates), for one model of m components: the kernels of
// every other model are marked done.  Case: int64 n; int32 d, m; double x[n][d]; double centres[m][d].
// Output: int32 labels[n], iterations; double centres[m][d].
static void run_lloyd(const char* in, const char* out, uint64_t seed) {
  FILE* f = fopen(in, "rb");
  REQUIRE(f != nullptr, "cannot open %s", in);
  int64_t n = 0;
  int32_t d = 0, m = 0;
  REQUIRE(fread(&n, 8, 1, f) == 1 && fread(&d, 4, 1, f) == 1 && fread(&m, 4, 1, f) == 1, "short header");
  std::vector<double> x, c0;
  read_into(f, x, n * d);
  read_into(f, c0, int64_t(m) * d);
  fclose(f);
  const int M = m;
  warp_emu::Workspace ws(plan_gmm(n, d, M).total, kWsAlign, 0xFF);
  const GmmPlan p = plan_gmm(n, d, M, ws.base);
  const int R = p.chunks;
  const size_t assign_smem = sizeof(double) * size_t(M * d + kGmmThreads * d) + sizeof(int32_t) * 2 * kGmmThreads;
  const size_t update_smem = sizeof(double) * size_t(M * (d + 1) + kGmmThreads) +
                             sizeof(int64_t) * (kGmmMaxM + kGmmThreads) + sizeof(int) * (kGmmMaxM + 1);
  uint64_t s = seed;
  auto next = [&]() { return seed ? ++s : 0; };
  launch(next(), 1, 1024, sizeof(double) * 1024, [&] { gmm_moments_kernel(x.data(), n, d, M, p.glob, p.state); });
  launch(next(), 4, kGmmThreads, 0, [&] { gmm_centre_kernel(x.data(), n, d, M, p.glob, p.xc, p.labels); });
  for (int k = 0; k + 1 < M; ++k) p.state[k].lloyd_done = p.state[k].lloyd_strict = 1;
  memcpy(p.centres + int64_t(gmm_comp_off(m)) * d, c0.data(), c0.size() * sizeof(double));
  for (int it = 0; it < kGmmLloydIters; ++it) {
    launch(next(), unsigned(R * M), kGmmThreads, assign_smem, [&] {
      gmm_lloyd_assign_kernel(p.xc, n, d, M, R, p.chunk_rows, 1, p.state, p.centres, p.labels, p.dist, p.lsum, p.lchg);
    });
    launch(next(), M, kGmmThreads, update_smem, [&] {
      gmm_lloyd_update_kernel(p.xc, n, d, M, R, it, p.glob, p.state, p.centres, p.labels, p.dist, p.lsum, p.lchg);
    });
  }
  launch(next(), unsigned(R * M), kGmmThreads, assign_smem, [&] {
    gmm_lloyd_assign_kernel(p.xc, n, d, M, R, p.chunk_rows, 0, p.state, p.centres, p.labels, p.dist, p.lsum, p.lchg);
  });
  FILE* o = fopen(out, "wb");
  REQUIRE(o != nullptr, "cannot write %s", out);
  REQUIRE(fwrite(p.labels + int64_t(m - 1) * n, 4, size_t(n), o) == size_t(n), "short write");
  REQUIRE(fwrite(&p.state[m - 1].lloyd_iters, 4, 1, o) == 1, "short write");
  REQUIRE(fwrite(p.centres + int64_t(gmm_comp_off(m)) * d, 8, c0.size(), o) == c0.size(), "short write");
  fclose(o);
}

template <class T>
static bool same(const std::vector<T>& a, const std::vector<T>& b) {
  return a.size() == b.size() && memcmp(a.data(), b.data(), a.size() * sizeof(T)) == 0;
}

template <class T>
static void put(FILE* f, const std::vector<T>& v) {
  REQUIRE(fwrite(v.data(), sizeof(T), v.size(), f) == v.size(), "short write");
}

int main(int argc, char** argv) {
  if (argc == 4 && strcmp(argv[1], "--lloyd") == 0) {
    run_lloyd(argv[2], argv[3], 0);
    printf("ALL OK\n");
    return 0;
  }
  REQUIRE(argc >= 3 && argc % 2 == 1, "usage: gmm_emu_test case.bin out.bin [case.bin out.bin ...]");
  for (int a = 1; a < argc; a += 2) {
    const Case c = read_case(argv[a]);
    const Out base = run(c, 0);
    const Out again = run(c, 20251017ull);
    REQUIRE(same(base.bic, again.bic) && same(base.memb, again.memb) && same(base.means, again.means) &&
                same(base.weights, again.weights) && same(base.iters, again.iters) && same(base.labels, again.labels) &&
                same(base.seeds, again.seeds) && same(base.best, again.best) && same(base.lloyd_iters, again.lloyd_iters),
            "%s: output differs between block interleavings", argv[a]);
    FILE* f = fopen(argv[a + 1], "wb");
    REQUIRE(f != nullptr, "cannot write %s", argv[a + 1]);
    put(f, base.bic); put(f, base.iters); put(f, base.conv); put(f, base.best); put(f, base.weights);
    put(f, base.means); put(f, base.memb); put(f, base.seeds); put(f, base.labels);
    put(f, base.lloyd_iters);
    fclose(f);
    printf("ok  %s: n=%lld d=%d M=%d best=%d, 2 interleavings bit-identical\n", argv[a], (long long)c.n, c.d, c.M,
           base.best[0]);
  }
  printf("ALL OK\n");
  return 0;
}
