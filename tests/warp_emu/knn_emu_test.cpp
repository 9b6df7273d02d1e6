// knn_select_kernel (csrc/knn_select.cuh, the header search.cu compiles into crag_knn_topk) on emulated thread blocks
// (warp_emu.h), against a plain C++ model: every row's key make_key(score, row), std::sort descending, the first
// min(k, n_rows) keys -> (row + row_offset, score), -1 / -inf past n_rows, and (min, max) over all rows ordered as
// orderable_f32 orders them ((+inf, -inf) for an empty shard).  Ids, scores and (min, max) must match bit for bit.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <random>
#include <string>
#include <vector>

#include <cuda_runtime.h>   // the stub

#include "knn_select.cuh"

using namespace crag;

static std::mt19937_64 rng(20251015);

#define REQUIRE(cond, ...)                                                \
  do {                                                                    \
    if (!(cond)) {                                                        \
      fprintf(stderr, "FAILED %s:%d: %s\n  ", __FILE__, __LINE__, #cond); \
      fprintf(stderr, __VA_ARGS__);                                       \
      fprintf(stderr, "\n");                                              \
      exit(1);                                                            \
    }                                                                     \
  } while (0)

enum Dist { kRandom, kAllEqual, kThreeLevels, kAscending, kSpecials, kNumDists };
static const char* kDistName[] = {"random", "all rows equal", "three score levels", "ascending with the row id",
                                  "+-0, +-inf and denormals"};

static float draw(Dist d, int row, int n) {
  switch (d) {
    case kRandom: return float(double(rng() % 2000001) / 1e6 - 1.0);
    case kAllEqual: return 0.25f;
    case kThreeLevels: return float(int(rng() % 3)) * 0.5f - 0.5f;
    case kAscending: return float(row) / float(n > 0 ? n : 1) - 0.5f;
    case kSpecials: {
      static const float sp[] = {0.0f, -0.0f, INFINITY, -INFINITY, 1e-42f, -1e-42f, 1e-39f, -3e-40f, 1e-45f};
      return (rng() % 3 == 0) ? float(double(rng() % 2001) / 1e3 - 1.0) : sp[rng() % 9];
    }
    default: return 0.f;
  }
}

static void check(int n_rows, int k, int64_t row_offset, const std::vector<Dist>& dists) {
  const int nq = int(dists.size());
  const int64_t ld = ((n_rows > 0 ? n_rows : 1) + 3) & ~int64_t(3);
  std::vector<float> block(size_t(nq) * ld + 4, __uint_as_float(0x7FC00123u));   // padding columns: NaN the kernel must skip
  float* base = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(block.data()) + 15) & ~uintptr_t(15));
  for (int q = 0; q < nq; ++q)
    for (int r = 0; r < n_rows; ++r) base[q * ld + r] = draw(dists[q], r, n_rows);
  std::vector<int64_t> ids(size_t(nq) * k, -7);
  std::vector<float> sc(size_t(nq) * k, -7.f), mm(size_t(nq) * 2, -7.f);
  warp_emu::launch(nq, kKnnThreads, [&] {
    knn_select_kernel(base, ld, n_rows, k, row_offset, ids.data(), sc.data(), mm.data());
  });
  for (int q = 0; q < nq; ++q) {
    std::vector<uint64_t> keys(n_rows);
    uint32_t mn = 0xFFFFFFFFu, mx = 0u;
    for (int r = 0; r < n_rows; ++r) {
      const float s = base[q * ld + r];
      keys[r] = make_key(s, uint32_t(r));
      mn = std::min(mn, orderable_f32(s));
      mx = std::max(mx, orderable_f32(s));
    }
    std::sort(keys.begin(), keys.end(), std::greater<uint64_t>());
    for (int j = 0; j < k; ++j) {
      const int64_t wi = j < n_rows ? int64_t(key_id(keys[j])) + row_offset : -1;
      const float ws = j < n_rows ? key_score(keys[j]) : -INFINITY;
      const int64_t gi = ids[size_t(q) * k + j];
      const float gs = sc[size_t(q) * k + j];
      REQUIRE(gi == wi && __float_as_uint(gs) == __float_as_uint(ws),
              "k=%d n_rows=%d %s: rank %d holds row %lld score %a, want row %lld score %a", k, n_rows, kDistName[dists[q]], j,
              (long long)gi, gs, (long long)wi, ws);
    }
    const float wmn = n_rows ? unorderable_f32(mn) : INFINITY, wmx = n_rows ? unorderable_f32(mx) : -INFINITY;
    REQUIRE(__float_as_uint(mm[q * 2]) == __float_as_uint(wmn) && __float_as_uint(mm[q * 2 + 1]) == __float_as_uint(wmx),
            "k=%d n_rows=%d %s: minmax (%a, %a) want (%a, %a)", k, n_rows, kDistName[dists[q]], mm[q * 2], mm[q * 2 + 1], wmn, wmx);
  }
}

int main(int argc, char** argv) {
  const bool ties_only = argc > 1 && std::string(argv[1]) == "ties";
  const int ks[] = {1, 2, 127, 128, 129, 2047, 2048};
  int combo = 0;
  for (int k : ks) {
    const int ns[] = {1, k - 1, k, k + 1, 5000, 70001};
    for (int n : ns) {
      if (n < 1) continue;
      // two query rows per launch, the distributions rotating over the grid so every (k, n) meets several of them
      std::vector<Dist> d = {Dist(combo % kNumDists), Dist((combo + 2) % kNumDists)};
      if (ties_only) d = {kAllEqual, kThreeLevels};
      const int64_t off = (combo % 3 == 0) ? 3000000000ll : 0;
      check(n, k, off, d);
      ++combo;
    }
    printf("ok  knn_select_kernel: k = %d, n_rows in {1, k-1, k, k+1, 5000, 70001}\n", k);
  }
  if (!ties_only) {
    for (int dist = 0; dist < kNumDists; ++dist) {
      check(70001, 2047, 123456789012ll, {Dist(dist)});
      check(5000, 129, 7, {Dist(dist)});
      printf("ok  knn_select_kernel: %s, k = 2047 of 70001 rows and k = 129 of 5000, row_offset != 0\n", kDistName[dist]);
    }
    check(0, 5, 11, {kRandom, kRandom});
    check(0, 2048, 0, {kRandom});
    printf("ok  knn_select_kernel: empty shard\n");
  }
  printf("ALL OK\n");
  return 0;
}
