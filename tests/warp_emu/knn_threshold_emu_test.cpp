// knn_threshold_kernel (csrc/knn_threshold.cuh, the header search.cu compiles into crag_knn_threshold) on emulated
// thread blocks (warp_emu.h), against a plain C++ model of the walk: every row's key make_key(score, row), std::sort
// descending, the first min(limit, n_rows) keys walked in order -- stop at the first !(score >= threshold), skip the
// self row and the excluded rows, accept the rest until `cap` are accepted.  Counts, ids and scores must match bit for
// bit, -1 / -inf past the count.  The padding columns [n_rows, ld) of every score row hold NaN: a kernel that took
// them as rows would stop its walk at once.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <random>
#include <set>
#include <string>
#include <vector>

#include <cuda_runtime.h>   // the stub

#include "knn_threshold.cuh"

using namespace crag;

static std::mt19937_64 rng(20261018);

#define REQUIRE(cond, ...)                                                \
  do {                                                                    \
    if (!(cond)) {                                                        \
      fprintf(stderr, "FAILED %s:%d: %s\n  ", __FILE__, __LINE__, #cond); \
      fprintf(stderr, __VA_ARGS__);                                       \
      fprintf(stderr, "\n");                                              \
      exit(1);                                                            \
    }                                                                     \
  } while (0)

static double uni(double a, double b) { return a + (b - a) * double(rng() % 1000001) / 1e6; }

// one query row: its scores, its self row
struct Query {
  std::vector<float> s;
  int64_t self;
};

struct Result {
  int count;
  std::vector<int64_t> ids;
  std::vector<float> sc;
};

static Result model(const std::vector<float>& s, float t, int limit, int cap, int64_t self, const std::vector<int64_t>& excl) {
  const int n = int(s.size());
  std::vector<uint64_t> keys(n);
  for (int r = 0; r < n; ++r) keys[r] = make_key(s[r], uint32_t(r));
  std::sort(keys.begin(), keys.end(), std::greater<uint64_t>());
  Result w{0, std::vector<int64_t>(cap, -1), std::vector<float>(cap, -INFINITY)};
  const int len = std::min(limit, n);
  for (int p = 0; p < len && w.count < cap; ++p) {
    const float v = key_score(keys[p]);
    if (!(v >= t)) break;
    const int64_t r = key_id(keys[p]);
    if (r == self || std::find(excl.begin(), excl.end(), r) != excl.end()) continue;
    w.ids[w.count] = r;
    w.sc[w.count] = v;
    ++w.count;
  }
  return w;
}

// which digit of knn_select's radix select tells the k-th best score word from the (k+1)-th (3 = they are equal)
static std::set<int> g_digits;
static int deciding_digit(const std::vector<float>& s, int k) {
  std::vector<uint32_t> o(s.size());
  for (size_t r = 0; r < s.size(); ++r) o[r] = orderable_f32(s[r]);
  std::sort(o.begin(), o.end(), std::greater<uint32_t>());
  const uint32_t a = o[k - 1], b = o[k];
  if (a >> 21 != b >> 21) return 0;
  if (a >> 10 != b >> 10) return 1;
  if (a != b) return 2;
  return 3;
}

static int g_overflow = 0;

static void check(const char* what, const std::vector<Query>& qs, float t, int limit, int cap,
                  const std::vector<int64_t>& excl, bool with_self = true) {
  const int nq = int(qs.size());
  const int n_rows = int(qs[0].s.size());
  const int64_t ld = ((n_rows > 0 ? n_rows : 1) + 3) & ~int64_t(3);
  std::vector<float> block(size_t(nq) * ld + 4, __uint_as_float(0x7FC00123u));   // padding columns: NaN
  float* base = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(block.data()) + 15) & ~uintptr_t(15));
  std::vector<int64_t> self(nq);
  for (int q = 0; q < nq; ++q) {
    for (int r = 0; r < n_rows; ++r) base[q * ld + r] = qs[q].s[r];
    self[q] = qs[q].self;
  }
  std::vector<int> cnt(nq, -7);
  std::vector<int64_t> ids(size_t(nq) * cap, -7);
  std::vector<float> sc(size_t(nq) * cap, -7.f);
  warp_emu::launch(nq, kKnnThreads, [&] {
    knn_threshold_kernel(base, ld, n_rows, t, limit, cap, with_self ? self.data() : nullptr, excl.data(), int(excl.size()),
                         cnt.data(), ids.data(), sc.data());
  });
  for (int q = 0; q < nq; ++q) {
    const Result w = model(qs[q].s, t, limit, cap, with_self ? self[q] : -1, excl);
    int c = 0;
    for (float v : qs[q].s) c += v >= t ? 1 : 0;
    REQUIRE(cnt[q] == w.count, "%s: query %d (n_rows=%d c=%d limit=%d cap=%d): count %d, want %d", what, q, n_rows, c,
            limit, cap, cnt[q], w.count);
    for (int j = 0; j < cap; ++j) {
      const int64_t gi = ids[size_t(q) * cap + j];
      const float gs = sc[size_t(q) * cap + j];
      REQUIRE(gi == w.ids[j] && __float_as_uint(gs) == __float_as_uint(w.sc[j]),
              "%s: query %d (n_rows=%d c=%d limit=%d cap=%d): rank %d holds row %lld score %a, want row %lld score %a",
              what, q, n_rows, c, limit, cap, j, (long long)gi, gs, (long long)w.ids[j], w.sc[j]);
    }
    if (c > kKnnMaxK) {   // the overflow path: record which radix digit decided its cut
      int m = 0;
      std::set<int64_t> skip(excl.begin(), excl.end());
      if (with_self) skip.insert(self[q]);
      for (int64_t r : skip)
        if (r >= 0 && r < n_rows && qs[q].s[r] >= t) ++m;
      const int k_sel = std::min({limit, c, cap + m});
      if (k_sel < n_rows) g_digits.insert(deciding_digit(qs[q].s, k_sel));
      ++g_overflow;
    }
  }
}

static std::vector<float> scores_uniform(int n, double lo, double hi) {
  std::vector<float> s(n);
  for (auto& v : s) v = float(uni(lo, hi));
  return s;
}

// n rows, `hits` of them (random places) drawn from [t, hi], the rest below t
static std::vector<float> scores_with_hits(int n, int hits, float t, double hi) {
  std::vector<float> s = scores_uniform(n, -1.0, double(t) - 1e-3);
  std::vector<int> rows(n);
  for (int r = 0; r < n; ++r) rows[r] = r;
  std::shuffle(rows.begin(), rows.end(), rng);
  for (int j = 0; j < hits && j < n; ++j) s[rows[j]] = float(uni(double(t), hi));
  return s;
}

static int64_t pick_self(const std::vector<float>& s, float t, int where) {
  // where: 0 = the best row (before the cut), 1 = a row scoring exactly at the threshold (if any), 2 = below the cut
  const int n = int(s.size());
  int best = 0, at = -1, below = -1;
  for (int r = 0; r < n; ++r) {
    if (make_key(s[r], r) > make_key(s[best], best)) best = r;
    if (s[r] == t && at < 0) at = r;
    if (!(s[r] >= t) && below < 0) below = r;
  }
  if (where == 0) return best;
  if (where == 1) return at >= 0 ? at : best;
  return below >= 0 ? below : -1;
}

int main(int argc, char** argv) {
  const bool quick = argc > 1 && std::string(argv[1]) == "quick";
  const float t = 0.8f;
  const std::vector<int64_t> none;

  // ---- c = 0, c <= cap, cap < c <= 2048: the common path; self rows before, at and after the cut; n_rows % 4 != 0
  for (int n : {1, 3, 130, 4097, 10001}) {
    for (int hits : {0, 1, 7, 101, 102, 500, 2048}) {
      if (hits > n) continue;
      std::vector<Query> qs;
      for (int q = 0; q < 3; ++q) {
        Query x{scores_with_hits(n, hits, t, 1.0), -1};
        if (hits > 2 && q == 1) x.s[(q * 977) % n] = t;   // one score exactly at the threshold
        x.self = pick_self(x.s, t, q);
        qs.push_back(x);
      }
      check("common path", qs, t, 2047, 101, none);
      std::vector<int64_t> excl = {int64_t(n / 2), pick_self(qs[0].s, t, 0), int64_t(n / 2), -1, int64_t(n) + 5};
      check("common path, excluded rows", qs, t, 2047, 101, excl);
      check("common path, limit 5", qs, t, 5, 101, excl);
      check("common path, no self rows", qs, t, 2047, 3, excl, false);
    }
    printf("ok  knn_threshold_kernel: n_rows = %d, c in {0, 1, 7, 101, 102, 500, 2048}\n", n);
  }

  // ---- ties straddling the threshold and the limit, exactly-at-threshold scores, +-0 at threshold 0
  {
    std::vector<Query> qs;
    for (int q = 0; q < 4; ++q) {
      std::vector<float> s(3001);
      const float lv[] = {0.9f, 0.8f, 0.8f, std::nextafter(0.8f, 0.f)};
      for (auto& v : s) v = lv[rng() % 4];
      qs.push_back({s, int64_t(q * 5)});
    }
    for (int limit : {1, 2, 3, 700, 1500, 2047, 5000}) {
      check("three levels at the threshold", qs, t, limit, 101, {4, 9, 9});
      check("three levels at the threshold, cap 2000", qs, t, limit, 2000, {4});
    }
    std::vector<Query> z;
    for (int q = 0; q < 2; ++q) {
      std::vector<float> s(1001);
      const float lv[] = {0.0f, -0.0f, 1e-42f, -1e-42f, -1.f};
      for (auto& v : s) v = lv[rng() % 5];
      z.push_back({s, int64_t(q)});
    }
    check("+-0 at threshold 0", z, 0.0f, 2047, 101, none);
    check("+-0 at threshold -0", z, -0.0f, 700, 1000, {0});
    printf("ok  knn_threshold_kernel: ties at the threshold and the limit, +-0 at threshold 0\n");
  }

  // ---- c > 2048: the overflow path, each radix digit deciding the cut, and tie runs
  {
    const int n = 9001;
    // digit 0: the limit's rows sit an exponent above the rest
    std::vector<Query> qs;
    for (int q = 0; q < 2; ++q) {
      std::vector<float> s = scores_uniform(n, 1.0, 1.99);
      for (int r = q; r < n; r += 30) s[r] = float(uni(2.0, 3.9));   // 300 rows
      qs.push_back({s, int64_t(q)});
    }
    check("overflow, exponent cut", qs, t, 300, 1000, none);
    check("overflow, exponent cut, limit 5", qs, t, 5, 1000, none);
    // digit 1 / 2: dense scores, a few ulps apart
    std::vector<Query> dense;
    for (int q = 0; q < 2; ++q) dense.push_back({scores_uniform(n, 0.8, 1.0), int64_t(q * 100)});
    std::vector<Query> ulps;
    for (int q = 0; q < 2; ++q) {
      std::vector<float> s(n);
      for (int r = 0; r < n; ++r) s[r] = __uint_as_float(0x3F600000u + uint32_t(rng() % 1000000) * (q + 1));
      ulps.push_back({s, int64_t(q * 3)});
    }
    std::vector<Query> fine;
    for (int q = 0; q < 2; ++q) {
      std::vector<float> s(n);
      for (int r = 0; r < n; ++r) s[r] = __uint_as_float(0x3F600000u + uint32_t(r * 7919 % n));   // distinct, 1 ulp apart
      fine.push_back({s, int64_t(q * 3)});
    }
    for (auto* set : {&dense, &ulps, &fine}) {
      check("overflow, dense scores", *set, t, 2047, 101, {7, 8});
      check("overflow, dense scores, cap 1983", *set, t, 2047, 1983, std::vector<int64_t>(64, 5));
    }
    // ties: every row equal (all above the threshold), the first rows decide
    std::vector<Query> eq;
    for (int q = 0; q < 2; ++q) eq.push_back({std::vector<float>(n, 0.9f), int64_t(q)});
    check("overflow, all rows equal", eq, t, 2047, 101, {0, 3, 2});
    check("overflow, all rows equal, limit 50", eq, t, 50, 101, {0, 3, 2});
    // a positive NaN among the rows ranks first and stops the walk; a negative NaN ranks last
    std::vector<Query> nan = dense;
    nan[0].s[n / 3] = __uint_as_float(0x7FC00000u);
    nan[1].s[n / 3] = __uint_as_float(0xFFC00000u);
    check("NaN rows", nan, t, 2047, 101, none);
    REQUIRE(g_overflow >= 20, "only %d overflow queries", g_overflow);
    for (int d = 0; d < 4; ++d) REQUIRE(g_digits.count(d), "no overflow case decided by digit %d (3 = tie)", d);
    printf("ok  knn_threshold_kernel: c > 2048 (overflow), cut by radix digits 0, 1, 2 and by a tie\n");
  }

  // ---- every row excluded, and a row count that is not a multiple of 4 with every row above the threshold
  {
    std::vector<Query> qs;
    for (int q = 0; q < 2; ++q) qs.push_back({scores_uniform(41, 0.85, 1.0), int64_t(40 - q)});
    std::vector<int64_t> all;
    for (int r = 0; r < 41; ++r)
      if (r != 40 && r != 39) all.push_back(r);
    all.push_back(39);
    check("every row excluded", {qs[0]}, t, 2047, 101, all);
    check("all but one excluded", qs, t, 2047, 101, all);
    for (int n : {5, 6, 7, 2049, 2050, 2051}) {
      std::vector<Query> w;
      for (int q = 0; q < 2; ++q) w.push_back({scores_uniform(n, 0.9, 1.0), int64_t(n - 1)});
      check("n_rows % 4 != 0", w, t, 2047, 101, none);
    }
    printf("ok  knn_threshold_kernel: every row excluded, n_rows %% 4 != 0 with NaN padding\n");
  }
  if (!quick) {
    std::vector<Query> big;
    for (int q = 0; q < 2; ++q) big.push_back({scores_with_hits(70001, 3000 * (q + 1), t, 1.0), int64_t(q)});
    check("70001 rows", big, t, 2047, 101, {1, 2});
    printf("ok  knn_threshold_kernel: 70001 rows\n");
  }
  printf("ALL OK\n");
  return 0;
}
