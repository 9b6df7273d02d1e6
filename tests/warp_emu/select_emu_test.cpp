// The select warps of the shard-scan kernel on the CPU.  select_shell.h calls the kernel's own select_warps() and
// SelectSmem (csrc/select_warps.cuh) with
//   score-tile source     -> a score matrix this test supplies (the selection logic does not care where scores come
//                            from: any fp32 matrix is a valid "q . x" for it, ties and adversarial orders included)
//   named barriers        -> the fiber emulator's (warp_emu.h)
// so that everything the four select warps do runs for real: the per-row admission test against thr_f / thr_key / the
// continuation bound, the warp-ballot compaction into the candidate buffers, flushes, the pooled-floor publishes and
// refreshes across CTAs, the first-tile fast path, the tail drain, the per-CTA lists and (min, max); also the rank
// continuation (k > 128), the score-all variant with its assignment mode, and the IVF variant (with the emulated plan
// kernel in front).  The per-CTA
// lists then go through the emulated merge_topk_kernel and the answer is compared, bit for bit, with the exact top-k
// of the score matrix under the engine's rule (score descending, row ascending).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <random>
#include <string>
#include <vector>

#include <cuda_runtime.h>   // the stub


static std::mt19937_64 rng(99);

#define REQUIRE(cond, ...)                              \
  do {                                                  \
    if (!(cond)) {                                      \
      fprintf(stderr, "FAILED %s:%d: %s\n  ", __FILE__, __LINE__, #cond); \
      fprintf(stderr, __VA_ARGS__);                     \
      fprintf(stderr, "\n");                            \
      exit(1);                                          \
    }                                                   \
  } while (0)

#include "select_shell.h"

using namespace crag;

// ------------------------------------------------------------------------------------------------ score matrices
enum class Data { Random, Ascending, AllEqual, FewLevels, PlantedTail };
static const char* name_of(Data d) {
  switch (d) { case Data::Random: return "random"; case Data::Ascending: return "ascending with the row id"; case Data::AllEqual: return "all rows equal";
               case Data::FewLevels: return "three score levels"; default: return "planted neighbours in the last rows"; }
}
static std::vector<float> make_scores(int64_t rows, Data d) {
  std::vector<float> s(size_t(rows) * kNQ);
  for (int64_t r = 0; r < rows; ++r)
    for (int q = 0; q < kNQ; ++q) {
      float v = float(double(rng() % 2000001) / 1e6 - 1.0) * 0.2f;
      if (d == Data::Ascending) v = float(r) / float(rows) + 0.001f * float(rng() % 100);
      if (d == Data::AllEqual) v = 0.25f;
      if (d == Data::FewLevels) v = float(int(rng() % 3)) * 0.1f;
      if (d == Data::PlantedTail && r >= rows - 300 && int(r % 32) == q) v = 0.9f - 0.0001f * float(rows - r);
      s[size_t(r) * kNQ + q] = v;
    }
  return s;
}
static std::vector<uint64_t> exact_keys(const std::vector<float>& s, int64_t rows, int q, uint64_t below = ~0ull) {
  std::vector<uint64_t> all;
  all.reserve(rows);
  for (int64_t r = 0; r < rows; ++r) {
    const uint64_t key = make_key(s[size_t(r) * kNQ + q], uint32_t(r));
    if (key < below) all.push_back(key);
  }
  std::sort(all.begin(), all.end(), std::greater<uint64_t>());
  return all;
}

// 0: the scan's blocks run one after the other; otherwise: all resident together, advancing in a random interleaving drawn
// from this seed (warp_emu::launch_concurrent) -- what one CTA publishes to the pool reaches the others mid-scan
static uint64_t g_concurrent_seed = 0;

// one pass = crag_search_scan + crag_search_finalize: scan shell on `grid` blocks, then the emulated merge kernel
template <int KLIST, int CAP>
static void run_pass(const std::vector<float>& scores, int64_t rows, int grid, int nq, int k, bool use_pool, uint32_t perm_mul, int perm_shift,
                     const uint64_t* after, std::vector<int64_t>& ids, std::vector<float>& sc, std::vector<float>& mm, std::vector<uint64_t>& last) {
  std::vector<uint64_t> part_keys(size_t(grid) * kNQ * k, 0xDEADull), pool(size_t(grid) * kPoolSlots * kNQ, 0ull);
  std::vector<float> part_mm(size_t(grid) * kNQ * 2, -5.f);
  g_src = MatrixScoreTiles{scores.data(), rows, nullptr};
  auto scan = [&] {
    search_select_shell<KLIST, CAP>(int(rows), nq, k, after, use_pool ? pool.data() : nullptr, perm_mul, perm_shift, part_keys.data(), part_mm.data(), NoIvfArgs{});
  };
  if (g_concurrent_seed) warp_emu::launch_concurrent(grid, kSearchThreads, scan, SelectSmem<KLIST, CAP>::bytes(), g_concurrent_seed);
  else warp_emu::launch(grid, kSearchThreads, scan, SelectSmem<KLIST, CAP>::bytes());
  ids.assign(size_t(nq) * k, -5); sc.assign(size_t(nq) * k, -5.f); mm.assign(size_t(nq) * 2, -5.f); last.assign(nq, 1);
  warp_emu::launch(nq, 128, [&] {
    merge_topk_kernel<KLIST, CAP, false>(part_keys.data(), nullptr, nullptr, part_mm.data(), grid, kNQ, nq, k, 1000, 0, 0, 0, ids.data(), sc.data(), mm.data(), last.data());
  });
}

constexpr uint32_t kAutoPerm = 0xFFFFFFFFu;     // "ask perm_multiplier()", as the library's host code does

template <int KLIST, int CAP>
static void test_topk(Data d, int grid, int tiles_per_cta, int ragged, int nq, int k, bool use_pool, uint32_t perm_mul, int perm_shift) {
  const int64_t rows = int64_t(grid) * tiles_per_cta * kTileRows - ragged;
  const int64_t n_tiles = (rows + kTileRows - 1) / kTileRows;
  if (perm_mul == kAutoPerm) perm_mul = perm_multiplier(n_tiles >> perm_shift);
  else if (perm_mul) {      // a hand-picked multiplier must be a bijection of the tile groups
    int64_t a = perm_mul, b = n_tiles >> perm_shift;
    while (b) { const int64_t t = a % b; a = b; b = t; }
    REQUIRE(a == 1, "test bug: multiplier %u is not coprime to %lld tile groups", perm_mul, (long long)(n_tiles >> perm_shift));
  }
  std::vector<float> scores = make_scores(rows, d);
  std::vector<int64_t> ids;
  std::vector<float> sc, mm;
  std::vector<uint64_t> last;
  run_pass<KLIST, CAP>(scores, rows, grid, nq, k, use_pool, perm_mul, perm_shift, nullptr, ids, sc, mm, last);
  for (int q = 0; q < nq; ++q) {
    std::vector<uint64_t> want = exact_keys(scores, rows, q);
    for (int j = 0; j < k; ++j) {
      const int64_t wi = j < int(want.size()) ? int64_t(key_id(want[j])) + 1000 : -1;
      const float ws = j < int(want.size()) ? key_score(want[j]) : -INFINITY;
      REQUIRE(ids[size_t(q) * k + j] == wi && sc[size_t(q) * k + j] == ws, "%s, grid %d x %d tiles, k=%d nq=%d: query %d rank %d holds row %lld (%g), want %lld (%g)",
              name_of(d), grid, tiles_per_cta, k, nq, q, j, (long long)ids[size_t(q) * k + j], sc[size_t(q) * k + j], (long long)wi, ws);
    }
    float mn = INFINITY, mx = -INFINITY;
    for (int64_t r = 0; r < rows; ++r) { mn = fminf(mn, scores[size_t(r) * kNQ + q]); mx = fmaxf(mx, scores[size_t(r) * kNQ + q]); }
    REQUIRE(mm[q * 2] == mn && mm[q * 2 + 1] == mx, "%s: (min, max) of query %d", name_of(d), q);
  }
  printf("ok  select warps <%d, %d>: %s, %lld rows on %d CTAs (%d tiles each), nq = %d, k = %d, pool %s, permutation %s, CTAs %s\n", KLIST, CAP, name_of(d),
         (long long)rows, grid, tiles_per_cta, nq, k, use_pool ? "on" : "off", perm_mul ? "on" : "off", g_concurrent_seed ? "interleaved" : "one after the other");
}

// rank continuation (crag_search_topk_after): pages of k ranks, each admitting only keys below the previous page's last
template <int KLIST, int CAP>
static void test_continuation(Data d, int grid, int tiles_per_cta, int nq, int k, int pages) {
  const int64_t rows = int64_t(grid) * tiles_per_cta * kTileRows - 17;
  std::vector<float> scores = make_scores(rows, d);
  std::vector<uint64_t> after;
  for (int page = 0; page < pages; ++page) {
    std::vector<int64_t> ids;
    std::vector<float> sc, mm;
    std::vector<uint64_t> last;
    run_pass<KLIST, CAP>(scores, rows, grid, nq, k, true, perm_multiplier(((rows + kTileRows - 1) / kTileRows) >> 1), 1,
                                 page ? after.data() : nullptr, ids, sc, mm, last);
    for (int q = 0; q < nq; ++q) {
      std::vector<uint64_t> want = exact_keys(scores, rows, q);
      for (int j = 0; j < k; ++j) {
        const size_t rank = size_t(page) * k + j;
        const int64_t wi = rank < want.size() ? int64_t(key_id(want[rank])) + 1000 : -1;
        REQUIRE(ids[size_t(q) * k + j] == wi, "continuation %s: page %d query %d rank %zu: row %lld, want %lld", name_of(d), page, q, rank,
                (long long)ids[size_t(q) * k + j], (long long)wi);
      }
    }
    after = last;
  }
  printf("ok  rank continuation <%d, %d>: %s, %lld rows, %d pages of %d ranks, nq = %d\n", KLIST, CAP, name_of(d), (long long)rows, pages, k, nq);
}

// score-all variant (crag_search_scores): every score stored, (min, max) per query
static void test_score_all(int grid, int tiles_per_cta, int nq) {
  const int64_t rows = int64_t(grid) * tiles_per_cta * kTileRows - 5;
  std::vector<float> scores = make_scores(rows, Data::Random);
  std::vector<float> out(size_t(nq) * rows, -7.f), part_mm(size_t(grid) * kNQ * 2, -5.f);
  g_src = MatrixScoreTiles{scores.data(), rows, nullptr};
  warp_emu::launch(grid, kSearchThreads, [&] {
    search_select_shell<16, 16, false, true>(int(rows), nq, 1, nullptr, nullptr, 0u, 0, nullptr, part_mm.data(), ScoreArgs{out.data(), rows, nullptr, nullptr, 0});
  }, SelectSmem<16, 16>::bytes());
  for (int q = 0; q < nq; ++q) {
    float mn = INFINITY, mx = -INFINITY;
    for (int64_t r = 0; r < rows; ++r) {
      REQUIRE(out[size_t(q) * rows + r] == scores[size_t(r) * kNQ + q], "score-all: row %lld query %d", (long long)r, q);
      mn = fminf(mn, scores[size_t(r) * kNQ + q]); mx = fmaxf(mx, scores[size_t(r) * kNQ + q]);
    }
    float a = INFINITY, b = -INFINITY;
    for (int p = 0; p < grid; ++p) { a = fminf(a, part_mm[(size_t(p) * kNQ + q) * 2]); b = fmaxf(b, part_mm[(size_t(p) * kNQ + q) * 2 + 1]); }
    REQUIRE(a == mn && b == mx, "score-all (min, max) query %d", q);
  }
  printf("ok  score-all variant: %lld rows on %d CTAs, nq = %d: every score stored, (min, max) exact\n", (long long)rows, grid, nq);
}

// assignment mode (crag_ivf_assign): one score-all pass per block of 32 centroids, each row keeping its running argmax;
// three score levels, so most rows tie their best score across blocks -- the smallest centroid id must win
static void test_assign(int grid, int tiles_per_cta, int nlist) {
  const int64_t rows = int64_t(grid) * tiles_per_cta * kTileRows - 11;
  std::vector<float> all(size_t(rows) * nlist);
  for (auto& v : all) v = float(int(rng() % 3)) * 0.1f;
  std::vector<float> best_score(rows, -7.f), part_mm(size_t(grid) * kNQ * 2, -5.f);
  std::vector<int32_t> best_id(rows, -7);
  for (int q0 = 0; q0 < nlist; q0 += kNQ) {
    const int nqc = std::min(kNQ, nlist - q0);
    std::vector<float> block(size_t(rows) * kNQ, 0.f);
    for (int64_t r = 0; r < rows; ++r)
      for (int q = 0; q < nqc; ++q) block[size_t(r) * kNQ + q] = all[size_t(r) * nlist + q0 + q];
    g_src = MatrixScoreTiles{block.data(), rows, nullptr};
    warp_emu::launch(grid, kSearchThreads, [&] {
      search_select_shell<16, 16, false, true>(int(rows), nqc, 1, nullptr, nullptr, 0u, 0, nullptr, part_mm.data(),
                                               ScoreArgs{nullptr, 0, best_score.data(), best_id.data(), q0});
    }, SelectSmem<16, 16>::bytes());
  }
  int64_t tied_across_blocks = 0;
  for (int64_t r = 0; r < rows; ++r) {
    int want = 0;
    for (int c = 1; c < nlist; ++c)
      if (all[size_t(r) * nlist + c] > all[size_t(r) * nlist + want]) want = c;
    const float ws = all[size_t(r) * nlist + want];
    for (int c = kNQ; c < nlist; ++c) tied_across_blocks += (want < kNQ && all[size_t(r) * nlist + c] == ws) ? 1 : 0;
    REQUIRE(best_id[r] == want && __float_as_uint(best_score[r]) == __float_as_uint(ws),
            "assign: row %lld holds centroid %d (%g), want %d (%g)", (long long)r, best_id[r], best_score[r], want, ws);
  }
  REQUIRE(tied_across_blocks > 0, "test bug: no row ties its best score across centroid blocks");
  printf("ok  assign mode: %lld rows on %d CTAs, %d centroids in %d blocks: running argmax exact, ties to the smaller id\n",
         (long long)rows, grid, nlist, (nlist + kNQ - 1) / kNQ);
}

// IVF variant (crag_ivf_search): the plan kernel builds query masks / coarse terms / the work-list, the select warps walk
// the work-list, add the coarse term and skip the queries that do not probe the tile's list; model = oracle/ivf_oracle.py
// restated over the given residual scores: candidates of query q = the real rows of the lists it probes, score =
// residual score + coarse score (fp32, in that order), best k by (score desc, stored row asc)
template <int KLIST, int CAP>
static void test_ivf(int nlist, int nprobe, int grid, int nq, int k) {
  std::vector<int32_t> list_rows(nlist), tile_start(nlist + 1, 0);
  for (int l = 0; l < nlist; ++l) {
    list_rows[l] = (rng() % 7 == 0) ? 0 : 1 + int(rng() % 400);
    tile_start[l + 1] = tile_start[l] + (list_rows[l] + kTileRows - 1) / kTileRows;
  }
  const int64_t stored = int64_t(tile_start[nlist]) * kTileRows;
  std::vector<float> resid = make_scores(stored, Data::Random);
  std::vector<int64_t> probed(size_t(nq) * nprobe);
  std::vector<float> pscore(size_t(nq) * nprobe);
  for (int q = 0; q < nq; ++q) {
    std::vector<int> perm(nlist);
    for (int l = 0; l < nlist; ++l) perm[l] = l;
    std::shuffle(perm.begin(), perm.end(), rng);
    for (int j = 0; j < nprobe; ++j) { probed[size_t(q) * nprobe + j] = perm[j]; pscore[size_t(q) * nprobe + j] = float(double(rng() % 1000) / 1000.0); }
  }
  std::vector<uint32_t> mask(nlist, 0u);
  std::vector<float> coarse(size_t(nlist) * kNQ, 0.f);
  std::vector<int4> work(size_t(tile_start[nlist]) + 1);
  int n_work = 0;
  warp_emu::launch(1, 1024, [&] {
    ivf_plan_kernel(probed.data(), pscore.data(), nq, nprobe, nlist, tile_start.data(), list_rows.data(), mask.data(), coarse.data(), work.data(), &n_work);
  });
  std::vector<uint64_t> part_keys(size_t(grid) * kNQ * k, 0xDEADull), pool(size_t(grid) * kPoolSlots * kNQ, 0ull);
  std::vector<float> part_mm(size_t(grid) * kNQ * 2, -5.f);
  g_src = MatrixScoreTiles{resid.data(), stored, work.data()};
  const IvfArgs args{work.data(), &n_work, mask.data(), coarse.data()};
  warp_emu::launch(grid, kSearchThreads, [&] {
    search_select_shell<KLIST, CAP, true, false>(0, nq, k, nullptr, pool.data(), 0u, 0, part_keys.data(), part_mm.data(), args);
  }, SelectSmem<KLIST, CAP>::bytes());
  std::vector<int64_t> ids(size_t(nq) * k, -5);
  std::vector<float> sc(size_t(nq) * k, -5.f), mm(size_t(nq) * 2, -5.f);
  warp_emu::launch(nq, 128, [&] {
    merge_topk_kernel<KLIST, CAP, false>(part_keys.data(), nullptr, nullptr, part_mm.data(), grid, kNQ, nq, k, 0, 0, 0, 0, ids.data(), sc.data(), mm.data(), nullptr);
  });
  for (int q = 0; q < nq; ++q) {
    std::vector<uint64_t> want;
    float mn = INFINITY, mx = -INFINITY;
    for (int j = 0; j < nprobe; ++j) {
      const int l = int(probed[size_t(q) * nprobe + j]);
      for (int r = 0; r < list_rows[l]; ++r) {
        const int64_t row = int64_t(tile_start[l]) * kTileRows + r;
        const float s = resid[size_t(row) * kNQ + q] + pscore[size_t(q) * nprobe + j];
        want.push_back(make_key(s, uint32_t(row)));
        mn = fminf(mn, s); mx = fmaxf(mx, s);
      }
    }
    std::sort(want.begin(), want.end(), std::greater<uint64_t>());
    for (int j = 0; j < k; ++j) {
      const int64_t wi = j < int(want.size()) ? int64_t(key_id(want[j])) : -1;
      const float ws = j < int(want.size()) ? key_score(want[j]) : -INFINITY;
      REQUIRE(ids[size_t(q) * k + j] == wi && sc[size_t(q) * k + j] == ws, "ivf nlist=%d nprobe=%d k=%d: query %d rank %d: stored row %lld (%g), want %lld (%g)",
              nlist, nprobe, k, q, j, (long long)ids[size_t(q) * k + j], sc[size_t(q) * k + j], (long long)wi, ws);
    }
    if (!want.empty()) REQUIRE(mm[q * 2] == mn && mm[q * 2 + 1] == mx, "ivf (min, max) of query %d", q);
  }
  printf("ok  IVF variant <%d, %d>: %d lists (%lld stored rows), %d probes, %d work tiles on %d CTAs, nq = %d, k = %d\n", KLIST, CAP, nlist,
         (long long)stored, nprobe, n_work, grid, nq, k);
}

int main(int argc, char** argv) {
  if (argc > 1 && std::string(argv[1]) == "ties") {     // the tie-heavy cases only (what the mutation tests run)
    test_topk<64, 64>(Data::AllEqual, 4, 8, 33, 32, 10, true, 37u, 3);
    test_topk<64, 64>(Data::FewLevels, 4, 8, 33, 32, 10, true, 37u, 3);
    test_continuation<128, 128>(Data::FewLevels, 4, 6, 32, 128, 3);
    test_continuation<64, 64>(Data::AllEqual, 3, 4, 3, 50, 5);
    printf("ALL OK\n");
    return 0;
  }
  if (argc > 2 && std::string(argv[1]) == "fuzz") {     // fuzz FIRST_SEED COUNT: random regimes, CTAs interleaved by seed
    const uint64_t first = strtoull(argv[2], nullptr, 10), count = argc > 3 ? strtoull(argv[3], nullptr, 10) : 10;
    for (uint64_t seed = first; seed < first + count; ++seed) {
      rng.seed(seed * 7919);
      g_concurrent_seed = getenv("FUZZ_SEQUENTIAL") ? 0 : seed;
      const Data d = Data(rng() % 5);
      const int regime = int(rng() % 6);
      const int ragged = int(rng() % 128), nq = (rng() % 3 == 0) ? 1 + int(rng() % 32) : 32;
      // kAutoPerm: the multiplier search.cu's perm_multiplier() picks for the drawn shape (it must be coprime to the
      // number of tile groups -- an arbitrary constant would visit some tiles twice and others never)
      if (regime == 0) test_topk<64, 64>(d, 2 + int(rng() % 10), 3 + int(rng() % 20), ragged, nq, 1 + int(rng() % 16), true, kAutoPerm, int(rng() % 4));
      else if (regime == 1) test_topk<64, 64>(d, 20 + int(rng() % 60), 3 + int(rng() % 6), ragged, nq, 17 + int(rng() % 48), true, kAutoPerm, int(rng() % 3));
      else if (regime == 2) test_topk<128, 128>(d, 130 + int(rng() % 30), 3 + int(rng() % 3), ragged, nq, 65 + int(rng() % 40), true, kAutoPerm, 1);
      else if (regime == 3) test_topk<128, 128>(d, 4 + int(rng() % 12), 4 + int(rng() % 12), ragged, nq, 100 + int(rng() % 29), true, kAutoPerm, int(rng() % 3));
      else if (regime == 4) {
        if (rng() % 2) test_continuation<128, 128>(d, 2 + int(rng() % 6), 2 + int(rng() % 8), nq, 65 + int(rng() % 64), 2 + int(rng() % 3));
        else test_continuation<64, 64>(d, 2 + int(rng() % 6), 2 + int(rng() % 8), nq, 1 + int(rng() % 64), 2 + int(rng() % 4));
      } else {
        if (rng() % 2) test_ivf<128, 128>(8 + int(rng() % 200), 1 + int(rng() % 8), 1 + int(rng() % 9), nq, 65 + int(rng() % 64));
        else test_ivf<64, 64>(8 + int(rng() % 200), 1 + int(rng() % 8), 1 + int(rng() % 9), nq, 1 + int(rng() % 64));
      }
    }
    printf("ALL OK\n");
    return 0;
  }
  const int scale = argc > 1 ? atoi(argv[1]) : 1;
  // the headline regime: k = 10, long scans (refresh schedule 2 / 12 / 48 / 128), every data set
  for (Data d : {Data::Random, Data::Ascending, Data::AllEqual, Data::FewLevels, Data::PlantedTail})
    test_topk<64, 64>(d, 4, 50 * scale, 33, 32, 10, true, 37u, 3);
  test_topk<64, 64>(Data::Random, 3, 132, 0, 32, 10, true, 0u, 0);          // no permutation; refresh at tile 128
  test_topk<64, 64>(Data::Random, 3, 5, 100, 7, 64, false, 0u, 0);          // no pool (short scans), nq < 32, k = KLIST
  test_topk<64, 64>(Data::FewLevels, 5, 9, 1, 1, 1, true, 3u, 1);           // k = 1, one query
  // config 4's regime: k = 100 on the 128-key selector, batch-of-8 bisection floor (k <= 0.8 x CTAs) on 148 CTAs
  test_topk<128, 128>(Data::Random, 148, 4, 77, 32, 100, true, 11u, 1);
  test_topk<128, 128>(Data::Ascending, 40, 10, 0, 32, 32, true, 7u, 2);     // 16 < k <= 0.8 x 40 CTAs
  // k > 0.8 x CTAs: all four keys per CTA pooled (pooled_kth_key), k = 128
  test_topk<128, 128>(Data::Ascending, 8, 20, 5, 32, 128, true, 3u, 2);
  test_topk<128, 128>(Data::Random, 2, 1, 100, 32, 100, false, 0u, 0);       // fewer rows than k per CTA list: -1 padding
  // the same regimes with all CTAs resident together, in two random interleavings each
  for (uint64_t seed : {11ull, 12ull}) {
    g_concurrent_seed = seed;
    test_topk<64, 64>(seed == 11 ? Data::Random : Data::FewLevels, 6, 30, 9, 32, 10, true, 37u, 3);
    test_topk<128, 128>(seed == 11 ? Data::AllEqual : Data::PlantedTail, 148, 4, 77, 32, 100, true, 11u, 1);
    test_topk<128, 128>(seed == 11 ? Data::FewLevels : Data::Random, 8, 20, 5, 32, 128, true, 3u, 2);
  }
  g_concurrent_seed = 0;
  test_continuation<128, 128>(Data::Random, 4, 12, 5, 128, 4);
  test_continuation<128, 128>(Data::FewLevels, 4, 6, 32, 128, 3);
  test_continuation<64, 64>(Data::AllEqual, 3, 4, 3, 50, 5);
  test_ivf<128, 128>(64, 8, 5, 32, 100);
  test_ivf<64, 64>(200, 16, 7, 9, 10);
  test_ivf<128, 128>(12, 12, 3, 32, 128);      // nprobe = nlist: exact search over every list
  test_score_all(5, 7, 32);
  test_score_all(2, 3, 9);
  test_assign(3, 4, 103);
  printf("ALL OK\n");
  return 0;
}
