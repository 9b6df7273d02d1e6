// Whole kernels of the search path on emulated thread blocks (warp_emu.h), compiled from the headers the library itself
// includes (csrc/rank_kernels.cuh, merge_kernels.cuh):
//   rank     hist / scan / scatter kernels, driven pass by pass exactly as crag_rank_scores drives them, against
//            std::stable_sort -- the full permutation of ComoRAG.py:965-966 (descending score, ascending row on ties)
//   ivf      ivf_plan_kernel (query masks, coarse terms, work-list of probed tiles) and ivf_map_ids_kernel against a direct
//            restatement of oracle/ivf_oracle.py's plan
//   merge    merge_topk_kernel, both input layouts (per-CTA key lists; packed per-shard (id, score) records)
//   exchange finalize_exchange_kernel with `world` ranks, ONE OS THREAD PER RANK pushing into each other's buffers
//            through release / acquire flags, several calls in a row (slot parity reuse): every rank must end with the
//            same global answer, equal to the merge rule stated in plain C++ (score desc, then rank, then position)
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <random>
#include <thread>
#include <vector>

#include <cuda_runtime.h>   // the stub

#include "ivf_kernels.cuh"
#include "merge_kernels.cuh"
#include "rank_kernels.cuh"

using namespace crag;

static std::mt19937_64 rng(424242);

#define REQUIRE(cond, ...)                              \
  do {                                                  \
    if (!(cond)) {                                      \
      fprintf(stderr, "FAILED %s:%d: %s\n  ", __FILE__, __LINE__, #cond); \
      fprintf(stderr, __VA_ARGS__);                     \
      fprintf(stderr, "\n");                            \
      exit(1);                                          \
    }                                                   \
  } while (0)

static float random_score(int levels) {
  if (levels > 0) return float(int(rng() % levels)) / float(levels) - 0.3f;
  return float(double(rng() % 2000001) / 1e6 - 1.0);
}

// ------------------------------------------------------------------------------------------------------- rank
static void test_rank(int64_t n, int levels, bool specials) {
  std::vector<float> scores(n);
  for (auto& s : scores) s = random_score(levels);
  if (specials && n >= 8) {
    scores[0] = 0.0f; scores[1] = -0.0f; scores[2] = INFINITY; scores[3] = -INFINITY;
    scores[4] = 1e-42f; scores[5] = -1e-42f; scores[6] = scores[7];
  }
  warp_emu::Workspace ws(plan_sort(n).total, kWsAlign, 0xAB);
  const SortPlan p = plan_sort(n, ws.base);
  uint32_t* hist = p.hist;
  uint32_t* totals = hist + size_t(256) * p.n_warps;
  std::vector<int64_t> out_ids(n, -7);
  std::vector<float> out_scores(n, -7.f);
  const float* sc = scores.data();
  for (int pass = 0; pass < 4; ++pass) {          // the launch sequence of crag_rank_scores (rank_all.cu)
    const int shift = pass * 8;
    const uint32_t* kin = pass ? p.keys[(pass - 1) & 1] : nullptr;
    const uint32_t* vin = pass ? p.vals[(pass - 1) & 1] : nullptr;
    uint32_t* kout = p.keys[pass & 1];
    uint32_t* vout = p.vals[pass & 1];
    memset(totals, 0, 256 * 4);
    if (pass == 0) warp_emu::launch(p.grid, kSortThreads, [&] { hist_kernel<true>(sc, nullptr, n, p.run, p.n_warps, shift, hist, totals); });
    else warp_emu::launch(p.grid, kSortThreads, [&] { hist_kernel<false>(nullptr, kin, n, p.run, p.n_warps, shift, hist, totals); });
    warp_emu::launch(256, 256, [&] { scan_kernel(hist, totals, p.n_warps); });
    if (pass == 0) warp_emu::launch(p.grid, kSortThreads, [&] { scatter_kernel<true, false>(sc, nullptr, nullptr, n, p.run, p.n_warps, shift, hist, kout, vout, nullptr, nullptr); });
    else if (pass < 3) warp_emu::launch(p.grid, kSortThreads, [&] { scatter_kernel<false, false>(nullptr, kin, vin, n, p.run, p.n_warps, shift, hist, kout, vout, nullptr, nullptr); });
    else warp_emu::launch(p.grid, kSortThreads, [&] { scatter_kernel<false, true>(nullptr, kin, vin, n, p.run, p.n_warps, shift, hist, nullptr, nullptr, out_ids.data(), out_scores.data()); });
  }
  std::vector<int64_t> want(n);
  for (int64_t i = 0; i < n; ++i) want[i] = i;
  std::stable_sort(want.begin(), want.end(), [&](int64_t a, int64_t b) { return orderable_f32(scores[a]) > orderable_f32(scores[b]); });
  for (int64_t i = 0; i < n; ++i) {
    REQUIRE(out_ids[i] == want[i], "rank n=%lld levels=%d: position %lld holds row %lld, want %lld", (long long)n, levels,
            (long long)i, (long long)out_ids[i], (long long)want[i]);
    REQUIRE(__float_as_uint(out_scores[i]) == __float_as_uint(scores[want[i]]), "rank n=%lld: score bits at %lld", (long long)n, (long long)i);
  }
  printf("ok  rank kernels: n = %lld (%d warps, %d blocks), %s: permutation == stable descending sort, scores bit-equal\n",
         (long long)n, p.n_warps, p.grid, levels ? "heavy ties" : "random scores");
}

// -------------------------------------------------------------------------------------------------------- ivf
#include <map>
#include <set>
#include <tuple>
static void test_ivf_plan(int nlist, int nq, int nprobe) {
  std::vector<int32_t> list_rows(nlist), list_tile_start(nlist + 1, 0);
  for (int l = 0; l < nlist; ++l) {
    list_rows[l] = (rng() % 6 == 0) ? 0 : int(rng() % 700);               // some lists are empty
    list_tile_start[l + 1] = list_tile_start[l] + (list_rows[l] + kTileRows - 1) / kTileRows;
  }
  std::vector<int64_t> probed(size_t(nq) * nprobe);
  std::vector<float> pscore(size_t(nq) * nprobe);
  for (int q = 0; q < nq; ++q) {
    std::vector<int> perm(nlist);
    for (int l = 0; l < nlist; ++l) perm[l] = l;
    std::shuffle(perm.begin(), perm.end(), rng);
    for (int j = 0; j < nprobe; ++j) {
      const bool absent = j >= nlist || rng() % 11 == 0;                  // fewer than nprobe lists: id -1
      probed[size_t(q) * nprobe + j] = absent ? -1 : perm[j];
      pscore[size_t(q) * nprobe + j] = random_score(0);
    }
  }
  std::vector<uint32_t> mask(nlist, 0xFFFFFFFFu);
  std::vector<float> coarse(size_t(nlist) * kNQ, -77.f);
  std::vector<int4> work(size_t(list_tile_start[nlist]) + 1, int4{-1, -1, -1, -1});
  int n_work = -1;
  warp_emu::launch(1, 1024, [&] {
    ivf_plan_kernel(probed.data(), pscore.data(), nq, nprobe, nlist, list_tile_start.data(), list_rows.data(), mask.data(), coarse.data(), work.data(), &n_work);
  });
  std::vector<uint32_t> want_mask(nlist, 0u);
  std::map<std::pair<int, int>, float> want_coarse;
  for (int q = 0; q < nq; ++q)
    for (int j = 0; j < nprobe; ++j) {
      const int64_t l = probed[size_t(q) * nprobe + j];
      if (l < 0) continue;
      want_mask[l] |= 1u << q;
      want_coarse[{int(l), q}] = pscore[size_t(q) * nprobe + j];
    }
  std::set<std::tuple<int, int, int>> want_work, got_work;
  for (int l = 0; l < nlist; ++l) {
    REQUIRE(mask[l] == want_mask[l], "ivf plan: mask of list %d", l);
    if (!want_mask[l] || list_rows[l] <= 0) continue;
    for (int j = 0; j * kTileRows < list_rows[l]; ++j)
      want_work.insert({(list_tile_start[l] + j) * kTileRows, std::min(kTileRows, list_rows[l] - j * kTileRows), l});
  }
  for (auto& kv : want_coarse) REQUIRE(coarse[size_t(kv.first.first) * kNQ + kv.first.second] == kv.second, "ivf plan: coarse term list %d query %d", kv.first.first, kv.first.second);
  REQUIRE(n_work == int(want_work.size()), "ivf plan: %d work items, want %zu", n_work, want_work.size());
  for (int i = 0; i < n_work; ++i) got_work.insert({work[i].x, work[i].y, work[i].z});
  REQUIRE(got_work == want_work, "ivf plan: work-list differs (nlist %d nq %d nprobe %d)", nlist, nq, nprobe);
  // merged answer's stored-row ids -> original ids
  std::vector<int64_t> row_ids(1000), ids(300);
  for (size_t i = 0; i < row_ids.size(); ++i) row_ids[i] = (i % 9 == 0) ? -1 : int64_t(rng() % (int64_t(1) << 40));
  std::vector<int64_t> before(ids.size());
  for (size_t i = 0; i < ids.size(); ++i) before[i] = ids[i] = (i % 7 == 0) ? -1 : int64_t(rng() % row_ids.size());
  warp_emu::launch((unsigned(ids.size()) + 255) / 256, 256, [&] { ivf_map_ids_kernel(ids.data(), int(ids.size()), row_ids.data()); });
  for (size_t i = 0; i < ids.size(); ++i) REQUIRE(ids[i] == (before[i] >= 0 ? row_ids[before[i]] : -1), "ivf id map at %zu", i);
  printf("ok  ivf_plan_kernel + ivf_map_ids_kernel: nlist = %d, %d queries x %d probes, %d work items\n", nlist, nq, nprobe, n_work);
}

// ------------------------------------------------------------------------------------------------------ merge
// `parts` sorted lists of (score, local row) per query as the scan leaves them: part_keys[(p * kNQ + q) * k + j]
struct Partials {
  int parts, k;
  std::vector<uint64_t> keys;
  std::vector<float> minmax;
};
static Partials make_partials(int parts, int k, int levels, uint32_t row_base) {
  Partials P;
  P.parts = parts; P.k = k;
  P.keys.assign(size_t(parts) * kNQ * k, 0ull);
  P.minmax.assign(size_t(parts) * kNQ * 2, 0.f);
  for (int q = 0; q < kNQ; ++q) {
    uint32_t next_row = row_base + uint32_t(rng() % 1000);
    for (int p = 0; p < parts; ++p) {
      const int have = (rng() % 5 == 0) ? int(rng() % (k + 1)) : k;
      std::vector<uint64_t> mine;
      float mn = INFINITY, mx = -INFINITY;
      for (int j = 0; j < have; ++j) {
        const float s = random_score(levels);
        mine.push_back(make_key(s, next_row));
        next_row += 1 + uint32_t(rng() % 3);          // rows are distinct within a shard
        mn = fminf(mn, s); mx = fmaxf(mx, s);
      }
      std::sort(mine.begin(), mine.end(), std::greater<uint64_t>());
      for (int j = 0; j < have; ++j) P.keys[(size_t(p) * kNQ + q) * k + j] = mine[j];
      P.minmax[(size_t(p) * kNQ + q) * 2 + 0] = mn - float(rng() % 100) / 100.f;   // (min, max) cover ALL rows, not only the kept ones
      P.minmax[(size_t(p) * kNQ + q) * 2 + 1] = mx;
    }
  }
  return P;
}
static std::vector<uint64_t> best_keys(const Partials& P, int q) {
  std::vector<uint64_t> all;
  for (int p = 0; p < P.parts; ++p)
    for (int j = 0; j < P.k; ++j)
      if (P.keys[(size_t(p) * kNQ + q) * P.k + j]) all.push_back(P.keys[(size_t(p) * kNQ + q) * P.k + j]);
  std::sort(all.begin(), all.end(), std::greater<uint64_t>());
  if (int(all.size()) > P.k) all.resize(P.k);
  return all;
}

template <int KLIST, int CAP>
static void test_merge_keys(int rounds) {
  for (int r = 0; r < rounds; ++r) {
    const int k = 1 + int(rng() % KLIST), parts = 1 + int(rng() % 20), nq = 1 + int(rng() % kNQ);
    const int64_t row_offset = int64_t(rng() % 5) * 1000000000ll;
    Partials P = make_partials(parts, k, (r % 2) ? 3 : 0, 0);
    std::vector<int64_t> ids(size_t(nq) * k, -5);
    std::vector<float> sc(size_t(nq) * k, -5.f), mm(size_t(nq) * 2, -5.f);
    std::vector<uint64_t> last(nq, 1);
    warp_emu::launch(nq, 128, [&] {
      merge_topk_kernel<KLIST, CAP, false>(P.keys.data(), nullptr, nullptr, P.minmax.data(), parts, kNQ, nq, k, row_offset, 0, 0, 0,
                                           ids.data(), sc.data(), mm.data(), last.data());
    });
    for (int q = 0; q < nq; ++q) {
      std::vector<uint64_t> want = best_keys(P, q);
      for (int j = 0; j < k; ++j) {
        const int64_t wi = j < int(want.size()) ? int64_t(key_id(want[j])) + row_offset : -1;
        const float ws = j < int(want.size()) ? key_score(want[j]) : -INFINITY;
        REQUIRE(ids[size_t(q) * k + j] == wi && sc[size_t(q) * k + j] == ws, "merge<%d,%d> keys: k=%d parts=%d q=%d rank %d", KLIST, CAP, k, parts, q, j);
      }
      REQUIRE(last[q] == (int(want.size()) == k ? want[k - 1] : 0ull), "merge last_keys q=%d", q);
      float mn = INFINITY, mx = -INFINITY;
      for (int p = 0; p < parts; ++p) { mn = fminf(mn, P.minmax[(size_t(p) * kNQ + q) * 2]); mx = fmaxf(mx, P.minmax[(size_t(p) * kNQ + q) * 2 + 1]); }
      REQUIRE(mm[q * 2] == mn && mm[q * 2 + 1] == mx, "merge minmax q=%d", q);
    }
  }
  printf("ok  merge_topk_kernel<%d, %d, keys>: %d random (k, parts, nq)\n", KLIST, CAP, rounds);
}

// packed per-shard records (the all-gather layout): record p = [ids int64 nq*k][scores fp32 nq*k][minmax fp32 nq*2]
template <int KLIST, int CAP>
static void test_merge_pairs(int rounds) {
  for (int r = 0; r < rounds; ++r) {
    const int k = 1 + int(rng() % KLIST), parts = 1 + int(rng() % 8), nq = 1 + int(rng() % kNQ);
    const size_t rec = ((size_t(nq) * k * 12 + size_t(nq) * 8 + 15) / 16) * 16;
    std::vector<uint8_t> buf(rec * parts, 0);
    struct Cand { float s; int64_t id; int p, j; };
    std::vector<std::vector<Cand>> cands(nq);
    const int levels = (r % 2) ? 3 : 0;
    for (int p = 0; p < parts; ++p) {
      int64_t* ids = reinterpret_cast<int64_t*>(buf.data() + rec * p);
      float* sc = reinterpret_cast<float*>(buf.data() + rec * p + size_t(nq) * k * 8);
      float* mm = reinterpret_cast<float*>(buf.data() + rec * p + size_t(nq) * k * 12);
      for (int q = 0; q < nq; ++q) {
        const int have = (rng() % 4 == 0) ? int(rng() % (k + 1)) : k;
        std::vector<float> s(have);
        for (auto& x : s) x = random_score(levels);
        std::sort(s.begin(), s.end(), std::greater<float>());
        for (int j = 0; j < k; ++j) {
          ids[size_t(q) * k + j] = j < have ? int64_t(p) * 1000000 + int64_t(rng() % 1000) * 1000 + j : -1;
          sc[size_t(q) * k + j] = j < have ? s[j] : -INFINITY;
          if (j < have) cands[q].push_back({s[j], ids[size_t(q) * k + j], p, j});
        }
        mm[q * 2] = have ? s[have - 1] - 0.5f : INFINITY;
        mm[q * 2 + 1] = have ? s[0] : -INFINITY;
      }
    }
    std::vector<int64_t> ids(size_t(nq) * k, -5);
    std::vector<float> sc(size_t(nq) * k, -5.f), mm(size_t(nq) * 2, -5.f);
    const int64_t* in_ids = reinterpret_cast<const int64_t*>(buf.data());
    const float* in_sc = reinterpret_cast<const float*>(buf.data() + size_t(nq) * k * 8);
    const float* in_mm = reinterpret_cast<const float*>(buf.data() + size_t(nq) * k * 12);
    warp_emu::launch(nq, 128, [&] {
      merge_topk_kernel<KLIST, CAP, true>(nullptr, in_sc, in_ids, in_mm, parts, nq, nq, k, 0, int64_t(rec), int64_t(rec), int64_t(rec),
                                          ids.data(), sc.data(), mm.data(), nullptr);
    });
    for (int q = 0; q < nq; ++q) {
      auto& c = cands[q];
      std::stable_sort(c.begin(), c.end(), [](const Cand& a, const Cand& b) {      // score desc, then (part, position)
        if (orderable_f32(a.s) != orderable_f32(b.s)) return orderable_f32(a.s) > orderable_f32(b.s);
        return a.p != b.p ? a.p < b.p : a.j < b.j;
      });
      for (int j = 0; j < k; ++j) {
        const int64_t wi = j < int(c.size()) ? c[j].id : -1;
        const float ws = j < int(c.size()) ? c[j].s : -INFINITY;
        REQUIRE(ids[size_t(q) * k + j] == wi && sc[size_t(q) * k + j] == ws, "merge<%d,%d> pairs: k=%d parts=%d q=%d rank %d: id %lld want %lld",
                KLIST, CAP, k, parts, q, j, (long long)ids[size_t(q) * k + j], (long long)wi);
      }
    }
  }
  printf("ok  merge_topk_kernel<%d, %d, packed records>: %d random (k, parts, nq)\n", KLIST, CAP, rounds);
}

// --------------------------------------------------------------------------------------------------- exchange
// Every rank is an OS thread that runs ALL its calls back to back (no join between calls): a fast rank is already
// pushing call c + 1 (the other slot parity) while a slow one still merges call c, as on the GPUs.
template <int KLIST, int CAP>
static void test_exchange(int world, int k, int nq, int calls, int slow_reader_nap_us = 300) {
  const size_t xbytes = xchg_total_bytes(world);
  std::vector<std::vector<uint64_t>> xbuf(world, std::vector<uint64_t>(xbytes / 8 + 1, 0ull));   // zero-filled once
  std::vector<uint64_t> peer_table(world);
  for (int r = 0; r < world; ++r) peer_table[r] = reinterpret_cast<uint64_t>(xbuf[r].data());
  std::vector<std::vector<uint64_t>> epochs(world, std::vector<uint64_t>(32, 0ull));
  std::vector<int> status(world, 0);
  struct Out { std::vector<int64_t> ids; std::vector<float> sc, mm; };
  std::vector<int64_t> offs(world);
  for (int r = 0; r < world; ++r) offs[r] = int64_t(r) * 3000000000ll;     // global ids beyond 2^32: the id widening matters
  std::vector<std::vector<Partials>> P(calls);                             // [call][rank]
  std::vector<std::vector<Out>> out(calls, std::vector<Out>(world));
  std::vector<std::vector<int>> nap_us(calls, std::vector<int>(world, 0));
  for (int call = 0; call < calls; ++call) {
    const int parts = 1 + int(rng() % 6);
    for (int r = 0; r < world; ++r) {
      P[call].push_back(make_partials((call == 1 && r == world - 1) ? 0 : parts, k, (call % 2) ? 2 : 0, 0));   // one call: an EMPTY last shard
      out[call][r].ids.assign(size_t(nq) * k, -5); out[call][r].sc.assign(size_t(nq) * k, -5.f); out[call][r].mm.assign(size_t(nq) * 2, -5.f);
      nap_us[call][r] = (rng() % 3 == 0) ? int(rng() % 2000) : 0;          // ranks drift apart
    }
  }
  std::vector<std::thread> th;
  for (int r = 0; r < world; ++r) {
    th.emplace_back([&, r] {
      // the last rank is slow exactly where it hurts: it dawdles before reading the records its peers pushed, while
      // they run ahead into the next call (which must use the OTHER slot parity and cannot pass the call after that)
      warp_emu::nap_us() = (r == world - 1) ? slow_reader_nap_us : 0;
      for (int call = 0; call < calls; ++call) {
        if (nap_us[call][r]) std::this_thread::sleep_for(std::chrono::microseconds(nap_us[call][r]));
        Out& o = out[call][r];
        const Partials& mine = P[call][r];
        warp_emu::launch(nq, 128, [&] {
          finalize_exchange_kernel<KLIST, CAP>(mine.keys.data(), mine.minmax.data(), mine.parts, nq, k, offs[r], peer_table.data(), r, world,
                                               epochs[r].data(), &status[r], o.ids.data(), o.sc.data(), o.mm.data());
        });
      }
    });
  }
  for (auto& t : th) t.join();
  for (int r = 0; r < world; ++r) REQUIRE(status[r] == 0, "exchange: rank %d reported a missing peer record", r);
  for (int call = 0; call < calls; ++call) {
    for (int q = 0; q < nq; ++q) {
      struct Cand { float s; int64_t id; int r, j; };
      std::vector<Cand> c;
      float mn = INFINITY, mx = -INFINITY;
      for (int r = 0; r < world; ++r) {
        const Partials& pr = P[call][r];
        std::vector<uint64_t> b = best_keys(pr, q);
        for (int j = 0; j < int(b.size()); ++j) c.push_back({key_score(b[j]), int64_t(key_id(b[j])) + offs[r], r, j});
        for (int p = 0; p < pr.parts; ++p) { mn = fminf(mn, pr.minmax[(size_t(p) * kNQ + q) * 2]); mx = fmaxf(mx, pr.minmax[(size_t(p) * kNQ + q) * 2 + 1]); }
      }
      std::stable_sort(c.begin(), c.end(), [](const Cand& a, const Cand& b) {
        if (orderable_f32(a.s) != orderable_f32(b.s)) return orderable_f32(a.s) > orderable_f32(b.s);
        return a.r != b.r ? a.r < b.r : a.j < b.j;
      });
      for (int r = 0; r < world; ++r) {
        const Out& o = out[call][r];
        for (int j = 0; j < k; ++j) {
          const int64_t wi = j < int(c.size()) ? c[j].id : -1;
          const float ws = j < int(c.size()) ? c[j].s : -INFINITY;
          REQUIRE(o.ids[size_t(q) * k + j] == wi && o.sc[size_t(q) * k + j] == ws,
                  "exchange world=%d call=%d: rank %d q=%d rank-in-answer %d: id %lld want %lld", world, call, r, q, j,
                  (long long)o.ids[size_t(q) * k + j], (long long)wi);
        }
        REQUIRE(o.mm[q * 2] == mn && o.mm[q * 2 + 1] == mx, "exchange minmax world=%d call=%d rank %d q=%d", world, call, r, q);
      }
    }
  }
  for (int r = 0; r < world; ++r)
    for (int q = 0; q < nq; ++q) REQUIRE(epochs[r][q] == uint64_t(calls), "exchange epoch counter rank %d q=%d", r, q);
  printf("ok  finalize_exchange_kernel<%d, %d>: world = %d (one OS thread per rank), k = %d, nq = %d, %d calls back to back: every rank == merge rule\n",
         KLIST, CAP, world, k, nq, calls);
}

int main(int argc, char** argv) {
  const int scale = argc > 1 ? atoi(argv[1]) : 1;
  test_rank(1, 0, false);
  test_rank(4097, 0, true);
  test_rank(6000, 3, true);
  if (scale > 1) test_rank(20000, 5, true);
  test_ivf_plan(64, 32, 8);
  test_ivf_plan(4096, 32, 32);
  test_ivf_plan(10, 5, 16);
  test_merge_keys<32, 32>(6 * scale);
  test_merge_keys<64, 64>(6 * scale);
  test_merge_keys<128, 128>(6 * scale);
  test_merge_pairs<32, 32>(6 * scale);
  test_merge_pairs<64, 64>(6 * scale);
  test_merge_pairs<128, 128>(6 * scale);
  // nq = 1: the emulator runs a launch's blocks one after the other, so only with a single block per call can a fast
  // rank be a whole call ahead of a slow one that still reads -- the situation the two slot parities exist for
  test_exchange<64, 64>(3, 20, 1, 24, 4000);
  test_exchange<32, 32>(2, 10, 32, 12);
  test_exchange<64, 64>(4, 50, 7, 10);
  test_exchange<128, 128>(8, 100, 5, 8);
  printf("ALL OK\n");
  return 0;
}
