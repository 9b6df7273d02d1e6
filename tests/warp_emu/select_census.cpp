// Census of what the select warps of search_topk_kernel DO at a given shape, by running them on the CPU emulator
// (select_shell.h): how many warp shuffles (the bitonic sorts), warp reductions (the pooled-floor bisections), ballots
// and shared-memory atomics (candidate reservations) and named barriers one select warp executes per scan.  Not a
// timing -- an instruction-class count that says where a fixed cost can come from.
//   select_census ROWS K [NQ [CONCURRENT]]   e.g. 1250000 100 32 1   (one rank's shard of the 8-GPU split, config 4's k)
// Random unit-variance scores (the regime of a random corpus: admissions are rare once the floor has converged).
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "select_shell.h"

using namespace crag;

template <int KLIST, int CAP>
static void census(int64_t rows, int k, int nq, int grid, bool concurrent) {
  std::mt19937_64 rng(5);
  std::normal_distribution<float> nd(0.f, 0.03125f);     // q . x of unit vectors at dim 1024
  std::vector<float> scores(size_t(rows) * kNQ);
  for (auto& v : scores) v = nd(rng);
  std::vector<uint64_t> part_keys(size_t(grid) * kNQ * k), pool(size_t(grid) * kPoolSlots * kNQ, 0ull);
  std::vector<float> part_mm(size_t(grid) * kNQ * 2);
  g_src = MatrixScoreTiles{scores.data(), rows, nullptr};
  const int64_t tiles = (rows + kTileRows - 1) / kTileRows;
  const int shift = 3;
  const uint32_t perm = perm_multiplier(tiles >> shift);
  warp_emu::census() = warp_emu::Census{};
  auto scan = [&] {
    search_select_shell<KLIST, CAP>(int(rows), nq, k, nullptr, pool.data(), perm, shift, part_keys.data(), part_mm.data(), NoIvfArgs{});
  };
  if (concurrent) warp_emu::launch_concurrent(grid, kSearchThreads, scan, SelectSmem<KLIST, CAP>::bytes(), 7);
  else warp_emu::launch(grid, kSearchThreads, scan, SelectSmem<KLIST, CAP>::bytes());
  const warp_emu::Census c = warp_emu::census();
  const double warps = double(grid) * 4.0, lanes = warps * 32.0;
  const double tiles_per_cta = double(tiles) / grid;
  // a 256-key sort (KLIST + CAP = 256) is 15 cross-lane stages x 8 keys x 2 shuffles = 240 shuffles per lane, a 128-key
  // sort 120; the (min, max) reduction at the end adds 32 x 5 x 2 = 320 per lane
  const double shf = double(c.shuffles) / lanes;
  printf("{\"rows\": %lld, \"k\": %d, \"nq\": %d, \"ctas\": %d, \"ctas_run\": \"%s\", \"tiles_per_cta\": %.1f, \"selector\": \"<%d, %d>\",\n"
         " \"per_select_warp\": {\"shuffles_per_lane\": %.0f, \"equivalent_%d_key_sorts\": %.1f, \"warp_reductions\": %.0f, \"ballots\": %.0f,\n"
         "                     \"shared_atomics_per_warp\": %.0f, \"named_barriers_per_thread\": %.0f}}\n",
         (long long)rows, k, nq, grid, concurrent ? "interleaved (all resident)" : "one after the other", tiles_per_cta, KLIST, CAP, shf, KLIST + CAP, (shf - 320.0) / (KLIST + CAP == 256 ? 240.0 : 120.0),
         double(c.reductions) / lanes, double(c.ballots) / lanes, double(c.atomics) / warps, double(c.named_barriers) / (warps * 32.0));
}

int main(int argc, char** argv) {
  const int64_t rows = argc > 1 ? atoll(argv[1]) : 1250000;
  const int k = argc > 2 ? atoi(argv[2]) : 100;
  const int nq = argc > 3 ? atoi(argv[3]) : 32;
  const bool concurrent = argc > 4 && atoi(argv[4]) != 0;     // all 148 CTAs resident together, as on the GPU
  if (k <= 64) census<64, 64>(rows, k, nq, 148, concurrent);
  else census<128, 128>(rows, k, nq, 148, concurrent);
  return 0;
}
