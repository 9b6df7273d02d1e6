// Constants and argument structs of the shard scan kernel (search.cu), in a header of their own so that tests/warp_emu
// can build the select warps (select_warps.cuh) for the host.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

#include "ivf_kernels.cuh"   // kTileRows
#include "pool_floor.cuh"    // kNQ

namespace crag {

constexpr int kBlockK = 64;     // bf16 per 128-byte swizzle row
constexpr int kStageBytes = kTileRows * kBlockK * 2;  // 16 KB
constexpr int kQBlockBytes = kNQ * kBlockK * 2;       // 4 KB
// One pipeline stage: a corpus box and the query block's slice of the same 64 columns.  Streaming the query slices
// (L2 hits after the first tile) instead of keeping the whole [32, dim] block resident frees 64 KB at dim = 1024 for
// stages and score tiles.
constexpr int kStageTotalBytes = kStageBytes + kQBlockBytes;  // 20 KB
// warps 0-3 select, warps 4-7 the wgmma warpgroup, warp 8 the TMA producer
constexpr int kSearchThreads = 288;
constexpr int kEpiThreads = 128;
constexpr int kMmaWarp0 = 4;
constexpr int kProducerWarp = 8;
// One score tile in shared memory: 128 rows x 32 fp32 scores, row r's score of query q at r * 32 + (q ^ (r % 32)) so
// that a select warp reading one row per lane hits 32 distinct banks.  The wgmma warpgroup's stores of its accumulator
// fragment (8 rows x 4 column pairs per warp instruction) still meet 4-way bank conflicts: 16 KB of stores per tile
// against 256 KB of corpus reads at dim 1024, so the scan stays HBM-bound.
constexpr int kScoreTileBytes = kTileRows * kNQ * 4;  // 16 KB
__host__ __device__ constexpr int score_slot(int row, int q) { return row * kNQ + (q ^ (row & 31)); }
// score-tile buffers: the scan may run this many tiles ahead of the select warps.  Together with the pipeline stages
// they fill what the 227 KB of shared memory leave beside the candidate lists.
constexpr int kAccStages = 4;

// IVF variant of the scan (BASELINE config 4; semantic: oracle/ivf_oracle.py): the shard holds bf16 RESIDUALS grouped
// by coarse list, every list padded to whole 128-row tiles, and a pass touches only the tiles of probed lists.
//   work[i]   = (first stored row of the tile, valid rows in it, list id, 0), written by ivf_plan_kernel
//   n_work    = number of work items (device scalar: the plan is built on the device, no host round trip)
//   list_mask = per list, bit q set when query q probes it; coarse[list * 32 + q] = q . c_list from the coarse pass
// The flat instantiations (IVF = false) take an empty struct instead and compile to the same SASS as before.
// r[q] for a runtime q without sending the score registers to local memory: a 5-level select tree on the bits of q
__device__ __forceinline__ uint32_t pick32(const uint32_t (&r)[32], int q) {
  uint32_t a[16], b[8], c[4], d[2];
#pragma unroll
  for (int i = 0; i < 16; ++i) a[i] = (q & 16) ? r[i + 16] : r[i];
#pragma unroll
  for (int i = 0; i < 8; ++i) b[i] = (q & 8) ? a[i + 8] : a[i];
#pragma unroll
  for (int i = 0; i < 4; ++i) c[i] = (q & 4) ? b[i + 4] : b[i];
#pragma unroll
  for (int i = 0; i < 2; ++i) d[i] = (q & 2) ? c[i + 2] : c[i];
  return (q & 1) ? d[1] : d[0];
}

struct IvfArgs {
  const int4* work;
  const int* n_work;
  const uint32_t* list_mask;
  const float* coarse;
};
struct NoIvfArgs {};
// Score-all variant (SCORES = true): the full-array contracts of the reference -- get_fact_scores returns the score
// of EVERY fact row (ComoRAG.py:937-948) and dense_passage_retrieval a permutation of ALL rows (:950-967, consumed
// rank by rank by PPR at :1034-1042).  Same TMA -> wgmma -> score-tile stream; the select warps write the fp32 scores
// (out[q * ld + row], one coalesced 128-byte store per warp and query) instead of running the selector.
struct ScoreArgs {
  float* out;
  int64_t ld;
  // assignment mode (best_id != nullptr): instead of storing the scores, each row keeps the running argmax over the
  // query blocks it has met -- the IVF build's "which centroid does this row belong to" (rows = corpus, centroids =
  // queries, 32 per pass).  A row is owned by one thread per pass and passes are stream-ordered: plain read-modify-write.
  float* best_score;
  int32_t* best_id;
  int32_t base_id;
};
template <bool IVF, bool SCORES> struct IvfParam { using type = NoIvfArgs; };
template <> struct IvfParam<true, false> { using type = IvfArgs; };
template <> struct IvfParam<false, true> { using type = ScoreArgs; };

// multiplier of the group permutation g -> (g * P) mod n_groups: near n_groups / golden ratio, coprime to n_groups
// (0 = identity / permutation off)
inline uint32_t perm_multiplier(int64_t num_tiles) {
  if (num_tiles < 4) return 0u;
  auto gcd = [](uint64_t a, uint64_t b) { while (b) { const uint64_t t = a % b; a = b; b = t; } return a; };
  uint64_t p = (uint64_t(double(num_tiles) * 0.6180339887498949) | 1ull);
  while (gcd(p, uint64_t(num_tiles)) != 1) p += 2;
  return uint32_t(p % uint64_t(num_tiles));
}

}  // namespace crag
