// Pooled admission floor of the shard scan (search.cu): the warp-level routines that turn the keys all CTAs have
// published so far into a per-query floor key.  Pure SIMT code -- loads, compares, warp reductions -- with no
// wgmma / TMA / mbarrier in it, kept in its own header so that tests/warp_emu can compile exactly these functions
// for the host (32 emulated lanes) and check the one property exactness rests on: at least k published keys are at
// or above the floor a refresh returns, so no row with a smaller key can belong to the shard's top-k.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace crag {

constexpr int kNQ = 32;         // wgmma N: queries per pass
constexpr int kTileRows = 128;  // corpus rows per tile (two wgmma M = 64 halves)

// Pooled admission floor.  Every CTA publishes its current best kPoolM KEYS per query (after each flush of that
// query's candidate buffer) in pool[cta][m][q] (packed u64 keys, 0 = nothing yet; query-contiguous so a warp reads
// one CTA's entry for all 32 queries as a single 256-byte line).  Published keys belong to distinct rows of THIS
// shard (one CTA's j-th best key only ever improves, so values read at different times still stand for distinct rows
// at least that good).  A refresh turns them into a floor key per query.  For k <= 16 (after tiles 2, 12, 48 and
// every 128th): select warp w looks at the BEST key of the CTAs c = w (mod 4), each LANE keeps the kp = ceil(k / 4)
// largest of ITS query in registers (no cross-lane traffic at all), and the floor is the minimum over the four warps
// of their kp-th largest: every quarter of the CTAs then holds kp rows at or above it, i.e. at least k shard rows
// reach the floor and no row with a smaller key can rank in the top-k.  For larger k (after tiles 2, 4, 8, 16, 32
// and every 64th): the k-th largest of the CTAs' BEST keys by bisection, the eight queries a warp owns together
// (pooled_floor_batch8); only when k exceeds 0.8 x the CTA count do all four keys per CTA enter (pooled_kth_key).  All CTAs thus work with (almost) the global k-th best seen so far
// instead of their private one.  This replaces the separate sample pre-pass of round 1 (two launches fewer), cuts
// admissions at k = 100 by about two orders of magnitude, and -- because the floor is a full key, row id included --
// keeps tie-heavy corpora (duplicate rows) from flooding the selector with rows that only tie the k-th score.
constexpr int kPoolM = 4;
constexpr int kPoolSlots = kPoolM + 1;   // + slot kPoolM: the CTA's OWN k-th key (0 until its list is full)
constexpr int kPoolMaxCtas = 160;
constexpr int kPoolSmallK = 16;     // up to this k only each CTA's BEST key is pooled (37 CTA maxima per warp decide)

// kp-th largest (kp <= KP) of the keys query `q` (= lane) finds in the pool entries of CTAs w, w + 4, ...
template <int KP>
__device__ __forceinline__ uint64_t lane_kth_of_pool(const uint64_t* __restrict__ pool, int n_ctas, int w, int q,
                                                     int m_eff, int kp) {
  uint64_t t[KP];
#pragma unroll
  for (int j = 0; j < KP; ++j) t[j] = 0ull;
  auto offer = [&](uint64_t v) {
    if (v <= t[KP - 1]) return;
#pragma unroll
    for (int j = KP - 1; j >= 1; --j) {
      if (v > t[j - 1]) t[j] = t[j - 1];
      else if (v > t[j]) t[j] = v;
    }
    if (v > t[0]) t[0] = v;
  };
  constexpr int U = 8;   // loads in flight per lane (L2 latency ~1 us: the entries of 8 CTAs travel together)
  if (m_eff == 1) {
    for (int c0 = w; c0 < n_ctas; c0 += 4 * U) {
      uint64_t v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int c = c0 + 4 * u;
        v[u] = c < n_ctas ? __ldcg(pool + (size_t(c) * kPoolSlots) * kNQ + q) : 0ull;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) offer(v[u]);
    }
  } else {
    for (int c0 = w; c0 < n_ctas; c0 += 4 * (U / 4)) {
      uint64_t v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int c = c0 + 4 * (u / kPoolM);
        v[u] = c < n_ctas ? __ldcg(pool + (size_t(c) * kPoolSlots + (u % kPoolM)) * kNQ + q) : 0ull;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) offer(v[u]);
    }
  }
  uint64_t r = 0ull;
#pragma unroll
  for (int j = 0; j < KP; ++j) r = (j == kp - 1) ? t[j] : r;
  return r;
}

// k > kPoolSmallK: the owning warp of a query pools ALL CTAs' kPoolM keys (20 per lane) and finds their k-th largest
// by bisection on the score bits (four independent counters per step; ties at the k-th score -- duplicate rows --
// are resolved by a second bisection on the row word).  Per-lane top-k lists, as used for small k, would need
// k / 4 registers per lane and an insertion chain that long; measured slower by 35 % at k = 100.
template <int NV>
__device__ __forceinline__ uint64_t kth_largest_key(const uint32_t (&hi)[NV], const uint32_t (&lo)[NV], int k) {
  auto count_ge = [&](uint32_t cand) -> int {
    int c[4] = {0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < NV; ++i) c[i & 3] += (hi[i] >= cand) ? 1 : 0;
    return __reduce_add_sync(0xffffffffu, (c[0] + c[1]) + (c[2] + c[3]));
  };
  uint32_t t = 0;
#pragma unroll 1
  for (int bit = 31; bit >= 0; --bit) {
    const uint32_t cand = t | (1u << bit);
    if (count_ge(cand) >= k) t = cand;
  }
  if (t == 0) return 0ull;   // fewer than k rows published so far
  int c_gt = 0, c_eq = 0;
  uint32_t lo_min = 0xFFFFFFFFu;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    c_gt += (hi[i] > t) ? 1 : 0;
    if (hi[i] == t) { ++c_eq; lo_min = lo[i] < lo_min ? lo[i] : lo_min; }
  }
  c_gt = __reduce_add_sync(0xffffffffu, c_gt);
  c_eq = __reduce_add_sync(0xffffffffu, c_eq);
  const int need = k - c_gt;             // rank wanted among the keys that share the k-th score (>= 1, <= c_eq)
  if (need >= c_eq) return (uint64_t(t) << 32) | __reduce_min_sync(0xffffffffu, lo_min);   // the usual case: no tie
  uint32_t l = 0;
#pragma unroll 1
  for (int bit = 31; bit >= 0; --bit) {
    const uint32_t cand = l | (1u << bit);
    int c = 0;
#pragma unroll
    for (int i = 0; i < NV; ++i) c += (hi[i] == t && lo[i] >= cand) ? 1 : 0;
    if (__reduce_add_sync(0xffffffffu, c) >= need) l = cand;
  }
  return (uint64_t(t) << 32) | l;
}

__device__ __forceinline__ uint64_t pooled_kth_key(const uint64_t* __restrict__ pool, int n_ctas, int q, int k, int lane) {
  constexpr int NV = (kPoolMaxCtas / 32) * kPoolM;
  uint32_t hi[NV], lo[NV];
#pragma unroll
  for (int i = 0; i < kPoolMaxCtas / 32; ++i) {
    const int c = lane + 32 * i;
    uint64_t x[kPoolM];
#pragma unroll
    for (int m = 0; m < kPoolM; ++m) x[m] = c < n_ctas ? __ldcg(pool + (size_t(c) * kPoolSlots + m) * kNQ + q) : 0ull;
    // The four slots of a CTA are four separate 8-byte stores: a publish that lands between two of these loads can
    // show ONE row in two slots (when a better row arrives the CTA's keys move down a slot).  The floor must be the
    // k-th largest over DISTINCT rows, so a key already seen in an earlier slot of the same CTA is dropped (keys are
    // unique per row; entries of different CTAs are different rows by construction).
#pragma unroll
    for (int m = 1; m < kPoolM; ++m)
#pragma unroll
      for (int p = 0; p < m; ++p)
        if (x[m] == x[p]) x[m] = 0ull;
#pragma unroll
    for (int m = 0; m < kPoolM; ++m) {
      lo[kPoolM * i + m] = uint32_t(x[m]);
      hi[kPoolM * i + m] = uint32_t(x[m] >> 32);
    }
  }
  return kth_largest_key<NV>(hi, lo, k);
}

// The usual refresh (k <= 0.8 * CTAs): only each CTA's BEST key is pooled -- the k-th largest of ~132 CTA maxima is
// within a factor ~1.6 in admission rate of the true k-th best of everything seen, because k < #CTAs -- and a select
// warp bisects the floors of ALL EIGHT queries it owns at once: the eight bisections are independent, so their
// warp reductions pipeline instead of costing one full REDUX latency per step and query (measured before: 3.3 us per
// query done one after the other, 26 us per warp and refresh; the lane-per-query variant of GPU call 6 was fine at
// k = 10 but needed k / 4 registers per lane and spilled at k = 100).
// Returns a bit mask of the queries (bit j = query ew + 4 j) whose k-th pooled SCORE is shared by several keys: the
// signature of a tie-heavy corpus, where the caller also consults the CTAs' own k-th keys (pooled_max_kth).
__device__ __forceinline__ uint32_t pooled_floor_batch8(const uint64_t* __restrict__ pool, int n_ctas, int ew, int nq,
                                                        int k, int lane, uint64_t (&out)[8]) {
  uint32_t ties = 0u;
  constexpr int NC = kPoolMaxCtas / 32;
  uint32_t hi[8][NC], lo[8][NC];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int q = ew + 4 * j;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int c = lane + 32 * i;
      const uint64_t x = (q < nq && c < n_ctas) ? __ldcg(pool + (size_t(c) * kPoolSlots) * kNQ + q) : 0ull;
      lo[j][i] = uint32_t(x);
      hi[j][i] = uint32_t(x >> 32);
    }
  }
  uint32_t t[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) t[j] = 0u;
#pragma unroll 1
  for (int bit = 31; bit >= 0; --bit) {
    int cnt[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t cand = t[j] | (1u << bit);
      int c = 0;
#pragma unroll
      for (int i = 0; i < NC; ++i) c += (hi[j][i] >= cand) ? 1 : 0;
      cnt[j] = c;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (__reduce_add_sync(0xffffffffu, cnt[j]) >= k) t[j] |= (1u << bit);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    out[j] = 0ull;
    if (t[j] == 0u) continue;          // fewer than k CTAs have published for this query (warp-uniform)
    int c_gt = 0, c_eq = 0;
    uint32_t lo_min = 0xFFFFFFFFu;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      c_gt += (hi[j][i] > t[j]) ? 1 : 0;
      if (hi[j][i] == t[j]) { ++c_eq; lo_min = lo[j][i] < lo_min ? lo[j][i] : lo_min; }
    }
    c_gt = __reduce_add_sync(0xffffffffu, c_gt);
    c_eq = __reduce_add_sync(0xffffffffu, c_eq);
    if (c_eq > 1) ties |= 1u << j;      // warp-uniform (c_eq is a reduction result)
    const int need = k - c_gt;
    if (need >= c_eq) {
      out[j] = (uint64_t(t[j]) << 32) | __reduce_min_sync(0xffffffffu, lo_min);
    } else {                            // ties at the k-th score (duplicate rows): bisect the row word among them
      uint32_t l = 0;
#pragma unroll 1
      for (int bit = 31; bit >= 0; --bit) {
        const uint32_t cand = l | (1u << bit);
        int c = 0;
#pragma unroll
        for (int i = 0; i < NC; ++i) c += (hi[j][i] == t[j] && lo[j][i] >= cand) ? 1 : 0;
        if (__reduce_add_sync(0xffffffffu, c) >= need) l = cand;
      }
      out[j] = (uint64_t(t[j]) << 32) | l;
    }
  }
  return ties;
}

__device__ __forceinline__ uint64_t warp_max_u64(uint64_t v) {
  const uint32_t hi = __reduce_max_sync(0xffffffffu, uint32_t(v >> 32));
  const uint32_t lo = __reduce_max_sync(0xffffffffu, (uint32_t(v >> 32) == hi) ? uint32_t(v) : 0u);
  return (uint64_t(hi) << 32) | lo;
}
// max over the CTAs of their own k-th key for query q (the lanes split the CTAs)
__device__ __forceinline__ uint64_t pooled_max_kth(const uint64_t* __restrict__ pool, int n_ctas, int q, int lane) {
  uint64_t best = 0ull;
#pragma unroll
  for (int i = 0; i < kPoolMaxCtas / 32; ++i) {
    const int c = lane + 32 * i;
    const uint64_t x = c < n_ctas ? __ldcg(pool + (size_t(c) * kPoolSlots + kPoolM) * kNQ + q) : 0ull;
    best = x > best ? x : best;
  }
  return warp_max_u64(best);
}

}  // namespace crag
