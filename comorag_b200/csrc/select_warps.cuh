// The select warps of search_topk_kernel (search.cu): warps 0-3 of the shard scan, which turn the stream of score tiles
// into this CTA's exact top-k per query and its (min, max).  Pure SIMT code over shared memory with named barriers --
// no wgmma, TMA or mbarrier: the score tiles arrive through a source type the caller supplies (the kernel's waits on
// the wgmma warpgroup's mbarriers; tests/warp_emu's reads a score matrix), so tests/warp_emu runs exactly this code on
// emulated thread blocks.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

#include "pool_floor.cuh"
#include "search_types.cuh"
#include "topk.cuh"

namespace crag {

#ifndef CRAG_EMULATED_PTX   // tests/warp_emu supplies host versions (the fiber emulator's barriers)
// Named barrier among a subset of the CTA's warps (id 1..15; 0 is __syncthreads).
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("barrier.cta.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Barrier + OR-reduction of a predicate over the participating threads.
__device__ __forceinline__ bool named_bar_or(uint32_t id, uint32_t nthreads, bool pred) {
  uint32_t out;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.b32 p, %1, 0;\n\t"
      "barrier.cta.red.or.pred q, %2, %3, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(out)
      : "r"(static_cast<uint32_t>(pred)), "r"(id), "r"(nthreads)
      : "memory");
  return out != 0;
}
#endif

// Flat scans walk GROUPS of 2^shift consecutive tiles in a multiplicative permutation of the row order (mul coprime to
// the number of whole groups; a ragged tail keeps its place; mul = 0: row order): at any moment the CTAs sample the
// whole shard, so a corpus whose scores drift along the row order (rows appended in narrative order, planted
// neighbours in the tail) looks like a random one to the selector.  Neighbouring CTAs still stream neighbouring tiles
// of one group (2 MB at shift 3 = one page of address translation), which is what HBM and the TLBs like.
struct TileOrder {
  int groups, shift;
  uint32_t mul;
  __device__ __forceinline__ TileOrder(int num_tiles, uint32_t perm_mul, int perm_shift)
      : groups(perm_mul ? (num_tiles >> perm_shift) : 0), shift(perm_shift), mul(perm_mul) {}
  // the tile visited j-th
  __device__ __forceinline__ int operator()(int j) const {
    const int g = j >> shift;
    if (g >= groups) return j;
    return (int((uint64_t(uint32_t(g)) * mul) % uint32_t(groups)) << shift) + (j & ((1 << shift) - 1));
  }
};

// The selector's shared memory, and what the four select warps do with it.
template <int KLIST, int CAP>
struct SelectSmem {
  static constexpr int kKeysPerQuery = KLIST + CAP;
  uint64_t* keys;        // [kNQ][KLIST + CAP]: sorted list, then candidate buffer (topk.cuh)
  uint64_t* thr_key;     // [kNQ] admission threshold: max(local k-th key, pooled floor)
  float* thr_f;          // [kNQ] its score
  int* cnt;              // [kNQ] candidates in the buffer
  float* red;            // [4][kNQ][2] per-warp (min, max)
  uint64_t* bnd_key;     // [kNQ] rank continuation: admit only keys < bnd_key
  float* bnd_f;          // [kNQ] its score
  uint64_t* floor_key;   // [kNQ] pooled admission floor (see kPoolM)
  uint64_t* part_floor;  // [4][kNQ] scratch of a floor refresh

  __host__ __device__ static constexpr size_t bytes() {
    return size_t(kNQ) * kKeysPerQuery * 8 + kNQ * (8 + 4 + 4) + 4 * kNQ * 2 * 4 + kNQ * (8 + 4) + kNQ * 8 + 4 * kNQ * 8;
  }
  // `base`: 8-byte aligned, bytes() long
  __device__ __forceinline__ static SelectSmem carve(uint8_t* base) {
    SelectSmem s;
    s.keys = reinterpret_cast<uint64_t*>(base);
    s.thr_key = s.keys + kNQ * kKeysPerQuery;
    s.thr_f = reinterpret_cast<float*>(s.thr_key + kNQ);
    s.cnt = reinterpret_cast<int*>(s.thr_f + kNQ);
    s.red = reinterpret_cast<float*>(s.cnt + kNQ);
    s.bnd_key = reinterpret_cast<uint64_t*>(s.red + 4 * kNQ * 2);
    s.bnd_f = reinterpret_cast<float*>(s.bnd_key + kNQ);
    s.floor_key = reinterpret_cast<uint64_t*>(s.bnd_f + kNQ);
    s.part_floor = s.floor_key + kNQ;
    return s;
  }

  // Empty lists, thresholds at -inf.  All threads of the CTA, before the __syncthreads that starts the scan.
  __device__ __forceinline__ void init(int nq, const uint64_t* after_keys) const {
    for (int i = threadIdx.x; i < kNQ * kKeysPerQuery; i += kSearchThreads) keys[i] = 0ull;
    if (threadIdx.x < kNQ) {
      thr_key[threadIdx.x] = 0ull;
      floor_key[threadIdx.x] = 0ull;
      thr_f[threadIdx.x] = -INFINITY;
      cnt[threadIdx.x] = 0;
      // "search after": rank continuation for k > 128 -- only candidates strictly below the previous pass's last key
      const uint64_t b = (after_keys != nullptr && int(threadIdx.x) < nq) ? after_keys[threadIdx.x] : ~0ull;
      bnd_key[threadIdx.x] = b;
      bnd_f[threadIdx.x] = (b == ~0ull) ? INFINITY : (b == 0ull ? -INFINITY : key_score(b));
    }
  }

  // Row `row` with score s is a candidate of query q.  The float test rejects almost everything; survivors must also
  // beat the current k-th KEY, so rows that only tie its score with a larger row id (duplicate-heavy corpora) do not
  // flood the buffer.
  __device__ __forceinline__ bool admits(int q, float s, uint32_t row) const {
    return s >= thr_f[q] && s <= bnd_f[q] && make_key(s, row) > thr_key[q];
  }

  // publish this CTA's best kPoolM rows of query q (call after a flush, by the warp that owns q)
  __device__ __forceinline__ void publish(int q, uint64_t* pool, int k, int lane) const {
    if (pool != nullptr && lane < kPoolM) {
      const uint64_t kk = keys[q * kKeysPerQuery + lane];
      if (kk) pool[(size_t(blockIdx.x) * kPoolSlots + lane) * kNQ + q] = kk;
    }
    if (pool != nullptr && lane == kPoolM) {
      // this CTA's own k-th key: it alone holds k rows at or above it, so the MAXIMUM of these over the CTAs is a
      // floor too -- the tight one when scores tie massively (duplicate rows), where a CTA's best keys all sit in
      // one tile and the pooled best keys trail far behind the true k-th key
      const uint64_t kth = keys[q * kKeysPerQuery + k - 1];
      if (kth) pool[(size_t(blockIdx.x) * kPoolSlots + kPoolM) * kNQ + q] = kth;
    }
  }

  // raise the thresholds to the pooled floor (all four select warps; see the comment at kPoolM)
  __device__ __forceinline__ void raise_to(int q, uint64_t pf, int nq) const {
    if (q < nq && pf > floor_key[q]) {
      floor_key[q] = pf;
      if (pf > thr_key[q]) {
        thr_key[q] = pf;
        thr_f[q] = key_score(pf);
      }
    }
  }

  // new floors from the pool: select warp ew refreshes the queries it owns
  __device__ __forceinline__ void refresh(const uint64_t* pool, int k, int nq, int ew, int lane) const {
    if (pool == nullptr) return;
    if (k <= kPoolSmallK) {
      // lane = query: every warp scans a quarter of the CTAs' best keys, the floor is the minimum of the four
      part_floor[ew * kNQ + lane] = lane_kth_of_pool<4>(pool, int(gridDim.x), ew, lane, 1, (k + 3) / 4);
      named_bar_sync(1, kEpiThreads);
      if (lane < kNQ / 4) {                      // this warp owns queries ew, ew + 4, ...
        const int q = ew + 4 * lane;
        uint64_t pf = part_floor[q];
#pragma unroll
        for (int w2 = 1; w2 < 4; ++w2) pf = part_floor[w2 * kNQ + q] < pf ? part_floor[w2 * kNQ + q] : pf;
        raise_to(q, pf, nq);
      }
      for (int q = ew; q < nq; q += 4) {           // and the largest own-k-th key of any CTA
        const uint64_t mk = pooled_max_kth(pool, int(gridDim.x), q, lane);
        if (lane == 0) raise_to(q, mk, nq);
      }
    } else if (5 * k <= 4 * int(gridDim.x)) {
      // k below the CTA count: the CTAs' best keys suffice; this warp's eight queries are bisected together
      uint64_t pf[8];
      const uint32_t ties = pooled_floor_batch8(pool, int(gridDim.x), ew, nq, k, lane, pf);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int q = ew + 4 * j;
        // the CTAs' own k-th keys are consulted only where scores tie (it costs 5 loads + 2 reductions per query)
        const uint64_t mk = (q < nq && ((ties >> j) & 1u)) ? pooled_max_kth(pool, int(gridDim.x), q, lane) : 0ull;
        if (lane == 0) raise_to(q, mk > pf[j] ? mk : pf[j], nq);
      }
    } else {
      for (int q = ew; q < nq; q += 4) {
        const uint64_t pf = pooled_kth_key(pool, int(gridDim.x), q, k, lane);
        const uint64_t mk = pooled_max_kth(pool, int(gridDim.x), q, lane);
        if (lane == 0) raise_to(q, mk > pf ? mk : pf, nq);
      }
    }
  }

  // after a flush of query q (lane 0 of the owning warp): threshold = max(local k-th key, pooled floor)
  __device__ __forceinline__ void settle(int q) const {
    uint64_t t = thr_key[q];
    if (floor_key[q] > t) { t = floor_key[q]; thr_key[q] = t; }
    thr_f[q] = t ? key_score(t) : -INFINITY;
  }
};

// The body of select warp `warp` (0-3): every score tile of this CTA, then the drain of the candidate buffers and this
// CTA's lists and (min, max) in part_keys / part_minmax.  Each thread owns one row of a tile: it takes that row's kNQ
// scores from tiles.next(tile, quad, lane, r), updates the per-query (min, max) and offers the scores that beat the
// query's threshold to the candidate buffers.  IVF walks a work-list of probed tiles; SCORES stores every score
// (or keeps each row's running argmax) instead of selecting.
template <int KLIST, int CAP, bool IVF, bool SCORES, class Tiles>
__device__ __forceinline__ void select_warps(const SelectSmem<KLIST, CAP> s, Tiles& tiles, const TileOrder order, int num_tiles, int n_rows,
                                             int nq, int k, const uint64_t* after_keys, uint64_t* pool, uint64_t* part_keys,
                                             float* part_minmax, const typename IvfParam<IVF, SCORES>::type& args, int warp, int lane) {
  constexpr int KPQ = KLIST + CAP;
  const int quad = warp;      // rows quad * 32 .. quad * 32 + 31 of every score tile
  const int ew = warp;        // select-warp index 0..3 (query ownership for flushes)
  float mn[kNQ], mx[kNQ];
#pragma unroll
  for (int q = 0; q < kNQ; ++q) { mn[q] = INFINITY; mx[q] = -INFINITY; }

  // direct first tile needs room for 128 keys per query and no continuation bound
  const bool direct_first = !IVF && (KLIST + CAP >= 128) && after_keys == nullptr;
  int it = 0;
  for (int j = blockIdx.x; j < num_tiles; j += gridDim.x, ++it) {
    const int tile = IVF ? j : order(j);
    // after tiles 2, 12, 48 and every 128th: all four warps take the same branch (it is CTA-uniform); the smem
    // thresholds they update are read again only after the next named barrier.  (After two tiles per CTA the pool
    // already holds the best of ~38k rows; what is admitted later is k * ln(rows / 38k) keys per query over ALL
    // CTAs, so further refreshes are for long scans and drifting corpora only.)
    const bool due = k <= kPoolSmallK ? (it == 2 || it == 12 || it == 48 || (it >= 128 && (it & 127) == 0))
                                      : (it == 2 || it == 4 || it == 8 || it == 16 || it == 32 || (it >= 64 && (it & 63) == 0));
    if (due) {
      s.refresh(pool, k, nq, ew, lane);
      named_bar_sync(1, kEpiThreads);
    }
    uint32_t r[kNQ];
    tiles.next(tile, quad, lane, r);

    if constexpr (SCORES) {
      const int srow = tile * kTileRows + quad * 32 + lane;
      if (srow < n_rows) {
        if (args.best_id != nullptr) {
          const bool first = args.base_id == 0;       // the first centroid block starts every row's running best
          float bs = first ? -INFINITY : args.best_score[srow];
          int32_t bi = first ? 0 : args.best_id[srow];
#pragma unroll
          for (int q = 0; q < kNQ; ++q) {
            const float sc = __uint_as_float(r[q]);
            if (q < nq && sc > bs) { bs = sc; bi = args.base_id + q; }   // strict: ties stay with the smaller id
          }
          args.best_score[srow] = bs;
          args.best_id[srow] = bi;
        } else {
#pragma unroll
          for (int q = 0; q < kNQ; ++q) {
            const float sc = __uint_as_float(r[q]);
            mn[q] = fminf(mn[q], sc);
            mx[q] = fmaxf(mx[q], sc);
            if (q < nq) args.out[int64_t(q) * args.ld + srow] = sc;
          }
        }
      }
      continue;
    }
    int row;
    uint32_t pending = 0;
    if constexpr (!IVF) {
      row = tile * kTileRows + quad * 32 + lane;
      if (row < n_rows) {
#pragma unroll
        for (int q = 0; q < kNQ; ++q) {
          const float sc = __uint_as_float(r[q]);
          mn[q] = fminf(mn[q], sc);
          mx[q] = fmaxf(mx[q], sc);
          if (s.admits(q, sc, uint32_t(row))) pending |= 1u << q;
        }
        if (nq < kNQ) pending &= (1u << nq) - 1u;
      }
    } else {
      // this tile belongs to ONE coarse list: only the queries probing it see its rows, and a row's score is
      // q . c_list (coarse pass, fp32) + q . residual (this tile's wgmma)
      const int4 item = __ldg(&args.work[tile]);
      row = item.x + quad * 32 + lane;
      if (quad * 32 + lane < item.y) {
        const uint32_t probing = __ldg(&args.list_mask[item.z]);
        const float* co = args.coarse + size_t(item.z) * kNQ;
#pragma unroll
        for (int q = 0; q < kNQ; ++q) {
          if ((probing >> q) & 1u) {
            const float sc = __uint_as_float(r[q]) + __ldg(co + q);
            r[q] = __float_as_uint(sc);
            mn[q] = fminf(mn[q], sc);
            mx[q] = fmaxf(mx[q], sc);
            if (s.admits(q, sc, uint32_t(row))) pending |= 1u << q;
          }
        }
        if (nq < kNQ) pending &= (1u << nq) - 1u;
      }
    }
    // First tile of an unseeded pass: the lists are empty and every row is a candidate.  Skip the reservation
    // protocol (128-way contended atomics, several flush rounds): each row's key goes straight to slot
    // row_in_tile of the query's buffer and one 128-key sort per query builds the list.
    if (direct_first && it == 0) {
#pragma unroll
      for (int q = 0; q < kNQ; ++q)
        s.keys[q * KPQ + quad * 32 + lane] = ((pending >> q) & 1u) ? make_key(__uint_as_float(r[q]), uint32_t(row)) : 0ull;
      named_bar_sync(1, kEpiThreads);
      for (int q = ew; q < kNQ; q += 4) {
        // exactly 128 keys are live (slots 0..127): sort those, not the whole KLIST + CAP area
        flush_query<KLIST, 128 - KLIST>(s.keys + q * KPQ, 128 - KLIST, k, &s.thr_key[q], lane);
        if (lane == 0) s.settle(q);
        s.publish(q, pool, k, lane);
      }
      named_bar_sync(1, kEpiThreads);
      continue;
    }
    // Candidates are handed to the per-query buffers warp by warp: only the queries that HAVE a candidate in this
    // warp are visited (a set-bit walk over the OR of the lanes' pending masks), one shared-memory atomic reserves
    // the slots of all of a query's candidates in the warp, and the lanes take consecutive slots by ballot rank.
    // (Round 1 walked all 32 queries in every thread with one atomic per candidate; the k = 100 profile showed
    // that per-tile loop, not the sorts or the floor, as the largest share of the select warps' time.)
    const uint32_t lanes_below = (1u << lane) - 1u;
    while (true) {
      bool want_flush = false;
      uint32_t any = __reduce_or_sync(0xffffffffu, pending);
      while (any) {
        const int q = __ffs(any) - 1;
        any &= any - 1u;
        bool mine = (pending >> q) & 1u;
        uint64_t key = 0ull;
        if (mine) {
          key = make_key(__uint_as_float(pick32(r, q)), uint32_t(row));
          if (key >= s.bnd_key[q]) {             // rank continuation: at or above the previous pass's last key
            mine = false;
            pending &= ~(1u << q);
          }
        }
        const uint32_t m = __ballot_sync(0xffffffffu, mine);
        if (m == 0u) continue;
        const int leader = __ffs(m) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(&s.cnt[q], __popc(m));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (mine) {
          const int slot = base + __popc(m & lanes_below);
          if (slot < CAP) {
            s.keys[q * KPQ + KLIST + slot] = key;
            pending &= ~(1u << q);
          }
        }
        if (base + __popc(m) >= CAP) want_flush = true;
      }
      if (!named_bar_or(1, kEpiThreads, want_flush || pending != 0)) break;
      for (int q = ew; q < kNQ; q += 4) {
        const int c = s.cnt[q];
        if (c >= CAP) {
          flush_query<KLIST, CAP>(s.keys + q * KPQ, CAP, k, &s.thr_key[q], lane);
          if (lane == 0) {
            s.settle(q);
            s.cnt[q] = 0;
          }
          s.publish(q, pool, k, lane);
        }
      }
      named_bar_sync(1, kEpiThreads);
      for (uint32_t p2 = pending; p2; p2 &= p2 - 1u) {     // what is left and no longer beats the new k-th key: drop
        const int q = __ffs(p2) - 1;
        if (make_key(__uint_as_float(pick32(r, q)), uint32_t(row)) < s.thr_key[q]) pending &= ~(1u << q);
      }
    }
  }

  // drain candidate buffers, then publish this CTA's lists and (min, max)
  named_bar_sync(1, kEpiThreads);
  if constexpr (!SCORES) {
    for (int q = ew; q < kNQ; q += 4) {
      const int c = min(s.cnt[q], CAP);
      if (c > kInsertMax) flush_query<KLIST, CAP>(s.keys + q * KPQ, c, k, &s.thr_key[q], lane);
      else if (c > 0) insert_few<KLIST, CAP>(s.keys + q * KPQ, c, k, &s.thr_key[q], lane);
      __syncwarp();
      uint64_t* dst = part_keys + (size_t(blockIdx.x) * kNQ + q) * k;
      for (int j = lane; j < k; j += 32) dst[j] = s.keys[q * KPQ + j];
    }
  }
#pragma unroll
  for (int q = 0; q < kNQ; ++q) {
    float a = mn[q], b = mx[q];
    warp_minmax(a, b);
    if (lane == q) {
      s.red[(ew * kNQ + q) * 2 + 0] = a;
      s.red[(ew * kNQ + q) * 2 + 1] = b;
    }
  }
  named_bar_sync(1, kEpiThreads);
  if (ew == 0) {
    float a = s.red[lane * 2], b = s.red[lane * 2 + 1];
#pragma unroll
    for (int w = 1; w < 4; ++w) {
      a = fminf(a, s.red[(w * kNQ + lane) * 2]);
      b = fmaxf(b, s.red[(w * kNQ + lane) * 2 + 1]);
    }
    part_minmax[(size_t(blockIdx.x) * kNQ + lane) * 2 + 0] = a;
    part_minmax[(size_t(blockIdx.x) * kNQ + lane) * 2 + 1] = b;
  }
}

}  // namespace crag
