// Warp-level exact top-k selection on packed 64-bit keys.
//
// A candidate (score fp32, id u32) is packed so that an unsigned 64-bit
// comparison orders by score descending, then id ascending:
//   key = orderable(score) << 32 | (0xFFFFFFFF - id)
// which is the deterministic stand-in for the reference's
// np.argsort(scores)[::-1] ranking (ComoRAG.py:965; embed_utils.py:158) --
// equal scores are ordered by ascending row id.  key == 0 is the "empty"
// sentinel (orderable() never maps a finite score or +-inf to 0 together with
// id 0xFFFFFFFF).
//
// Per query the selector owns KLIST + CAP keys of shared memory: [0, KLIST) is
// the current sorted top-k (zero padded), [KLIST, KLIST + CAP) an unsorted
// candidate buffer.  flush_query() bitonic-sorts the whole thing in registers
// (32 lanes x EPL keys) and keeps the best k.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

namespace crag {

__device__ __forceinline__ uint32_t orderable_f32(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unorderable_f32(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u ^ 0x80000000u) : ~u);
}
__device__ __forceinline__ uint64_t make_key(float score, uint32_t id) {
  return (static_cast<uint64_t>(orderable_f32(score)) << 32) | static_cast<uint64_t>(0xFFFFFFFFu - id);
}
__device__ __forceinline__ float key_score(uint64_t key) { return unorderable_f32(static_cast<uint32_t>(key >> 32)); }
__device__ __forceinline__ uint32_t key_id(uint64_t key) { return 0xFFFFFFFFu - static_cast<uint32_t>(key); }

__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int lane_mask) {
  uint32_t lo = static_cast<uint32_t>(v), hi = static_cast<uint32_t>(v >> 32);
  lo = __shfl_xor_sync(0xffffffffu, lo, lane_mask);
  hi = __shfl_xor_sync(0xffffffffu, hi, lane_mask);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

// (min, max) of a warp's (a, b) pairs, left in every lane (xor butterfly, strides 16 .. 1)
__device__ __forceinline__ void warp_minmax(float& a, float& b) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a = fminf(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
}

// Bitonic sort, descending, of 32*EPL keys held EPL per lane in blocked order
// (global index g = lane*EPL + j).  EPL must be a power of two.
template <int EPL>
__device__ __forceinline__ void warp_sort_desc(uint64_t (&v)[EPL], int lane) {
#pragma unroll
  for (int size = 2; size <= 32 * EPL; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      if (stride >= EPL) {
        const int lstride = stride / EPL;
        const bool lower = (lane & lstride) == 0;
#pragma unroll
        for (int j = 0; j < EPL; ++j) {
          const uint64_t other = shfl_xor_u64(v[j], lstride);
          const int g = lane * EPL + j;
          const bool desc_block = (g & size) == 0;
          const uint64_t mx = v[j] > other ? v[j] : other;
          const uint64_t mn = v[j] > other ? other : v[j];
          v[j] = (lower == desc_block) ? mx : mn;
        }
      } else {
#pragma unroll
        for (int j = 0; j < EPL; ++j) {
          if ((j & stride) == 0) {
            const int g = lane * EPL + j;
            const bool desc_block = (g & size) == 0;
            const uint64_t a = v[j], b = v[j + stride];
            const uint64_t mx = a > b ? a : b;
            const uint64_t mn = a > b ? b : a;
            v[j] = desc_block ? mx : mn;
            v[j + stride] = desc_block ? mn : mx;
          }
        }
      }
    }
  }
}

// Merge the first `c` buffered candidates of one query into its sorted list and
// publish the new admission threshold.  Called by one full warp.
//   qkeys : KLIST + CAP keys in shared memory
//   thr_key : receives the k-th best key (0 while fewer than k are held)
template <int KLIST, int CAP>
__device__ __forceinline__ void flush_query(uint64_t* qkeys, int c, int k, uint64_t* thr_key, int lane) {
  constexpr int EPL = (KLIST + CAP) / 32;
  static_assert((KLIST + CAP) % 32 == 0 && (EPL & (EPL - 1)) == 0, "KLIST + CAP must be 32 * 2^n");
  uint64_t v[EPL];
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const int g = lane * EPL + j;
    uint64_t x = qkeys[g];
    if (g >= KLIST + c) x = 0;
    v[j] = x;
  }
  warp_sort_desc<EPL>(v, lane);
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const int g = lane * EPL + j;
    if (g < KLIST) qkeys[g] = (g < k) ? v[j] : 0ull;
    if (g == k - 1) *thr_key = v[j];
  }
  __syncwarp();
}

// Cheap flush for a handful of buffered candidates (c <= kInsertMax): each one is placed into the sorted list by a
// warp-parallel shift instead of re-sorting KLIST + CAP keys.  With the pooled admission floor a CTA ends its scan
// with 0-3 candidates pending per query, and 32 full bitonic sorts at the tail of a short scan (multi-GPU strong
// scaling: ~66 tiles per CTA) cost more than the candidates are worth.
constexpr int kInsertMax = 8;
template <int KLIST, int CAP>
__device__ __forceinline__ void insert_few(uint64_t* qkeys, int c, int k, uint64_t* thr_key, int lane) {
  constexpr int E = KLIST / 32;
  static_assert(KLIST % 32 == 0, "KLIST must be a multiple of 32");
  for (int i = 0; i < c; ++i) {
    const uint64_t cand = qkeys[KLIST + i];
    uint64_t nv[E];
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int g = lane * E + j;
      const uint64_t cur = qkeys[g];
      const uint64_t prev = g > 0 ? qkeys[g - 1] : ~0ull;
      // descending list: keys above the candidate stay, the first slot not above it takes it, the rest shift down
      nv[j] = cur > cand ? cur : (prev > cand ? cand : prev);
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < E; ++j) {
      const int g = lane * E + j;
      qkeys[g] = g < k ? nv[j] : 0ull;
    }
    __syncwarp();
  }
  if (lane == 0) *thr_key = qkeys[k - 1];
  __syncwarp();
}

// One warp streams `total` candidate keys (fetch(i), 0 = absent) through a KLIST+CAP selector (CAP >= 32).
template <int KLIST, int CAP, class Fetch>
__device__ __forceinline__ void select_stream(uint64_t* keys, uint64_t* thr_slot, int lane, int k, int total,
                                              uint64_t bound, Fetch fetch) {
  static_assert(CAP >= 32, "a batch of 32 candidates must fit the buffer");
  for (int i = lane; i < KLIST + CAP; i += 32) keys[i] = 0ull;
  if (lane == 0) *thr_slot = 0ull;
  __syncwarp();
  int c = 0;
  constexpr int U = 4;  // batches fetched ahead: the lists sit in L2 / HBM, so 4 loads per lane are kept in flight
  for (int base0 = 0; base0 < total; base0 += 32 * U) {
    uint64_t pre[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int idx = base0 + u * 32 + lane;
      pre[u] = idx < total ? fetch(idx) : 0ull;   // past-the-end batches are all zero and admit nothing
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t key = pre[u];
      const uint64_t thr = *thr_slot > bound ? *thr_slot : bound;
      const bool take = key != 0 && key >= thr;
      const uint32_t m = __ballot_sync(0xffffffffu, take);
      if (m != 0u) {
        if (take) keys[KLIST + c + __popc(m & ((1u << lane) - 1u))] = key;
        c += __popc(m);
        __syncwarp();
        if (c + 32 > CAP) {
          flush_query<KLIST, CAP>(keys, c, k, thr_slot, lane);
          c = 0;
        }
      }
    }
  }
  if (c > 0) flush_query<KLIST, CAP>(keys, c, k, thr_slot, lane);
  __syncwarp();
}

}  // namespace crag
