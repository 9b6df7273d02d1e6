// Merge kernels of the search path: the per-shard merge of the CTAs' partial lists (merge_topk_kernel) and the fused
// finalize + cross-rank exchange + global merge of the row-sharded index (finalize_exchange_kernel).  SIMT code over
// shared memory and, for the exchange, peer-mapped global memory with release / acquire flags -- no wgmma, TMA or
// mbarrier -- kept in a header so tests/warp_emu can run exactly these kernels on emulated thread blocks (one OS
// thread per rank for the exchange) and compare every rank's answer with the merge rule stated in plain C++.
#pragma once
#include <math.h>
#include <stdint.h>
#include <cuda_runtime.h>

#include "pool_floor.cuh"   // kNQ
#include "topk.cuh"

namespace crag {

// ---------------------------------------------------------------------------
// Two-level merge of `parts` sorted lists of k keys, fetch(p, j) = key j of list p (0 = absent), by one CTA of 4 warps:
// warp w streams lists w, w + 4, ... through its selector into s_keys[w], then warp 0 merges the four into s_keys[4].
// Keys below `bound` are skipped up front.  Returns true in warp 0, the warp that holds the result.
template <int KLIST, int CAP, class Fetch>
__device__ __forceinline__ bool merge_lists(uint64_t (&s_keys)[5][KLIST + CAP], uint64_t (&s_thr)[5], int parts, int k,
                                            uint64_t bound, Fetch fetch) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int my_parts = parts > w ? (parts - w + 3) / 4 : 0;
  select_stream<KLIST, CAP>(s_keys[w], &s_thr[w], lane, k, my_parts * k, bound, [&](int idx) -> uint64_t {
    const int pl = idx / k, j = idx - pl * k;
    return fetch(w + 4 * pl, j);
  });
  __syncthreads();
  if (w != 0) return false;
  select_stream<KLIST, CAP>(s_keys[4], &s_thr[4], lane, k, 4 * k, 0ull, [&](int idx) -> uint64_t { return s_keys[idx / k][idx % k]; });
  return true;
}

// Query q's top-k over the per-CTA lists of a scan, part_keys[(p * q_stride + q) * k + j] for p < parts, into s_keys[4].
// Returns true in warp 0, the warp that holds the result.
template <int KLIST, int CAP>
__device__ __forceinline__ bool merge_cta_lists(uint64_t (&s_keys)[5][KLIST + CAP], uint64_t (&s_thr)[5], const uint64_t* __restrict__ part_keys,
                                                int q_stride, int q, int parts, int k) {
  // Admission bound before any sorting: every part's list is sorted, so its k-th entry is a lower bound of the
  // global k-th best (that part alone already holds k candidates at least that good); the max over parts rejects
  // almost all of the parts*k candidates up front.
  const int lane = threadIdx.x & 31;
  uint64_t bound = 0;
  for (int p = lane; p < parts; p += 32) {
    const uint64_t kth = part_keys[(size_t(p) * q_stride + q) * k + (k - 1)];
    bound = kth > bound ? kth : bound;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint64_t other = shfl_xor_u64(bound, o);
    bound = other > bound ? other : bound;
  }
  return merge_lists<KLIST, CAP>(s_keys, s_thr, parts, k, bound, [&](int p, int j) { return part_keys[(size_t(p) * q_stride + q) * k + j]; });
}

// ---------------------------------------------------------------------------
// Merge kernels: one CTA per query streams candidate keys through the same
// selector.  PAIRS=false: raw keys (local row ids) from search_topk_kernel's
// CTAs, ids are widened and offset on output.  PAIRS=true: (score, int64 id)
// pairs from several shards; ties resolve by candidate position.
template <int KLIST, int CAP, bool PAIRS>
__global__ void __launch_bounds__(128) merge_topk_kernel(const uint64_t* __restrict__ part_keys,
                                                         const float* __restrict__ in_scores,
                                                         const int64_t* __restrict__ in_ids,
                                                         const float* __restrict__ part_minmax, int parts,
                                                         int q_stride, int nq, int k, int64_t row_offset,
                                                         int64_t ids_stride, int64_t scores_stride, int64_t mm_stride,
                                                         int64_t* __restrict__ out_ids,
                                                         float* __restrict__ out_scores,
                                                         float* __restrict__ out_minmax,
                                                         uint64_t* __restrict__ last_keys) {
  constexpr int KPQ = KLIST + CAP;
  __shared__ uint64_t s_keys[5][KPQ];
  __shared__ uint64_t s_thr[5];
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x;

  bool merged;
  if constexpr (PAIRS) {
    merged = merge_lists<KLIST, CAP>(s_keys, s_thr, parts, k, 0ull, [&](int p, int j) -> uint64_t {
      const size_t at = size_t(q) * k + j;
      const int64_t id = *reinterpret_cast<const int64_t*>(reinterpret_cast<const char*>(in_ids + at) + p * ids_stride);
      const float sc = *reinterpret_cast<const float*>(reinterpret_cast<const char*>(in_scores + at) + p * scores_stride);
      return id >= 0 ? make_key(sc, uint32_t(p * k + j)) : 0ull;
    });
  } else {
    merged = merge_cta_lists<KLIST, CAP>(s_keys, s_thr, part_keys, q_stride, q, parts, k);
  }
  if (!merged) return;
  uint64_t* keys = s_keys[4];
  for (int j = lane; j < k; j += 32) {
    const uint64_t key = keys[j];
    float s = -INFINITY;
    int64_t id = -1;
    if (key) {
      s = key_score(key);
      if (PAIRS) {
        const uint32_t ci = key_id(key);
        id = *reinterpret_cast<const int64_t*>(reinterpret_cast<const char*>(in_ids + size_t(q) * k + ci % k) +
                                               int64_t(ci / k) * ids_stride);
      } else {
        id = int64_t(key_id(key)) + row_offset;
      }
    }
    out_scores[size_t(q) * k + j] = s;
    out_ids[size_t(q) * k + j] = id;
  }
  if (last_keys != nullptr && lane == 0) last_keys[q] = keys[k - 1];  // 0 when fewer than k rows qualified
  if (out_minmax != nullptr) {
    float a = INFINITY, b = -INFINITY;
    if (part_minmax != nullptr) {
      for (int p = lane; p < parts; p += 32) {
        const float* mm = PAIRS ? reinterpret_cast<const float*>(reinterpret_cast<const char*>(part_minmax + size_t(q) * 2) + p * mm_stride)
                                : part_minmax + (size_t(p) * q_stride + q) * 2;
        a = fminf(a, mm[0]);
        b = fmaxf(b, mm[1]);
      }
    }
    warp_minmax(a, b);
    if (lane == 0) {
      out_minmax[size_t(q) * 2 + 0] = a;
      out_minmax[size_t(q) * 2 + 1] = b;
    }
  }
}

// ---------------------------------------------------------------------------
// Fused per-shard finalize + cross-rank exchange + global merge for the row-sharded index (SURVEY.md section 8e), over
// NVLink peer memory instead of an NCCL all-gather launch.  One CTA per query:
//   1. merge this rank's per-CTA partial lists into the shard's top-k (merge_cta_lists, as merge_topk_kernel);
//   2. PUSH the k (id, score) pairs + (min, max) into slot [parity][this rank][q] of EVERY rank's exchange buffer
//      (peer-mapped symmetric memory: plain stores that travel over NVLink), fence, then release-store the epoch
//      into flag [parity][this rank][q] of every rank;
//   3. wait (acquire loads, bounded) until the flags of all `world` ranks for query q show this epoch;
//   4. merge the world * k candidates now sitting in the LOCAL buffer (ties: source rank, then position == ascending
//      global id for contiguous ascending shards) and write the global answer.
// Every rank runs the same kernel for the same query block (a collective), ends with the same answer, and nothing
// but the 2.8 KB records crosses the links.  Epochs count calls per query slot on the device (graph-replay safe);
// two parities of slots make reuse safe: a rank can only start writing epoch e+2 after every peer pushed e+1, which
// each peer does after it finished reading epoch e.
constexpr int kXMaxWorld = 16;
constexpr int kXSlotBytes = 128 * 8 + 128 * 4 + 16;   // ids[128] | scores[128] | min, max, pad
__host__ __device__ inline size_t xchg_slot_off(int parity, int src, int q, int world) {
  return ((size_t(parity) * world + src) * kNQ + q) * kXSlotBytes;
}
__host__ __device__ inline size_t xchg_flags_off(int world) { return size_t(2) * world * kNQ * kXSlotBytes; }
__host__ __device__ inline size_t xchg_total_bytes(int world) { return xchg_flags_off(world) + size_t(2) * world * kNQ * 8; }

#ifndef CRAG_EMULATED_PTX   // tests/warp_emu supplies host versions (std::atomic release / acquire, steady_clock)
__device__ __forceinline__ void st_release_sys_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#endif

template <int KLIST, int CAP>
__global__ void __launch_bounds__(128) finalize_exchange_kernel(const uint64_t* __restrict__ part_keys,
                                                                const float* __restrict__ part_minmax, int parts,
                                                                int nq, int k, int64_t row_offset,
                                                                const uint64_t* __restrict__ peer_bufs, int rank,
                                                                int world, uint64_t* __restrict__ epochs,
                                                                int* __restrict__ status,
                                                                int64_t* __restrict__ out_ids,
                                                                float* __restrict__ out_scores,
                                                                float* __restrict__ out_minmax) {
  constexpr int KPQ = KLIST + CAP;
  __shared__ uint64_t s_keys[5][KPQ];
  __shared__ uint64_t s_thr[5];
  __shared__ float s_mm[2];
  __shared__ int s_bad;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x;
  const uint64_t epoch = epochs[q] + 1;
  const int parity = int(epoch & 1);
  if (threadIdx.x == 0) s_bad = 0;

  // ---- 1. this shard's top-k for query q (parts may be 0: empty shard)
  if (merge_cta_lists<KLIST, CAP>(s_keys, s_thr, part_keys, kNQ, q, parts, k)) {
    float a = INFINITY, b = -INFINITY;
    for (int p = lane; p < parts; p += 32) {
      a = fminf(a, part_minmax[(size_t(p) * kNQ + q) * 2 + 0]);
      b = fmaxf(b, part_minmax[(size_t(p) * kNQ + q) * 2 + 1]);
    }
    warp_minmax(a, b);
    if (lane == 0) { s_mm[0] = a; s_mm[1] = b; }
  }
  __syncthreads();

  // ---- 2. push the record into every rank's slot for (parity, this rank, q)
  const size_t slot = xchg_slot_off(parity, rank, q, world);
  for (int idx = threadIdx.x; idx < world * k; idx += blockDim.x) {
    const int d = idx / k, j = idx - d * k;
    const uint64_t key = s_keys[4][j];
    uint8_t* base = reinterpret_cast<uint8_t*>(peer_bufs[d]) + slot;
    reinterpret_cast<int64_t*>(base)[j] = key ? int64_t(key_id(key)) + row_offset : int64_t(-1);
    reinterpret_cast<float*>(base + 128 * 8)[j] = key ? key_score(key) : -INFINITY;
  }
  if (int(threadIdx.x) < world) {
    float* mm = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(peer_bufs[threadIdx.x]) + slot + 128 * 8 + 128 * 4);
    mm[0] = s_mm[0];
    mm[1] = s_mm[1];
  }
  __threadfence_system();
  __syncthreads();
  const size_t flag_idx = (size_t(parity) * world) * kNQ;   // + src * kNQ + q
  if (int(threadIdx.x) < world) {
    uint64_t* flags = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(peer_bufs[threadIdx.x]) + xchg_flags_off(world));
    st_release_sys_u64(flags + flag_idx + size_t(rank) * kNQ + q, epoch);
  }

  // ---- 3. wait for every rank's record of this epoch (bounded: a missing peer must not hang the GPU)
  uint8_t* mine = reinterpret_cast<uint8_t*>(peer_bufs[rank]);
  if (int(threadIdx.x) < world) {
    const uint64_t* f = reinterpret_cast<const uint64_t*>(mine + xchg_flags_off(world)) + flag_idx + size_t(threadIdx.x) * kNQ + q;
    const uint64_t t0 = global_timer_ns();
    while (ld_acquire_sys_u64(f) < epoch) {
      __nanosleep(64);
      if (global_timer_ns() - t0 > 4000000000ull) { s_bad = 1; break; }   // 4 s
    }
  }
  __syncthreads();
  if (s_bad) {
    if (threadIdx.x == 0) { *status = 1; epochs[q] = epoch; }
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
      out_ids[size_t(q) * k + j] = -1;
      out_scores[size_t(q) * k + j] = -INFINITY;
    }
    return;
  }

  // ---- 4. merge the world * k candidates of the local buffer
  if (w != 0) return;
  auto cand_id = [&](int src, int j) -> int64_t {
    return __ldcv(reinterpret_cast<const long long*>(mine + xchg_slot_off(parity, src, q, world)) + j);
  };
  auto cand_score = [&](int src, int j) -> float {
    return __ldcv(reinterpret_cast<const float*>(mine + xchg_slot_off(parity, src, q, world) + 128 * 8) + j);
  };
  select_stream<KLIST, CAP>(s_keys[0], &s_thr[0], lane, k, world * k, 0ull, [&](int idx) -> uint64_t {
    const int src = idx / k, j = idx - src * k;
    return cand_id(src, j) >= 0 ? make_key(cand_score(src, j), uint32_t(idx)) : 0ull;
  });
  for (int j = lane; j < k; j += 32) {
    const uint64_t key = s_keys[0][j];
    float sc = -INFINITY;
    int64_t id = -1;
    if (key) {
      const uint32_t ci = key_id(key);
      sc = key_score(key);
      id = cand_id(int(ci) / k, int(ci) % k);
    }
    out_scores[size_t(q) * k + j] = sc;
    out_ids[size_t(q) * k + j] = id;
  }
  if (out_minmax != nullptr) {
    float a = INFINITY, b = -INFINITY;
    if (lane < world) {
      const float* mm = reinterpret_cast<const float*>(mine + xchg_slot_off(parity, lane, q, world) + 128 * 8 + 128 * 4);
      a = __ldcv(mm);
      b = __ldcv(mm + 1);
    }
    warp_minmax(a, b);
    if (lane == 0) {
      out_minmax[size_t(q) * 2 + 0] = a;
      out_minmax[size_t(q) * 2 + 1] = b;
    }
  }
  if (lane == 0) epochs[q] = epoch;
}

}  // namespace crag
