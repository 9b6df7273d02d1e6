// The kernels of the full device ranking (rank_all.cu): a stable LSD radix sort, pure SIMT integer code (shared-memory
// histograms, a block scan, match.any ranking inside a warp) with nothing architecture-specific in it.  Kept in a header
// so tests/warp_emu can run exactly these kernels on emulated thread blocks and compare the permutation with
// std::stable_sort (descending score, ascending row on ties) -- the bit-exact contract of ComoRAG.py:965-966.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

#include "topk.cuh"
#include "workspace.cuh"

namespace crag {
namespace {

constexpr int kSortThreads = 256;                       // 8 warps per CTA
constexpr int kWarpsPerCta = kSortThreads / 32;

struct SortPlan {
  int run;         // elements per warp (multiple of 32)
  int n_warps;     // total warps
  int grid;
  uint32_t *keys[2], *vals[2];   // the workspace's double buffers (null when only sized)
  uint32_t* hist;                // [256][n_warps] digit counts, then the 256 digit totals
  size_t total;                  // workspace bytes
};

SortPlan plan_sort(int64_t n, void* ws = nullptr) {
  SortPlan p;
  // runs of 2048 elements; for big arrays grow the run so the histogram table stays small (<= 8192 warps)
  int64_t run = 2048;
  while ((n + run - 1) / run > 8192) run *= 2;
  p.run = int(run);
  p.n_warps = int((n + run - 1) / run);
  if (p.n_warps < 1) p.n_warps = 1;
  p.grid = (p.n_warps + kWarpsPerCta - 1) / kWarpsPerCta;
  WsCursor c(ws);
  p.keys[0] = c.take<uint32_t>(size_t(n));
  p.keys[1] = c.take<uint32_t>(size_t(n));
  p.vals[0] = c.take<uint32_t>(size_t(n));
  p.vals[1] = c.take<uint32_t>(size_t(n));
  p.hist = c.take<uint32_t>(size_t(256) * p.n_warps + 256);
  p.total = c.bytes;
  return p;
}

__device__ __forceinline__ uint32_t sort_key(float s) { return ~orderable_f32(s); }

template <bool FIRST>
__global__ void __launch_bounds__(kSortThreads) hist_kernel(const float* __restrict__ scores,
                                                            const uint32_t* __restrict__ keys_in, int64_t n, int run,
                                                            int n_warps, int shift, uint32_t* __restrict__ hist,
                                                            uint32_t* __restrict__ totals) {
  __shared__ uint32_t s_cnt[kWarpsPerCta][256];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * kWarpsPerCta + w;
  for (int i = lane; i < 256; i += 32) s_cnt[w][i] = 0;
  __syncwarp();
  if (gw < n_warps) {
    const int64_t lo = int64_t(gw) * run;
    const int64_t hi = lo + run < n ? lo + run : n;
    for (int64_t i = lo + lane; i < hi; i += 32) {
      const uint32_t key = FIRST ? sort_key(scores[i]) : keys_in[i];
      atomicAdd(&s_cnt[w][(key >> shift) & 255u], 1u);
    }
    __syncwarp();
    for (int d = lane; d < 256; d += 32) {
      const uint32_t c = s_cnt[w][d];
      hist[size_t(d) * n_warps + gw] = c;
      if (c) atomicAdd(&totals[d], c);
    }
  }
}

// block d: exclusive offsets of digit d's per-warp counts, starting at the number of elements with a smaller digit
__global__ void __launch_bounds__(256) scan_kernel(uint32_t* __restrict__ hist, const uint32_t* __restrict__ totals,
                                                   int n_warps) {
  __shared__ uint32_t s_part[256];
  __shared__ uint32_t s_base;
  const int d = blockIdx.x, t = threadIdx.x;
  s_part[t] = t < d ? totals[t] : 0u;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (t < o) s_part[t] += s_part[t + o];
    __syncthreads();
  }
  if (t == 0) s_base = s_part[0];
  __syncthreads();
  uint32_t carry = s_base;
  uint32_t* row = hist + size_t(d) * n_warps;
  for (int base = 0; base < n_warps; base += 256) {
    const int i = base + t;
    const uint32_t v = i < n_warps ? row[i] : 0u;
    // inclusive block scan (Hillis-Steele over 256 entries)
    __syncthreads();
    s_part[t] = v;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
      const uint32_t add = t >= o ? s_part[t - o] : 0u;
      __syncthreads();
      s_part[t] += add;
      __syncthreads();
    }
    if (i < n_warps) row[i] = carry + s_part[t] - v;
    carry += s_part[255];
  }
}

template <bool FIRST, bool LAST>
__global__ void __launch_bounds__(kSortThreads) scatter_kernel(const float* __restrict__ scores,
                                                               const uint32_t* __restrict__ keys_in,
                                                               const uint32_t* __restrict__ vals_in, int64_t n, int run,
                                                               int n_warps, int shift, const uint32_t* __restrict__ hist,
                                                               uint32_t* __restrict__ keys_out,
                                                               uint32_t* __restrict__ vals_out,
                                                               int64_t* __restrict__ out_ids,
                                                               float* __restrict__ out_scores) {
  __shared__ uint32_t s_off[kWarpsPerCta][256];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * kWarpsPerCta + w;
  if (gw >= n_warps) return;
  for (int d = lane; d < 256; d += 32) s_off[w][d] = hist[size_t(d) * n_warps + gw];
  __syncwarp();
  const int64_t lo = int64_t(gw) * run;
  const int64_t hi = lo + run < n ? lo + run : n;
  const uint32_t lt = (1u << lane) - 1u;
  for (int64_t base = lo; base < hi; base += 32) {
    const int64_t i = base + lane;
    const bool live = i < hi;
    uint32_t key = 0, val = 0;
    if (live) {
      key = FIRST ? sort_key(scores[i]) : keys_in[i];
      val = FIRST ? uint32_t(i) : vals_in[i];
    }
    // dead lanes get digits no live lane can have, so they never share a match group
    const uint32_t digit = live ? ((key >> shift) & 255u) : (256u + lane);
    const uint32_t peers = __match_any_sync(0xffffffffu, digit);
    const uint32_t rank = __popc(peers & lt);
    uint32_t pos = 0;
    if (live) pos = s_off[w][digit] + rank;
    __syncwarp();
    if (live && rank == 0) s_off[w][digit] += __popc(peers);
    __syncwarp();
    if (live) {
      if (LAST) {
        out_ids[pos] = int64_t(val);
        out_scores[pos] = unorderable_f32(~key);
      } else {
        keys_out[pos] = key;
        vals_out[pos] = val;
      }
    }
  }
}

}  // namespace
}  // namespace crag
