// The block-wide sort of up to 2048 packed keys (topk.cuh's make_key order) that ends crag_knn_topk's select
// (knn_select.cuh) and the wide rescore of crag_rescore_topk (quant_kernels.cuh), with the block shape both run at.
// Pure SIMT, so tests/warp_emu runs it on emulated blocks.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace crag {
namespace {

constexpr int kKnnMaxK = 2048;
constexpr int kKnnThreads = 512;
constexpr int kKnnWarps = kKnnThreads / 32;

// Bitonic sort (descending) of s_keys[0, count), zero-padded to a power of two, by a block of kKnnThreads threads;
// ends with the block synced
__device__ __forceinline__ void knn_bitonic_sort(uint64_t* s_keys, int count, int tid) {
  int n2 = 1;
  while (n2 < count) n2 <<= 1;
  __syncthreads();
  for (int i = count + tid; i < n2; i += kKnnThreads) s_keys[i] = 0ull;
  __syncthreads();
  for (int size = 2; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int p = tid; p < (n2 >> 1); p += kKnnThreads) {
        const int a = 2 * p - (p & (stride - 1));   // p with a zero bit inserted at `stride`
        const int b = a + stride;
        const uint64_t ka = s_keys[a], kb = s_keys[b];
        const bool desc = (a & size) == 0;
        if ((ka < kb) == desc) {
          s_keys[a] = kb;
          s_keys[b] = ka;
        }
      }
      __syncthreads();
    }
  }
}

}  // namespace
}  // namespace crag
