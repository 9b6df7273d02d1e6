// One-bit corpus shards (crag_search_topk_b1, DESIGN.md 3f): the map from a row's sign bits to the register A fragment
// of the s8 wgmma.  Pure integer code, so tests/warp_emu checks it on the CPU against a model of the PTX layout.
//
// A code row holds dim8 / 8 bytes; bit j of byte b stands for column 8 b + j, so the 32-bit word w (little endian) holds
// columns 32 w .. 32 w + 31 with column 32 w + j in bit j: one word is one 32-wide k-step of m64nNk32.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace crag {

constexpr int kB1QueryBytes = 32 * 1024;   // the resident int8 query block: 32 queries x 1024 columns at most

// 4 code bits -> the 4 int8 of one register, bit i -> byte i: +1 (0x01) for a set bit, -1 (0xFF) for a clear one
__host__ __device__ __forceinline__ uint32_t b1_widen4(uint32_t nibble) {
  const uint32_t spread = (nibble * 0x00204081u) & 0x01010101u;   // bit i -> bit 8 i (the four shifted copies never overlap)
  return spread * 0xFFFFFF02u + 0xFFFFFFFFu;                        // -254 * spread - 1 = ~(0xFE * spread), bytewise
}

// The A fragment of wgmma m64nNk32 .s8 for one k-step, from the PTX ISA's register layout for A: warp w of the
// warpgroup holds rows 16 w .. 16 w + 15; its lane (g = lane / 4, t = lane % 4) holds
//   a[0] = row g,     columns 4 t .. 4 t + 3        a[2] = row g,     columns 16 + 4 t .. 16 + 4 t + 3
//   a[1] = row g + 8, columns 4 t .. 4 t + 3        a[3] = row g + 8, columns 16 + 4 t .. 16 + 4 t + 3
// with the lowest column in the lowest byte.  lo / hi: the k-step's code word of rows g and g + 8.
__host__ __device__ __forceinline__ void b1_a_fragment(uint32_t lo, uint32_t hi, int t, uint32_t (&a)[4]) {
  a[0] = b1_widen4((lo >> (4 * t)) & 0xFu);
  a[1] = b1_widen4((hi >> (4 * t)) & 0xFu);
  a[2] = b1_widen4((lo >> (16 + 4 * t)) & 0xFu);
  a[3] = b1_widen4((hi >> (16 + 4 * t)) & 0xFu);
}

}  // namespace crag
