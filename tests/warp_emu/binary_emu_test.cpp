// The one-bit shard's binarize kernel (csrc/quant_kernels.cuh) on emulated thread blocks (warp_emu.h), and the map
// from code bits to the wgmma A fragment (csrc/binary.cuh) on every lane.  A driver for tests/test_binary_emulated.py,
// which writes the inputs, runs one mode and compares the outputs with tests/binary_oracle.py and a model of the PTX
// register layout:
//   binary_emu_test binarize <in> <out>   in: int32 n, dim, row_stride, dim8; uint16 rows[n * row_stride]
//                                         out: uint8 codes[n * dim8 / 8], float32 alpha[n]
//   binary_emu_test fragment <in> <out>   in: int32 m; uint32 words[m][16] (k-step words of rows 0 .. 15 of a warp)
//                                         out: uint32 a[m][32 lanes][4] (b1_a_fragment of each lane)
// Compiled with -ffp-contract=off, so the plain float expressions below round each operation as the device's
// __f*_rn intrinsics do.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include <cuda_runtime.h>   // the stub

static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline int __float2int_rn(float x) { return int(nearbyintf(x)); }
static inline float __int2float_rn(int x) { return float(x); }

#include "quant_kernels.cuh"
#include "binary.cuh"

using namespace crag;

static FILE* fin;
template <class T> static T rd() { T v; if (fread(&v, sizeof(T), 1, fin) != 1) { fprintf(stderr, "short input\n"); exit(2); } return v; }
template <class T> static std::vector<T> rdv(size_t n) {
  std::vector<T> v(n);
  if (n && fread(v.data(), sizeof(T), n, fin) != n) { fprintf(stderr, "short input\n"); exit(2); }
  return v;
}
template <class T> static void wr(FILE* f, const std::vector<T>& v) { fwrite(v.data(), sizeof(T), v.size(), f); }

int main(int argc, char** argv) {
  if (argc != 4) { fprintf(stderr, "usage: %s binarize|fragment <in> <out>\n", argv[0]); return 2; }
  fin = fopen(argv[2], "rb");
  FILE* fout = fopen(argv[3], "wb");
  if (!fin || !fout) { fprintf(stderr, "cannot open files\n"); return 2; }
  const char* mode = argv[1];
  if (!strcmp(mode, "binarize")) {
    const int n = rd<int32_t>(), dim = rd<int32_t>(), row_stride = rd<int32_t>(), dim8 = rd<int32_t>();
    auto rows = rdv<uint16_t>(size_t(n) * row_stride);
    std::vector<uint32_t> words(size_t(n) * dim8 / 32 + 1, 0x5A5A5A5Au);   // garbage the kernel must overwrite
    std::vector<float> alpha(n, -7.f);
    const int per_block = kBinarizeThreads / 32;
    warp_emu::launch((n + per_block - 1) / per_block, kBinarizeThreads, [&] {
      binarize_rows_kernel(rows.data(), n, dim, row_stride, dim8, reinterpret_cast<uint8_t*>(words.data()), dim8 / 8,
                           alpha.data());
    });
    std::vector<uint8_t> codes(size_t(n) * dim8 / 8);
    memcpy(codes.data(), words.data(), codes.size());
    wr(fout, codes);
    wr(fout, alpha);
  } else if (!strcmp(mode, "fragment")) {
    const int m = rd<int32_t>();
    auto words = rdv<uint32_t>(size_t(m) * 16);
    std::vector<uint32_t> out(size_t(m) * 32 * 4);
    for (int i = 0; i < m; ++i)
      warp_emu::run_warp([&](int lane) {
        uint32_t a[4];
        const int g = lane >> 2;
        b1_a_fragment(words[i * 16 + g], words[i * 16 + g + 8], lane & 3, a);
        for (int r = 0; r < 4; ++r) out[(size_t(i) * 32 + lane) * 4 + r] = a[r];
      });
    wr(fout, out);
  } else {
    fprintf(stderr, "unknown mode %s\n", mode);
    return 2;
  }
  fclose(fout);
  return 0;
}
