// The int8 shard's quantiser and rescore kernels (csrc/quant_kernels.cuh) on emulated thread blocks (warp_emu.h).
// A driver for tests/test_quant_emulated.py, which writes the inputs, runs one mode and compares the outputs with
// oracle/quant_oracle.py bit for bit:
//   quant_emu_test values  <in> <out>   in: int32 m; float32 x[m], s[m]         out: int32 quant_value(x, s) [m]
//   quant_emu_test quant   <in> <out>   in: int32 n, dim, row_stride, dim8; uint16 rows[n * row_stride]
//                                       out: int8 [n * dim8], float32 scales[n]
//   quant_emu_test rescore <in> <out>   in: int64 n_rows, row_offset; int32 dim, row_stride, nq, n_cand, k;
//                                           uint16 rows[n_rows * row_stride], queries[nq * dim]; int64 cand[nq * n_cand]
//                                       out: int64 ids[nq * k], float32 scores[nq * k]
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
static inline int __float2int_rn(float x) { return int(nearbyintf(x)); }   // default rounding mode: half to even
static inline float __int2float_rn(int x) { return float(x); }

#include "quant_kernels.cuh"

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
  if (argc != 4) { fprintf(stderr, "usage: %s values|quant|rescore <in> <out>\n", argv[0]); return 2; }
  fin = fopen(argv[2], "rb");
  FILE* fout = fopen(argv[3], "wb");
  if (!fin || !fout) { fprintf(stderr, "cannot open files\n"); return 2; }
  const char* mode = argv[1];
  if (!strcmp(mode, "values")) {
    const int m = rd<int32_t>();
    auto x = rdv<float>(m), s = rdv<float>(m);
    std::vector<int32_t> out(m);
    warp_emu::run_warp([&](int lane) {
      for (int i = lane; i < m; i += 32) out[i] = quant_value(x[i], s[i]);
    });
    wr(fout, out);
  } else if (!strcmp(mode, "quant")) {
    const int n = rd<int32_t>(), dim = rd<int32_t>(), row_stride = rd<int32_t>(), dim8 = rd<int32_t>();
    auto rows = rdv<uint16_t>(size_t(n) * row_stride);
    std::vector<int8_t> out(size_t(n) * dim8 + 4, int8_t(0x5A));   // garbage the kernel must overwrite
    std::vector<float> scales(n, -7.f);
    const int per_block = kQuantThreads / 32;
    warp_emu::launch((n + per_block - 1) / per_block, kQuantThreads, [&] {
      quantize_rows_kernel(rows.data(), n, dim, row_stride, dim8, out.data(), dim8, scales.data());
    });
    out.resize(size_t(n) * dim8);
    wr(fout, out);
    wr(fout, scales);
  } else if (!strcmp(mode, "rescore")) {
    const int64_t n_rows = rd<int64_t>(), row_offset = rd<int64_t>();
    const int dim = rd<int32_t>(), row_stride = rd<int32_t>(), nq = rd<int32_t>(), n_cand = rd<int32_t>(), k = rd<int32_t>();
    auto rows = rdv<uint16_t>(size_t(n_rows) * row_stride);
    auto queries = rdv<uint16_t>(size_t(nq) * dim);
    auto cand = rdv<int64_t>(size_t(nq) * n_cand);
    std::vector<int64_t> ids(size_t(nq) * k, -7);
    std::vector<float> scores(size_t(nq) * k, -7.f);
    warp_emu::launch(nq, kRescoreThreads, [&] {
      rescore_topk_kernel(rows.data(), n_rows, dim, row_stride, row_offset, queries.data(), cand.data(), n_cand, k,
                          ids.data(), scores.data());
    });
    wr(fout, ids);
    wr(fout, scores);
  } else {
    fprintf(stderr, "unknown mode %s\n", mode);
    return 2;
  }
  fclose(fout);
  return 0;
}
