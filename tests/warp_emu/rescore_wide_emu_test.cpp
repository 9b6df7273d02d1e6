// crag_rescore_topk's kernel for more than 128 candidates (rescore_wide_kernel, csrc/quant_kernels.cuh) on emulated
// 512-thread blocks (warp_emu.h).  A driver for tests/test_rescore_wide_emulated.py, which writes the inputs, runs it
// and compares the outputs with oracle/quant_oracle.py bit for bit:
//   rescore_wide_emu_test <in> <out>
//     in:  int64 n_rows, n_alloc, row_offset; int32 dim, row_stride, nq, n_cand, k;
//          uint16 rows[n_alloc * row_stride] (n_alloc >= n_rows: rows past n_rows exist but are not the shard's),
//          queries[nq * dim]; int64 cand[nq * n_cand]
//     out: int64 ids[nq * k], float32 scores[nq * k]
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
  if (argc != 3) { fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  fin = fopen(argv[1], "rb");
  FILE* fout = fopen(argv[2], "wb");
  if (!fin || !fout) { fprintf(stderr, "cannot open files\n"); return 2; }
  const int64_t n_rows = rd<int64_t>(), n_alloc = rd<int64_t>(), row_offset = rd<int64_t>();
  const int dim = rd<int32_t>(), row_stride = rd<int32_t>(), nq = rd<int32_t>(), n_cand = rd<int32_t>(), k = rd<int32_t>();
  if (n_cand <= kRescoreMaxCand || n_cand > kKnnMaxK || k < 1 || k > n_cand || n_alloc < n_rows) {
    fprintf(stderr, "need %d < n_cand <= %d, 1 <= k <= n_cand and n_alloc >= n_rows\n", kRescoreMaxCand, kKnnMaxK);
    return 2;
  }
  auto rows = rdv<uint16_t>(size_t(n_alloc) * row_stride);
  auto queries = rdv<uint16_t>(size_t(nq) * dim);
  auto cand = rdv<int64_t>(size_t(nq) * n_cand);
  std::vector<int64_t> ids(size_t(nq) * k, -7);
  std::vector<float> scores(size_t(nq) * k, -7.f);
  warp_emu::launch(nq, kKnnThreads, [&] {
    rescore_wide_kernel(rows.data(), n_rows, dim, row_stride, row_offset, queries.data(), cand.data(), n_cand, k,
                        ids.data(), scores.data());
  });
  wr(fout, ids);
  wr(fout, scores);
  fclose(fout);
  return 0;
}
