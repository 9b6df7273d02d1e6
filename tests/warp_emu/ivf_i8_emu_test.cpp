// The IVF rescore of crag_ivf_search_i8 (ivf_rescore_topk_kernel, csrc/quant_kernels.cuh) and the id map that follows
// it (ivf_map_ids_kernel, csrc/ivf_kernels.cuh) on emulated thread blocks (warp_emu.h).  A driver for
// tests/test_ivf_i8_emulated.py, which writes the inputs and compares the outputs with tests/ivf_i8_oracle.py:
//   ivf_i8_emu_test <in> <out>
//     in:  int64 n_rows; int32 dim, row_stride, nq, n_cand, k, nlist; uint16 rows[n_rows * row_stride],
//          queries[nq * dim]; int64 cand[nq * n_cand] (stored positions); int32 list_tile_start[nlist + 1];
//          float32 coarse[nlist * 32]; int64 row_ids[n_rows]
//     out: int64 ids[nq * k] (original ids), float32 scores[nq * k]
// Compiled with -ffp-contract=off, so the plain float expressions below round each operation as the device's
// __f*_rn intrinsics do.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include <cuda_runtime.h>   // the stub

static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline int __float2int_rn(float x) { return int(nearbyintf(x)); }   // default rounding mode: half to even
static inline float __int2float_rn(int x) { return float(x); }

#include "ivf_kernels.cuh"
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
  const int64_t n_rows = rd<int64_t>();
  const int dim = rd<int32_t>(), row_stride = rd<int32_t>(), nq = rd<int32_t>(), n_cand = rd<int32_t>(), k = rd<int32_t>(),
            nlist = rd<int32_t>();
  auto rows = rdv<uint16_t>(size_t(n_rows) * row_stride);
  auto queries = rdv<uint16_t>(size_t(nq) * dim);
  auto cand = rdv<int64_t>(size_t(nq) * n_cand);
  auto list_tile_start = rdv<int32_t>(size_t(nlist) + 1);
  auto coarse = rdv<float>(size_t(nlist) * kNQ);
  auto row_ids = rdv<int64_t>(size_t(n_rows));
  std::vector<int64_t> ids(size_t(nq) * k, -7);
  std::vector<float> scores(size_t(nq) * k, -7.f);
  warp_emu::launch(nq, kRescoreThreads, [&] {
    ivf_rescore_topk_kernel(rows.data(), n_rows, dim, row_stride, queries.data(), cand.data(), n_cand, k, ids.data(),
                            scores.data(), IvfListTerm{list_tile_start.data(), nlist, coarse.data()});
  });
  const int n = nq * k;
  warp_emu::launch((n + 255) / 256, 256, [&] { ivf_map_ids_kernel(ids.data(), n, row_ids.data()); });
  wr(fout, ids);
  wr(fout, scores);
  fclose(fout);
  return 0;
}
