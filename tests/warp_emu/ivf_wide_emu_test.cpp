// The wide IVF stage 1 and rescore of crag_ivf_search_i8_wide / _pq_wide on emulated thread blocks (warp_emu.h), for
// one 32-query pass: the IVF plan and the wide plan (ivf_kernels.cuh), the int8 or PQ fill (ivf_wide_kernels.cuh), the
// ragged select (knn_select.cuh), the slot map and the wide IVF rescore (quant_kernels.cuh).  A driver for
// tests/test_ivf_wide_emulated.py, which writes the inputs and compares every output with tests/ivf_wide_oracle.py:
//   ivf_wide_emu_test <in> <out>
//     in:  int32 mode (0 int8, 1 PQ), n_rows_padded, dim, nq, nprobe, nlist, n_cand, k, cap, slices, width (int8: dim8,
//          PQ: m); uint16 residuals[n_rows * dim]; uint16 queries[nq * dim]; int64 probed_ids[nq * nprobe];
//          float32 probed_scores[nq * nprobe]; int32 list_tile_start[nlist + 1], list_rows[nlist];
//          int8: int8 codes[n_rows * dim8], float32 row_scales[n_rows], int8 q8[nq * dim8], float32 qs[nq]
//          PQ:   uint8 codes[n_rows * code_stride(m)], float32 codebooks[m * 256 * dim / m]
//     out: int32 n_q[nq]; float32 block[nq * ld] (unwritten slots keep the sentinel 0x7FBADBAD); int64 slots[nq * n_cand];
//          int64 positions[nq * n_cand]; float32 cand_s1[nq * n_cand]; float32 minmax[nq * 2]; int64 pos[nq * k];
//          float32 s2[nq * k]
// Compiled with -ffp-contract=off, so the plain float expressions below round each operation as the device's
// __f*_rn intrinsics do.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include <cuda_runtime.h>   // the stub

static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline int __float2int_rn(float x) { return int(nearbyintf(x)); }
static inline float __int2float_rn(int x) { return float(x); }
// the signed dp4a: c + the four byte products of a and b
static inline int __dp4a(int a, int b, int c) {
  for (int i = 0; i < 4; ++i) c += int(int8_t(uint32_t(a) >> (8 * i))) * int(int8_t(uint32_t(b) >> (8 * i)));
  return c;
}

#include "warp_emu.h"
#include "ivf_kernels.cuh"
#include "ivf_wide_kernels.cuh"
#include "knn_select.cuh"
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
  const int mode = rd<int32_t>(), n_rows = rd<int32_t>(), dim = rd<int32_t>(), nq = rd<int32_t>(), nprobe = rd<int32_t>(),
            nlist = rd<int32_t>(), n_cand = rd<int32_t>(), k = rd<int32_t>(), cap = rd<int32_t>(), slices = rd<int32_t>(),
            width = rd<int32_t>();
  if (nq > kNQ || nprobe > kIvfMaxProbe || n_cand > kKnnMaxK || k > n_cand || cap < 1) { fprintf(stderr, "bad sizes\n"); return 2; }
  auto residuals = rdv<uint16_t>(size_t(n_rows) * dim);
  auto queries = rdv<uint16_t>(size_t(nq) * dim);
  auto probed_ids = rdv<int64_t>(size_t(nq) * nprobe);
  auto probed_scores = rdv<float>(size_t(nq) * nprobe);
  auto list_tile_start = rdv<int32_t>(size_t(nlist) + 1);
  auto list_rows = rdv<int32_t>(size_t(nlist));

  const int64_t total_tiles = n_rows / kTileRows;
  std::vector<uint32_t> list_mask(nlist, 0xFFFFFFFFu);
  std::vector<float> coarse(size_t(nlist) * kNQ, NAN);
  std::vector<int4> work(size_t(total_tiles) + 1);
  int n_work = -1;
  warp_emu::launch(1, 1024, [&] {
    ivf_plan_kernel(probed_ids.data(), probed_scores.data(), nq, nprobe, nlist, list_tile_start.data(), list_rows.data(),
                    list_mask.data(), coarse.data(), work.data(), &n_work);
  });
  const IvfArgs plan{work.data(), &n_work, list_mask.data(), coarse.data()};

  std::vector<int32_t> slot_base(size_t(nlist) * kNQ, -7), seg_list(kNQ * kIvfMaxProbe, -7), seg_slot(kNQ * kIvfMaxProbe, -7),
      n_seg(kNQ, -7), n_q(kNQ, -7);
  const IvfWidePlan wp{slot_base.data(), seg_list.data(), seg_slot.data(), n_seg.data(), n_q.data()};
  warp_emu::launch(nq, kIvfMaxProbe, [&] {
    ivf_wide_plan_kernel(probed_ids.data(), nprobe, nlist, list_rows.data(), cap, wp);
  });

  const int64_t ld = (cap + 3) & ~3;
  uint32_t sentinel = 0x7FBADBADu;
  float fill_value;
  memcpy(&fill_value, &sentinel, 4);
  std::vector<float> block(size_t(nq) * ld, fill_value);
  const IvfWideBlock out{list_tile_start.data(), slot_base.data(), block.data(), ld, cap};
  if (mode == 0) {
    const int dim8 = width;
    auto codes = rdv<int8_t>(size_t(n_rows) * dim8);
    auto row_scales = rdv<float>(size_t(n_rows));
    auto q8 = rdv<int8_t>(size_t(nq) * dim8);
    auto qs = rdv<float>(size_t(nq));
    warp_emu::launch(unsigned(nq * slices), kIvfFillThreads, [&] {
      ivf_fill_i8_kernel(codes.data(), dim8, dim8, row_scales.data(), q8.data(), qs.data(), slices, plan, out);
    });
  } else {
    const int m = width, cs = pq_code_stride(m);
    auto codes = rdv<uint8_t>(size_t(n_rows) * cs);
    auto codebooks = rdv<float>(size_t(dim) * kPqCodewords);
    std::vector<float> lut(size_t(nq) * m * kPqCodewords);
    warp_emu::launch(unsigned(nq * m), kPqTableThreads, [&] { pq_table_kernel(queries.data(), dim, codebooks.data(), m, lut.data()); });
    warp_emu::launch(unsigned(nq * slices), kIvfFillThreads, [&] {
      ivf_fill_pq_kernel(codes.data(), cs, m, lut.data(), slices, plan, out);
    }, size_t(m) * kPqCodewords * 4);
  }

  std::vector<int64_t> cand(size_t(nq) * n_cand, -7);
  std::vector<float> cand_s1(size_t(nq) * n_cand, -7.f), minmax(size_t(nq) * 2, -7.f);
  warp_emu::launch(nq, kKnnThreads, [&] {
    ivf_wide_select_kernel(block.data(), ld, n_q.data(), n_cand, cand.data(), cand_s1.data(), minmax.data());
  });
  const std::vector<int64_t> slots = cand;
  warp_emu::launch(unsigned((nq * n_cand + 255) / 256), 256, [&] {
    ivf_slot_map_kernel(cand.data(), nq, n_cand, wp, list_tile_start.data());
  });

  std::vector<int64_t> pos(size_t(nq) * k, -7);
  std::vector<float> s2(size_t(nq) * k, -7.f);
  warp_emu::launch(nq, kKnnThreads, [&] {
    ivf_rescore_wide_kernel(residuals.data(), n_rows, dim, dim, queries.data(), cand.data(), n_cand, k, pos.data(),
                            s2.data(), IvfListTerm{list_tile_start.data(), nlist, coarse.data()});
  });

  n_q.resize(nq);
  wr(fout, n_q);
  wr(fout, block);
  wr(fout, slots);
  wr(fout, cand);
  wr(fout, cand_s1);
  wr(fout, minmax);
  wr(fout, pos);
  wr(fout, s2);
  fclose(fout);
  return 0;
}
