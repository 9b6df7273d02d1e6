// The PQ kernels of crag_ivf_search_pq and crag_pq_encode (csrc/pq_kernels.cuh) on emulated thread blocks
// (warp_emu.h): the encode, the per-query tables, the IVF plan (ivf_kernels.cuh), the PQ scan and the merge of its
// per-CTA lists (merge_kernels.cuh) for one 32-query pass.  A driver for tests/test_ivf_pq_emulated.py, which writes the
// inputs and compares the outputs with tests/ivf_pq_oracle.py:
//   ivf_pq_emu_test <in> <out>
//     in:  int64 n_rows; int32 dim, m, code_stride, nq, nprobe, nlist, n_cand, slices, interleave_seed (0: blocks one
//          after the other); uint16 rows[n_rows * dim]; float32 codebooks[m * 256 * dim / m]; uint16 queries[nq * dim];
//          int64 probed_ids[nq * nprobe]; float32 probed_scores[nq * nprobe]; int32 list_tile_start[nlist + 1],
//          list_rows[nlist]
//     out: uint8 codes[n_rows * code_stride]; float32 lut[nq * m * 256]; int64 cand_pos[nq * n_cand];
//          float32 cand_s1[nq * n_cand]; float32 minmax[nq * 2]
// Compiled with -ffp-contract=off, so the plain float expressions below round each operation as the device's
// __f*_rn intrinsics do.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include <cuda_runtime.h>   // the stub

static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }

#include "warp_emu.h"
#include "ivf_kernels.cuh"
#include "merge_kernels.cuh"
#include "pq_kernels.cuh"

using namespace crag;

static FILE* fin;
template <class T> static T rd() { T v; if (fread(&v, sizeof(T), 1, fin) != 1) { fprintf(stderr, "short input\n"); exit(2); } return v; }
template <class T> static std::vector<T> rdv(size_t n) {
  std::vector<T> v(n);
  if (n && fread(v.data(), sizeof(T), n, fin) != n) { fprintf(stderr, "short input\n"); exit(2); }
  return v;
}
template <class T> static void wr(FILE* f, const std::vector<T>& v) { fwrite(v.data(), sizeof(T), v.size(), f); }

static void run(unsigned grid, int block, const std::function<void()>& body, size_t smem, uint64_t seed) {
  if (seed == 0) warp_emu::launch(grid, block, body, smem);
  else warp_emu::launch_concurrent(grid, block, body, smem, seed, 96 << 10);
}

template <int T>
static void scan_and_merge(const std::vector<uint8_t>& codes, int code_stride, int m, const std::vector<float>& lut,
                           int nq, int n_cand, int slices, const IvfArgs& plan, uint64_t seed, std::vector<int64_t>& pos,
                           std::vector<float>& s1, std::vector<float>& minmax) {
  warp_emu::Workspace parts(size_t(slices) * kNQ * n_cand * 8, 256, 0xFF), mm(size_t(slices) * kNQ * 2 * 4, 256, 0xFF);
  uint64_t* part_keys = reinterpret_cast<uint64_t*>(parts.base);
  float* part_minmax = reinterpret_cast<float*>(mm.base);
  run(unsigned(nq * slices), kPqThreads, [&] {
    pq_scan_kernel<T>(codes.data(), code_stride, m, lut.data(), slices, n_cand, plan, part_keys, part_minmax);
  }, PqScanSmem<T>::bytes(m), seed);
  warp_emu::launch(nq, 128, [&] {
    merge_topk_kernel<T, T, false>(part_keys, nullptr, nullptr, part_minmax, slices, kNQ, nq, n_cand, 0, 0, 0, 0,
                                   pos.data(), s1.data(), minmax.data(), nullptr);
  });
}

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s <in> <out>\n", argv[0]); return 2; }
  fin = fopen(argv[1], "rb");
  FILE* fout = fopen(argv[2], "wb");
  if (!fin || !fout) { fprintf(stderr, "cannot open files\n"); return 2; }
  const int64_t n_rows = rd<int64_t>();
  const int dim = rd<int32_t>(), m = rd<int32_t>(), code_stride = rd<int32_t>(), nq = rd<int32_t>(), nprobe = rd<int32_t>(),
            nlist = rd<int32_t>(), n_cand = rd<int32_t>(), slices = rd<int32_t>(), seed = rd<int32_t>();
  auto rows = rdv<uint16_t>(size_t(n_rows) * dim);
  auto codebooks = rdv<float>(size_t(dim) * 256);
  auto queries = rdv<uint16_t>(size_t(nq) * dim);
  auto probed_ids = rdv<int64_t>(size_t(nq) * nprobe);
  auto probed_scores = rdv<float>(size_t(nq) * nprobe);
  auto list_tile_start = rdv<int32_t>(size_t(nlist) + 1);
  auto list_rows = rdv<int32_t>(size_t(nlist));
  if (nq > kNQ) { fprintf(stderr, "one pass holds at most %d queries\n", kNQ); return 2; }

  std::vector<uint8_t> codes(size_t(n_rows) * code_stride, 0);
  warp_emu::launch(unsigned((n_rows + kPqThreads - 1) / kPqThreads) * unsigned(m), kPqThreads, [&] {
    pq_encode_kernel(rows.data(), n_rows, dim, dim, codebooks.data(), m, codes.data(), code_stride);
  }, pq_encode_smem_bytes(dim / m));

  std::vector<float> lut(size_t(nq) * m * kPqCodewords, -7.f);
  warp_emu::launch(unsigned(nq * m), kPqTableThreads, [&] { pq_table_kernel(queries.data(), dim, codebooks.data(), m, lut.data()); });

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

  std::vector<int64_t> pos(size_t(nq) * n_cand, -7);
  std::vector<float> s1(size_t(nq) * n_cand, -7.f), minmax(size_t(nq) * 2, -7.f);
  if (n_cand <= 32) scan_and_merge<32>(codes, code_stride, m, lut, nq, n_cand, slices, plan, uint64_t(seed), pos, s1, minmax);
  else if (n_cand <= 64) scan_and_merge<64>(codes, code_stride, m, lut, nq, n_cand, slices, plan, uint64_t(seed), pos, s1, minmax);
  else scan_and_merge<128>(codes, code_stride, m, lut, nq, n_cand, slices, plan, uint64_t(seed), pos, s1, minmax);

  wr(fout, codes);
  wr(fout, lut);
  wr(fout, pos);
  wr(fout, s1);
  wr(fout, minmax);
  fclose(fout);
  return 0;
}
