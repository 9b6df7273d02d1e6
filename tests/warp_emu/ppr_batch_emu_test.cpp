// The kernels of crag_ppr_batch (csrc/ppr_batch_kernels.cuh) against those of crag_ppr (csrc/ppr_kernels.cuh) on
// emulated thread blocks (warp_emu.h), both enqueued as ppr.cu enqueues them.  Every case holds B resets; each one
// runs alone through the single-source kernels, then the batch runs through the batched kernels for every batch size
// given, once block after block and `interleavings` times with all blocks resident in random interleavings.  Column
// b of every batched run must equal the single run of reset b bit for bit.
//
// usage: ppr_batch_emu_test <batch sizes, e.g. 1,2,3,8> <interleavings> case.bin [case.bin ...]
// Case file (little endian): int64 n, nnz, n_out (-1: out_vertices NULL), iterations, B; float damping;
// int64 row_ptr[n + 1]; int32 col[nnz]; float coef[nnz]; float resets[B][n]; int32 out_vertices[n_out].
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>   // the stub

#include "ppr_kernels.cuh"
#include "ppr_batch_kernels.cuh"

using namespace crag;

#define REQUIRE(cond, ...)                                                \
  do {                                                                    \
    if (!(cond)) {                                                        \
      fprintf(stderr, "FAILED %s:%d: %s\n  ", __FILE__, __LINE__, #cond); \
      fprintf(stderr, __VA_ARGS__);                                       \
      fprintf(stderr, "\n");                                              \
      exit(1);                                                            \
    }                                                                     \
  } while (0)

struct Case {
  int64_t n = 0, nnz = 0, n_out = 0, iterations = 0, batch = 0;
  float damping = 0.f;
  std::vector<int64_t> row_ptr;
  std::vector<int32_t> col, out_vertices;
  std::vector<float> coef, resets;
};

template <class T>
static void read_into(FILE* f, std::vector<T>& v, int64_t count) {
  v.resize(size_t(count));
  REQUIRE(fread(v.data(), sizeof(T), size_t(count), f) == size_t(count), "short case file");
}

static Case read_case(const char* path) {
  FILE* f = fopen(path, "rb");
  REQUIRE(f != nullptr, "cannot open %s", path);
  Case c;
  int64_t head[5];
  REQUIRE(fread(head, 8, 5, f) == 5 && fread(&c.damping, 4, 1, f) == 1, "short case header");
  c.n = head[0], c.nnz = head[1], c.n_out = head[2], c.iterations = head[3], c.batch = head[4];
  read_into(f, c.row_ptr, c.n + 1);
  read_into(f, c.col, c.nnz);
  read_into(f, c.coef, c.nnz);
  read_into(f, c.resets, c.batch * c.n);
  if (c.n_out >= 0) read_into(f, c.out_vertices, c.n_out);
  fclose(f);
  return c;
}

static void launch(uint64_t seed, unsigned grid, int block, size_t smem, const std::function<void()>& body) {
  if (grid == 0) return;
  if (seed == 0) warp_emu::launch(grid, block, body, smem);
  else warp_emu::launch_concurrent(grid, block, body, smem, seed, 64 << 10);
}

static unsigned blocks(int64_t items, int per_block) { return unsigned((items + per_block - 1) / per_block); }

// crag_ppr's sequence for reset b
static std::vector<float> run_single(const Case& c, int64_t b) {
  const int64_t n = c.n, nnz = c.nnz;
  const int64_t n_out = c.n_out < 0 ? n : c.n_out;
  const int32_t* out_vertices = c.n_out < 0 ? nullptr : c.out_vertices.data();
  warp_emu::Workspace ws(plan_ppr(n, nnz).total, kWsAlign, 0xFF);   // NaN everywhere
  const PprPlan p = plan_ppr(n, nnz, ws.base);
  const int64_t* row_ptr = c.row_ptr.data();
  const int32_t* col = c.col.data();
  const float* coef = c.coef.data();
  const float* reset = c.resets.data() + b * n;
  const float d = c.damping;
  std::vector<float> out(size_t(n_out), -7.f);
  if (c.iterations > 0)
    launch(0, blocks(p.segments + 1, kPprThreads), kPprThreads, 0,
           [&] { ppr_plan_kernel(row_ptr, n, nnz, p.segments, p.seg_row, p.head_row); });
  launch(0, blocks(n, kPprThreads), kPprThreads, 0, [&] { ppr_init_kernel(reset, d, n, p.y[0]); });
  for (int64_t t = 0; t < c.iterations; ++t) {
    const float* y_in = p.y[t & 1];
    float* y_out = p.y[(t + 1) & 1];
    launch(0, blocks(p.segments, kPprStepWarps), kPprStepThreads, kPprStepSmemBytes, [&] {
      ppr_step_kernel(row_ptr, col, coef, reset, d, y_in, y_out, p.seg_row, p.head_row, n, nnz, p.segments, p.head_val, p.carry);
    });
    launch(0, blocks(p.segments, kPprThreads), kPprThreads, 0,
           [&] { ppr_fixup_kernel(row_ptr, reset, d, p.head_row, p.head_val, p.carry, p.segments, y_out); });
  }
  const float* y_T = p.y[c.iterations & 1];
  launch(0, unsigned(p.sum_blocks), kPprThreads, kPprSumSmemBytes, [&] { ppr_sum_kernel(y_T, n, p.partials); });
  if (n_out > 0)
    launch(0, blocks(n_out, kPprThreads), kPprThreads, kPprSumSmemBytes,
           [&] { ppr_gather_kernel(y_T, p.partials, p.sum_blocks, out_vertices, n_out, out.data()); });
  return out;
}

// crag_ppr_batch's sequence (ppr.cu's launch_ppr_batch) for the first `batch` resets; out [batch][n_out]
template <int W>
static std::vector<float> run_batch(const Case& c, int batch, uint64_t seed) {
  const int64_t n = c.n, nnz = c.nnz;
  const int64_t n_out = c.n_out < 0 ? n : c.n_out;
  const int32_t* out_vertices = c.n_out < 0 ? nullptr : c.out_vertices.data();
  warp_emu::Workspace ws(plan_ppr_batch(n, nnz, batch).total, kWsAlign, 0xFF);
  const PprBatchPlan p = plan_ppr_batch(n, nnz, batch, ws.base);
  REQUIRE(p.width == W, "width %d for batch %d", p.width, batch);
  const int64_t* row_ptr = c.row_ptr.data();
  const int32_t* col = c.col.data();
  const float* coef = c.coef.data();
  const float* resets = c.resets.data();
  const float d = c.damping;
  std::vector<float> out(size_t(batch * n_out), -7.f);
  if (c.iterations > 0)
    launch(seed, blocks(p.segments + 1, kPprThreads), kPprThreads, 0,
           [&] { ppr_plan_kernel(row_ptr, n, nnz, p.segments, p.seg_row, p.head_row); });
  launch(seed, blocks(n * W, kPprThreads), kPprThreads, 0,
         [&] { ppr_batch_init_kernel<W>(resets, batch, d, n, p.v, p.y[0]); });
  for (int64_t t = 0; t < c.iterations; ++t) {
    const float* y_in = p.y[t & 1];
    float* y_out = p.y[(t + 1) & 1];
    launch(seed ? seed + 2 * t : 0, blocks(p.segments, kPprStepWarps), kPprStepThreads, kPprBatchStepSmemBytes, [&] {
      ppr_batch_step_kernel<W>(row_ptr, col, coef, p.v, d, y_in, y_out, p.seg_row, p.head_row, n, nnz, p.segments, p.head_val,
                               p.carry);
    });
    launch(seed ? seed + 2 * t + 1 : 0, blocks(p.segments * W, kPprThreads), kPprThreads, 0,
           [&] { ppr_batch_fixup_kernel<W>(row_ptr, p.v, d, p.head_row, p.head_val, p.carry, p.segments, y_out); });
  }
  const float* y_T = p.y[c.iterations & 1];
  launch(seed, unsigned(p.sum_blocks), kPprThreads, kPprSumSmemBytes, [&] { ppr_batch_sum_kernel<W>(y_T, n, p.partials); });
  launch(seed, unsigned(W), kPprThreads, kPprSumSmemBytes,
         [&] { ppr_batch_total_kernel<W>(p.partials, p.sum_blocks, p.totals); });
  const int64_t per_column = blocks(n_out, kPprThreads);
  if (n_out > 0)
    launch(seed, unsigned(per_column * batch), kPprThreads, 0,
           [&] { ppr_batch_gather_kernel<W>(y_T, p.totals, out_vertices, n_out, per_column, out.data()); });
  return out;
}

static std::vector<float> run_batch(const Case& c, int batch, uint64_t seed) {
  switch (ppr_batch_width(batch)) {
    case 2: return run_batch<2>(c, batch, seed);
    case 4: return run_batch<4>(c, batch, seed);
    case 8: return run_batch<8>(c, batch, seed);
    case 16: return run_batch<16>(c, batch, seed);
    default: return run_batch<32>(c, batch, seed);
  }
}

int main(int argc, char** argv) {
  REQUIRE(argc >= 4, "usage: ppr_batch_emu_test <batch sizes> <interleavings> case.bin [case.bin ...]");
  std::vector<int> sizes;
  for (const char* s = argv[1]; *s;) {
    sizes.push_back(atoi(s));
    while (*s && *s != ',') ++s;
    if (*s == ',') ++s;
  }
  const int interleavings = atoi(argv[2]);
  for (int a = 3; a < argc; ++a) {
    const Case c = read_case(argv[a]);
    const int64_t n_out = c.n_out < 0 ? c.n : c.n_out;
    std::vector<std::vector<float>> single;
    for (int64_t b = 0; b < c.batch; ++b) single.push_back(run_single(c, b));
    for (int batch : sizes) {
      REQUIRE(batch >= 1 && batch <= c.batch && batch <= kPprMaxBatch, "batch %d of %lld resets", batch, (long long)c.batch);
      for (int r = 0; r <= interleavings; ++r) {
        const uint64_t seed = r == 0 ? 0 : 11 + 20251016ull * uint64_t(r);
        const std::vector<float> got = run_batch(c, batch, seed);
        for (int b = 0; b < batch; ++b) {
          const float* col = got.data() + size_t(b) * size_t(n_out);
          if (memcmp(col, single[b].data(), size_t(n_out) * 4) == 0) continue;
          int64_t p = 0;
          while (memcmp(col + p, single[b].data() + p, 4) == 0) ++p;
          REQUIRE(false, "%s: batch %d, column %d, interleaving %d: out[%lld] = %.9g, crag_ppr alone gives %.9g", argv[a],
                  batch, b, r, (long long)p, double(col[p]), double(single[b][p]));
        }
      }
    }
    printf("ok  %s: n=%lld nnz=%lld T=%lld, batches", argv[a], (long long)c.n, (long long)c.nnz, (long long)c.iterations);
    for (int batch : sizes) printf(" %d", batch);
    printf(" x %d interleavings bit-identical to the single runs\n", interleavings + 1);
  }
  printf("ALL OK\n");
  return 0;
}
