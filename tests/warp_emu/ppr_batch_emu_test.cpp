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

// aligned workspace filled with NaN bytes: nothing may read what it did not write
struct Workspace {
  std::vector<uint8_t> mem;
  uint8_t* base;
  explicit Workspace(size_t bytes) : mem(bytes + 256, 0xFF) {
    base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(mem.data()) + 255) & ~uintptr_t(255));
  }
};

// crag_ppr's sequence for reset b
static std::vector<float> run_single(const Case& c, int64_t b) {
  const int64_t n = c.n, nnz = c.nnz;
  const int64_t n_out = c.n_out < 0 ? n : c.n_out;
  const int32_t* out_vertices = c.n_out < 0 ? nullptr : c.out_vertices.data();
  const PprPlan p = plan_ppr(n, nnz);
  Workspace w(p.total);
  uint8_t* ws = w.base;
  float* y[2] = {reinterpret_cast<float*>(ws), reinterpret_cast<float*>(ws + p.y_bytes)};
  int32_t* seg_row = reinterpret_cast<int32_t*>(ws + p.seg_row_off);
  int32_t* head_row = reinterpret_cast<int32_t*>(ws + p.head_row_off);
  float* head_val = reinterpret_cast<float*>(ws + p.head_val_off);
  float* carry = reinterpret_cast<float*>(ws + p.carry_off);
  float* partials = reinterpret_cast<float*>(ws + p.partial_off);
  const int64_t* row_ptr = c.row_ptr.data();
  const int32_t* col = c.col.data();
  const float* coef = c.coef.data();
  const float* reset = c.resets.data() + b * n;
  const float d = c.damping;
  std::vector<float> out(size_t(n_out), -7.f);
  if (c.iterations > 0)
    launch(0, blocks(p.segments + 1, kPprThreads), kPprThreads, 0,
           [&] { ppr_plan_kernel(row_ptr, n, nnz, p.segments, seg_row, head_row); });
  launch(0, blocks(n, kPprThreads), kPprThreads, 0, [&] { ppr_init_kernel(reset, d, n, y[0]); });
  for (int64_t t = 0; t < c.iterations; ++t) {
    const float* y_in = y[t & 1];
    float* y_out = y[(t + 1) & 1];
    launch(0, blocks(p.segments, kPprStepWarps), kPprStepThreads, kPprStepSmemBytes, [&] {
      ppr_step_kernel(row_ptr, col, coef, reset, d, y_in, y_out, seg_row, head_row, n, nnz, p.segments, head_val, carry);
    });
    launch(0, blocks(p.segments, kPprThreads), kPprThreads, 0,
           [&] { ppr_fixup_kernel(row_ptr, reset, d, head_row, head_val, carry, p.segments, y_out); });
  }
  const float* y_T = y[c.iterations & 1];
  launch(0, unsigned(p.sum_blocks), kPprThreads, kPprSumSmemBytes, [&] { ppr_sum_kernel(y_T, n, partials); });
  if (n_out > 0)
    launch(0, blocks(n_out, kPprThreads), kPprThreads, kPprSumSmemBytes,
           [&] { ppr_gather_kernel(y_T, partials, p.sum_blocks, out_vertices, n_out, out.data()); });
  return out;
}

// crag_ppr_batch's sequence (ppr.cu's launch_ppr_batch) for the first `batch` resets; out [batch][n_out]
template <int W>
static std::vector<float> run_batch(const Case& c, int batch, uint64_t seed) {
  const int64_t n = c.n, nnz = c.nnz;
  const int64_t n_out = c.n_out < 0 ? n : c.n_out;
  const int32_t* out_vertices = c.n_out < 0 ? nullptr : c.out_vertices.data();
  const PprBatchPlan p = plan_ppr_batch(n, nnz, batch);
  REQUIRE(p.width == W, "width %d for batch %d", p.width, batch);
  Workspace w(p.total);
  uint8_t* ws = w.base;
  float* y[2] = {reinterpret_cast<float*>(ws), reinterpret_cast<float*>(ws + p.y_bytes)};
  float* v = reinterpret_cast<float*>(ws + p.v_off);
  int32_t* seg_row = reinterpret_cast<int32_t*>(ws + p.seg_row_off);
  int32_t* head_row = reinterpret_cast<int32_t*>(ws + p.head_row_off);
  float* head_val = reinterpret_cast<float*>(ws + p.head_val_off);
  float* carry = reinterpret_cast<float*>(ws + p.carry_off);
  float* partials = reinterpret_cast<float*>(ws + p.partial_off);
  float* totals = reinterpret_cast<float*>(ws + p.total_off);
  const int64_t* row_ptr = c.row_ptr.data();
  const int32_t* col = c.col.data();
  const float* coef = c.coef.data();
  const float* resets = c.resets.data();
  const float d = c.damping;
  std::vector<float> out(size_t(batch * n_out), -7.f);
  if (c.iterations > 0)
    launch(seed, blocks(p.segments + 1, kPprThreads), kPprThreads, 0,
           [&] { ppr_plan_kernel(row_ptr, n, nnz, p.segments, seg_row, head_row); });
  launch(seed, blocks(n * W, kPprThreads), kPprThreads, 0,
         [&] { ppr_batch_init_kernel<W>(resets, batch, d, n, v, y[0]); });
  for (int64_t t = 0; t < c.iterations; ++t) {
    const float* y_in = y[t & 1];
    float* y_out = y[(t + 1) & 1];
    launch(seed ? seed + 2 * t : 0, blocks(p.segments, kPprStepWarps), kPprStepThreads, kPprBatchStepSmemBytes, [&] {
      ppr_batch_step_kernel<W>(row_ptr, col, coef, v, d, y_in, y_out, seg_row, head_row, n, nnz, p.segments, head_val,
                               carry);
    });
    launch(seed ? seed + 2 * t + 1 : 0, blocks(p.segments * W, kPprThreads), kPprThreads, 0,
           [&] { ppr_batch_fixup_kernel<W>(row_ptr, v, d, head_row, head_val, carry, p.segments, y_out); });
  }
  const float* y_T = y[c.iterations & 1];
  launch(seed, unsigned(p.sum_blocks), kPprThreads, kPprSumSmemBytes, [&] { ppr_batch_sum_kernel<W>(y_T, n, partials); });
  launch(seed, unsigned(W), kPprThreads, kPprSumSmemBytes,
         [&] { ppr_batch_total_kernel<W>(partials, p.sum_blocks, totals); });
  const int64_t per_column = blocks(n_out, kPprThreads);
  if (n_out > 0)
    launch(seed, unsigned(per_column * batch), kPprThreads, 0,
           [&] { ppr_batch_gather_kernel<W>(y_T, totals, out_vertices, n_out, per_column, out.data()); });
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
