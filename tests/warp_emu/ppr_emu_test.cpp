// The kernels of crag_ppr (csrc/ppr_kernels.cuh, the header ppr.cu includes) on emulated thread blocks (warp_emu.h):
// plan, init, T x (step, fix-up), sum and gather, enqueued as ppr.cu enqueues them.  Each case runs three times:
// blocks one after the other, then twice with all blocks resident and advancing in random interleavings (two
// seeds).  The three outputs must be bit-identical; the first is written for tests/test_ppr_emulated.py, which
// checks it against the float64 oracle and the derived error bound.
//
// Case file (little endian): int64 n, nnz, n_out (-1: out_vertices NULL), iterations; float damping;
// int64 row_ptr[n + 1]; int32 col[nnz]; float coef[nnz]; float reset[n]; int32 out_vertices[n_out].
// Output file: float out[n_out or n].
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>   // the stub

#include "ppr_kernels.cuh"

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
  int64_t n = 0, nnz = 0, n_out = 0, iterations = 0;
  float damping = 0.f;
  std::vector<int64_t> row_ptr;
  std::vector<int32_t> col, out_vertices;
  std::vector<float> coef, reset;
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
  int64_t head[4];
  REQUIRE(fread(head, 8, 4, f) == 4 && fread(&c.damping, 4, 1, f) == 1, "short case header");
  c.n = head[0], c.nnz = head[1], c.n_out = head[2], c.iterations = head[3];
  read_into(f, c.row_ptr, c.n + 1);
  read_into(f, c.col, c.nnz);
  read_into(f, c.coef, c.nnz);
  read_into(f, c.reset, c.n);
  if (c.n_out >= 0) read_into(f, c.out_vertices, c.n_out);
  fclose(f);
  return c;
}

// seed 0: blocks one after the other; otherwise all blocks resident, random interleaving drawn from the seed
static void launch(uint64_t seed, unsigned grid, int block, size_t smem, const std::function<void()>& body) {
  if (grid == 0) return;
  if (seed == 0) warp_emu::launch(grid, block, body, smem);
  else warp_emu::launch_concurrent(grid, block, body, smem, seed, 64 << 10);
}

static unsigned blocks(int64_t items, int per_block) { return unsigned((items + per_block - 1) / per_block); }

// ppr.cu's sequence for one call
static std::vector<float> run(const Case& c, uint64_t seed) {
  const int64_t n = c.n, nnz = c.nnz;
  const int64_t n_out = c.n_out < 0 ? n : c.n_out;
  const int32_t* out_vertices = c.n_out < 0 ? nullptr : c.out_vertices.data();
  warp_emu::Workspace ws(plan_ppr(n, nnz).total, kWsAlign, 0xFF);   // NaN everywhere
  const PprPlan p = plan_ppr(n, nnz, ws.base);
  const int64_t* row_ptr = c.row_ptr.data();
  const int32_t* col = c.col.data();
  const float* coef = c.coef.data();
  const float* reset = c.reset.data();
  const float d = c.damping;
  std::vector<float> out(size_t(n_out), -7.f);

  if (c.iterations > 0)
    launch(seed, blocks(p.segments + 1, kPprThreads), kPprThreads, 0,
           [&] { ppr_plan_kernel(row_ptr, n, nnz, p.segments, p.seg_row, p.head_row); });
  launch(seed, blocks(n, kPprThreads), kPprThreads, 0, [&] { ppr_init_kernel(reset, d, n, p.y[0]); });
  for (int64_t t = 0; t < c.iterations; ++t) {
    const float* y_in = p.y[t & 1];
    float* y_out = p.y[(t + 1) & 1];
    launch(seed ? seed + 2 * t : 0, blocks(p.segments, kPprStepWarps), kPprStepThreads, kPprStepSmemBytes, [&] {
      ppr_step_kernel(row_ptr, col, coef, reset, d, y_in, y_out, p.seg_row, p.head_row, n, nnz, p.segments, p.head_val, p.carry);
    });
    launch(seed ? seed + 2 * t + 1 : 0, blocks(p.segments, kPprThreads), kPprThreads, 0,
           [&] { ppr_fixup_kernel(row_ptr, reset, d, p.head_row, p.head_val, p.carry, p.segments, y_out); });
  }
  const float* y_T = p.y[c.iterations & 1];
  launch(seed, unsigned(p.sum_blocks), kPprThreads, kPprSumSmemBytes, [&] { ppr_sum_kernel(y_T, n, p.partials); });
  if (n_out > 0)
    launch(seed, blocks(n_out, kPprThreads), kPprThreads, kPprSumSmemBytes,
           [&] { ppr_gather_kernel(y_T, p.partials, p.sum_blocks, out_vertices, n_out, out.data()); });
  return out;
}

int main(int argc, char** argv) {
  REQUIRE(argc >= 3 && argc % 2 == 1, "usage: ppr_emu_test case.bin out.bin [case.bin out.bin ...]");
  for (int a = 1; a < argc; a += 2) {
    const Case c = read_case(argv[a]);
    const std::vector<float> base = run(c, 0);
    for (uint64_t seed : {11ull, 20251016ull}) {
      const std::vector<float> again = run(c, seed);
      REQUIRE(memcmp(base.data(), again.data(), base.size() * 4) == 0,
              "%s: output differs between block interleavings (seed %llu)", argv[a], (unsigned long long)seed);
    }
    FILE* f = fopen(argv[a + 1], "wb");
    REQUIRE(f != nullptr && fwrite(base.data(), 4, base.size(), f) == base.size(), "cannot write %s", argv[a + 1]);
    fclose(f);
    printf("ok  %s: n=%lld nnz=%lld T=%lld, 3 interleavings bit-identical\n", argv[a], (long long)c.n, (long long)c.nnz,
           (long long)c.iterations);
  }
  printf("ALL OK\n");
  return 0;
}
