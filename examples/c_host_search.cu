// A host that uses libcomorag_b200 the way a non-Python caller would: CUDA runtime + the C ABI of
// include/comorag_b200.h, nothing else (no torch, no Python).  It is the smallest proof that the drop-in boundary
// really is plain pointers and sizes, and a way to time / check the search path on a box where importing a framework
// costs more than the measurement.
//
// What it replaces in the reference, per query block: ComoRAG.dense_passage_retrieval (ComoRAG.py:950-967) --
// np.dot(E, q.T) -> min_max_normalize -> np.argsort[::-1][:k] -- as ONE crag_search_topk call over a bf16 shard.
//
// Self-checking without an oracle: the shard is pseudo-random rows of norm ~1 (inner product with a unit query
// ~ N(0, 1/dim), so < 0.2 at dim 1024) with PLANTED rows  bf16(q * (1 - j/256)),  j = 0..127, for every query q at
// known, scattered positions.  Those score ~(1 - j/256) >= 0.5, strictly decreasing in j, so the exact answer is known
// in closed form for any k <= 128: rank j of query q is planted row (q, j), its score is the host-computed dot
// product, and max over the shard is the rank-0 score.
//
//   c_host_search                      default suite (the shapes DESIGN.md section 3 quotes), one JSON object per line
//   c_host_search ROWS DIM NQ K [REPS] one case
// Exit code 0 = every case had exact ids; 1 = a mismatch; 2 = a CUDA / library error.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "comorag_b200.h"

#define CUDA_OK(x)                                                                                   \
  do {                                                                                               \
    cudaError_t e_ = (x);                                                                            \
    if (e_ != cudaSuccess) {                                                                         \
      fprintf(stderr, "%s:%d: %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));          \
      exit(2);                                                                                       \
    }                                                                                                \
  } while (0)
#define CRAG_CALL(x)                                                                                 \
  do {                                                                                               \
    int rc_ = (x);                                                                                   \
    if (rc_ != CRAG_OK) {                                                                            \
      fprintf(stderr, "%s:%d: %s -> rc %d: %s\n", __FILE__, __LINE__, #x, rc_, crag_last_error());   \
      exit(2);                                                                                       \
    }                                                                                                \
  } while (0)

static const int kPlanted = 128;   // planted rows per query (= the library's largest k per pass)

// ---- bf16 <-> fp32 on the host (round to nearest even, as torch.Tensor.bfloat16() does)
static uint16_t f32_to_bf16(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  u += 0x7FFFu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static float bf16_to_f32(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// ---- shard generation on the device: uniform in [-a, a] with a = sqrt(3 / dim)  (variance 1 / dim, row norm ~ 1)
__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__global__ void fill_rows(uint16_t* rows, size_t n_elems, float amp, uint64_t seed) {
  // four bf16 per 64-bit hash, eight per thread and step: one 16-byte store
  const size_t stride = (size_t)gridDim.x * blockDim.x * 8;
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; i < n_elems; i += stride) {
    __align__(16) uint16_t v[8];
    for (int h = 0; h < 2; ++h) {
      const uint64_t r = mix64(seed ^ (i + 4 * h));
      for (int j = 0; j < 4; ++j) {
        const float u = (float)((r >> (16 * j)) & 0xFFFFu) * (2.0f / 65535.0f) - 1.0f;
        const float x = u * amp;
        uint32_t bits = __float_as_uint(x);
        bits += 0x7FFFu + ((bits >> 16) & 1u);
        v[4 * h + j] = (uint16_t)(bits >> 16);
      }
    }
    if (i + 8 <= n_elems) {
      *reinterpret_cast<uint4*>(rows + i) = *reinterpret_cast<const uint4*>(v);
    } else {
      for (int j = 0; j < 8 && i + j < n_elems; ++j) rows[i + j] = v[j];
    }
  }
}

static uint64_t host_rng_state = 0x1234567ull;
static float host_uniform(void) {   // xorshift64*, (-1, 1)
  host_rng_state ^= host_rng_state >> 12;
  host_rng_state ^= host_rng_state << 25;
  host_rng_state ^= host_rng_state >> 27;
  const uint64_t r = host_rng_state * 0x2545F4914F6CDD1Dull;
  return (float)((r >> 40) & 0xFFFFFFu) * (2.0f / 16777215.0f) - 1.0f;
}

static int cmp_float(const void* a, const void* b) {
  const float x = *(const float*)a, y = *(const float*)b;
  return (x > y) - (x < y);
}

// position of planted row (q, j): scattered over the whole shard, distinct for distinct (q, j)
static int64_t planted_row(int64_t rows, int nq, int q, int j) {
  const int64_t step = (rows - 64) / ((int64_t)nq * kPlanted);
  return 17 + ((int64_t)q * kPlanted + j) * step;
}

struct CaseResult {
  double us_median, us_min;
  int id_mismatches;
  double max_score_err, max_maxerr;
};

static CaseResult run_case(int64_t rows, int dim, int nq, int k, int reps, uint16_t* d_rows /* capacity >= rows * dim */) {
  CaseResult res;
  memset(&res, 0, sizeof res);
  if (rows < (int64_t)nq * kPlanted + 128 || k > kPlanted || nq > 32 || dim % 64) {
    fprintf(stderr, "case needs rows >= nq * 128 + 128, k <= 128, nq <= 32, dim %% 64 == 0\n");
    exit(2);
  }
  cudaStream_t st;
  CUDA_OK(cudaStreamCreate(&st));
  const size_t n_elems = (size_t)rows * dim;
  fill_rows<<<132 * 8, 256, 0, st>>>(d_rows, n_elems, sqrtf(3.0f / dim), 0xC0FFEEull + (uint64_t)rows);
  CUDA_OK(cudaGetLastError());

  // queries: random unit vectors, rounded to bf16; planted rows from the ROUNDED query values
  uint16_t* h_q = (uint16_t*)malloc((size_t)nq * dim * 2);
  uint16_t* h_plant = (uint16_t*)malloc((size_t)kPlanted * dim * 2);
  double* want_score = (double*)malloc((size_t)nq * kPlanted * sizeof(double));
  float* qf = (float*)malloc((size_t)dim * 4);
  host_rng_state = 0x1234567ull + (uint64_t)rows * 31 + (uint64_t)k;
  for (int q = 0; q < nq; ++q) {
    double n2 = 0;
    for (int i = 0; i < dim; ++i) { qf[i] = host_uniform(); n2 += (double)qf[i] * qf[i]; }
    const float inv = (float)(1.0 / sqrt(n2));
    for (int i = 0; i < dim; ++i) h_q[(size_t)q * dim + i] = f32_to_bf16(qf[i] * inv);
    for (int j = 0; j < kPlanted; ++j) {
      const float f = 1.0f - (float)j / 256.0f;
      double dot = 0;
      for (int i = 0; i < dim; ++i) {
        const float qv = bf16_to_f32(h_q[(size_t)q * dim + i]);
        const uint16_t pv = f32_to_bf16(qv * f);
        h_plant[(size_t)j * dim + i] = pv;
        dot += (double)qv * (double)bf16_to_f32(pv);
      }
      want_score[q * kPlanted + j] = dot;
      CUDA_OK(cudaMemcpyAsync(d_rows + (size_t)planted_row(rows, nq, q, j) * dim, h_plant + (size_t)j * dim,
                              (size_t)dim * 2, cudaMemcpyHostToDevice, st));
    }
    CUDA_OK(cudaStreamSynchronize(st));   // h_plant is reused by the next query
  }

  uint16_t* d_q;
  int64_t* d_ids;
  float *d_scores, *d_mm;
  void* d_ws;
  const size_t ws_bytes = crag_search_workspace_bytes(nq, k);
  CUDA_OK(cudaMalloc(&d_q, (size_t)nq * dim * 2));
  CUDA_OK(cudaMalloc(&d_ids, (size_t)nq * k * 8));
  CUDA_OK(cudaMalloc(&d_scores, (size_t)nq * k * 4));
  CUDA_OK(cudaMalloc(&d_mm, (size_t)nq * 2 * 4));
  CUDA_OK(cudaMalloc(&d_ws, ws_bytes));
  CUDA_OK(cudaMemcpyAsync(d_q, h_q, (size_t)nq * dim * 2, cudaMemcpyHostToDevice, st));

  // warm-up (tensor maps, function attributes), then `reps` timed calls, each bracketed by events on the launch stream
  for (int w = 0; w < 3; ++w)
    CRAG_CALL(crag_search_topk(d_rows, rows, dim, dim, 0, d_q, nq, k, d_ids, d_scores, d_mm, d_ws, ws_bytes, st));
  CUDA_OK(cudaStreamSynchronize(st));
  float* us = (float*)malloc((size_t)reps * 4);
  cudaEvent_t a, b;
  CUDA_OK(cudaEventCreate(&a));
  CUDA_OK(cudaEventCreate(&b));
  for (int r = 0; r < reps; ++r) {
    CUDA_OK(cudaEventRecord(a, st));
    CRAG_CALL(crag_search_topk(d_rows, rows, dim, dim, 0, d_q, nq, k, d_ids, d_scores, d_mm, d_ws, ws_bytes, st));
    CUDA_OK(cudaEventRecord(b, st));
    CUDA_OK(cudaEventSynchronize(b));
    float ms;
    CUDA_OK(cudaEventElapsedTime(&ms, a, b));
    us[r] = ms * 1000.0f;
  }
  qsort(us, (size_t)reps, 4, cmp_float);
  res.us_median = us[reps / 2];
  res.us_min = us[0];

  int64_t* h_ids = (int64_t*)malloc((size_t)nq * k * 8);
  float* h_scores = (float*)malloc((size_t)nq * k * 4);
  float* h_mm = (float*)malloc((size_t)nq * 2 * 4);
  CUDA_OK(cudaMemcpy(h_ids, d_ids, (size_t)nq * k * 8, cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(h_scores, d_scores, (size_t)nq * k * 4, cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(h_mm, d_mm, (size_t)nq * 2 * 4, cudaMemcpyDeviceToHost));
  for (int q = 0; q < nq; ++q) {
    for (int j = 0; j < k; ++j) {
      if (h_ids[q * k + j] != planted_row(rows, nq, q, j)) ++res.id_mismatches;
      const double e = fabs((double)h_scores[q * k + j] - want_score[q * kPlanted + j]);
      if (e > res.max_score_err) res.max_score_err = e;
    }
    const double em = fabs((double)h_mm[q * 2 + 1] - want_score[q * kPlanted]);
    if (em > res.max_maxerr) res.max_maxerr = em;
  }
  free(us); free(h_ids); free(h_scores); free(h_mm); free(h_q); free(h_plant); free(want_score); free(qf);
  CUDA_OK(cudaFree(d_q)); CUDA_OK(cudaFree(d_ids)); CUDA_OK(cudaFree(d_scores)); CUDA_OK(cudaFree(d_mm)); CUDA_OK(cudaFree(d_ws));
  CUDA_OK(cudaEventDestroy(a)); CUDA_OK(cudaEventDestroy(b));
  CUDA_OK(cudaStreamDestroy(st));
  return res;
}

static int report(int64_t rows, int dim, int nq, int k, int reps, const CaseResult& r) {
  const double bytes = (double)rows * dim * 2.0;
  const int ok = r.id_mismatches == 0 && r.max_score_err < 1e-3 && r.max_maxerr < 1e-3;
  printf("{\"rows\": %lld, \"dim\": %d, \"nq\": %d, \"k\": %d, \"reps\": %d, \"topk_call_us_median\": %.1f, "
         "\"topk_call_us_min\": %.1f, \"algorithmic_GBps\": %.1f, \"id_mismatches\": %d, \"max_score_err\": %.3g, "
         "\"max_of_minmax_err\": %.3g, \"ok\": %s}\n",
         (long long)rows, dim, nq, k, reps, r.us_median, r.us_min, bytes / r.us_median / 1e3, r.id_mismatches,
         r.max_score_err, r.max_maxerr, ok ? "true" : "false");
  fflush(stdout);
  return ok;
}

int main(int argc, char** argv) {
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) {
    fprintf(stderr, "c_host_search: no CUDA device (the library has no CPU path)\n");
    return 2;
  }
  CUDA_OK(cudaSetDevice(0));
  if (crag_version() < 1000) return 2;
  int all_ok = 1;
  if (argc >= 5) {
    const int64_t rows = atoll(argv[1]);
    const int dim = atoi(argv[2]), nq = atoi(argv[3]), k = atoi(argv[4]);
    const int reps = argc >= 6 ? atoi(argv[5]) : 15;
    uint16_t* d_rows;
    CUDA_OK(cudaMalloc(&d_rows, (size_t)rows * dim * 2));
    all_ok &= report(rows, dim, nq, k, reps, run_case(rows, dim, nq, k, reps, d_rows));
    CUDA_OK(cudaFree(d_rows));
    return all_ok ? 0 : 1;
  }
  // default suite: one rank's shard of the 8-GPU split (1.25M x 1024) and the one-GPU headline shape (10M x 1024)
  static const struct { int64_t rows; int k; int reps; } suite[] = {
      {1250000, 10, 25}, {1250000, 32, 25}, {1250000, 100, 25}, {1250000, 128, 15},
      {10000000, 10, 9}, {10000000, 100, 9},
  };
  const int dim = 1024, nq = 32;
  uint16_t* d_rows;
  CUDA_OK(cudaMalloc(&d_rows, (size_t)10000000 * dim * 2));
  for (size_t i = 0; i < sizeof suite / sizeof suite[0]; ++i)
    all_ok &= report(suite[i].rows, dim, nq, suite[i].k, suite[i].reps,
                     run_case(suite[i].rows, dim, nq, suite[i].k, suite[i].reps, d_rows));
  CUDA_OK(cudaFree(d_rows));
  return all_ok ? 0 : 1;
}
