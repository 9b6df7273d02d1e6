// Internal interface of the wgmma GEMM (gemm.cu), used by the encoder driver.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/comorag_b200.h"

namespace crag {

enum : int {
  GEMM_EPI_BIAS = CRAG_GEMM_BIAS,
  GEMM_EPI_BIAS_GELU = CRAG_GEMM_BIAS_GELU,
  GEMM_EPI_BIAS_RESIDUAL = CRAG_GEMM_BIAS_RESIDUAL,
  GEMM_EPI_SCORES_F32 = 3,   // internal (gemm_scores_f32): crag_gemm_bf16 does not accept it
};

// out[M,N] (bf16) = epi(A[M,K] (bf16) . W[N,K]^T (bf16) + bias[N] (fp32)); leading dims in elements.
int gemm_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, const float* bias, const void* residual,
              int64_t ldr, void* out, int64_t ldo, int M, int N, int K, int epi, cudaStream_t stream);

// Score block of crag_knn_topk: out[m, n] (fp32, leading dimension ldo, even) = A[m, :] . W[n, :] with no bias, for
// any M, N >= 1 (K a multiple of 64).  A = queries, W = corpus rows.
int gemm_scores_f32(const void* a, int64_t lda, const void* w, int64_t ldw, float* out, int64_t ldo, int M, int N,
                    int K, cudaStream_t stream);

}  // namespace crag
