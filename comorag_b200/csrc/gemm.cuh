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
};

// out[M,N] (bf16) = epi(A[M,K] (bf16) . W[N,K]^T (bf16) + bias[N] (fp32)); leading dims in elements.
int gemm_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, const float* bias, const void* residual,
              int64_t ldr, void* out, int64_t ldo, int M, int N, int K, int epi, cudaStream_t stream);

}  // namespace crag
