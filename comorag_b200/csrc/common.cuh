// Host-side helpers shared by the translation units of libcomorag_b200:
// error reporting for the C ABI, TMA tensor-map construction (driver entry
// point fetched through the runtime, so the library links only cudart),
// device queries and the dynamic shared-memory opt-in of a kernel.
#pragma once
#include <atomic>
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/comorag_b200.h"

namespace crag {

// Thread-local last-error text (the C ABI never throws; see crag_last_error()).
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);

#define CRAG_CUDA_OK(expr)                                                                     \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return ::crag::fail(CRAG_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                          __FILE__, __LINE__);                                                 \
  } while (0)

// 2-D bf16 row-major tensor [rows, cols] with `row_stride_bytes` between rows;
// box = box_rows x 64 columns (one 128-byte swizzle span), SWIZZLE_128B,
// out-of-bounds elements read as zero.
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols = 64);
// The same for int8 / uint8 elements: box = box_rows x 128 columns, again one 128-byte swizzle span.
int make_tmap_u8_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                    uint32_t box_rows, uint32_t box_cols = 128);

int sm_count();

// Raise Kernel's dynamic shared-memory limit to `bytes` once per device, not per launch.  The flags belong to the kernel
// itself (two instantiations of one kernel template do not share them) and are safe under concurrent host threads; a
// race at most repeats the idempotent attribute call.
template <auto Kernel>
int allow_dynamic_smem(size_t bytes) {
  static std::atomic<bool> done[64];
  int dev = 0;
  CRAG_CUDA_OK(cudaGetDevice(&dev));
  const bool tracked = dev >= 0 && dev < 64;
  if (tracked && done[dev].load(std::memory_order_acquire)) return CRAG_OK;
  CRAG_CUDA_OK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes)));
  if (tracked) done[dev].store(true, std::memory_order_release);
  return CRAG_OK;
}

// A workspace argument (workspace.cuh): CRAG_ERR_INVALID when null or not kWsAlign-aligned, CRAG_ERR_WORKSPACE when
// `bytes` < `need`; `who` heads the message.
int check_workspace(const char* who, const void* ws, size_t bytes, size_t need);

// quant.cu.  The address a kernel reads `p` through: device memory as is, page-locked host memory through its device
// mapping; anything else (pageable host memory) fails with CRAG_ERR_INVALID, `who` heading the message.
int device_readable(const void* p, const void** out, const char* who);
// quant.cu: the IVF rescore (quant_kernels.cuh) of one 32-query pass of the rescored IVF searches:
// ivf_rescore_topk_kernel up to 128 candidates, ivf_rescore_wide_kernel up to 2048
int launch_ivf_rescore(const void* rows, int64_t n_rows, int dim, int64_t row_stride, const void* queries, int nq,
                       const int64_t* cand, int n_cand, int k, const int32_t* list_tile_start, int nlist,
                       const float* coarse, int64_t* out_ids, float* out_scores, cudaStream_t stream);

}  // namespace crag
