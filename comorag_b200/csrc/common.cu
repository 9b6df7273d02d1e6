// Error plumbing, TMA tensor-map construction and device queries for the C ABI.
#include "common.cuh"
#include "workspace.cuh"

#include <stdarg.h>
#include <string.h>

#include <mutex>

namespace crag {

namespace {
thread_local char g_err[512] = {0};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}
}  // namespace

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

namespace {
int make_tmap_2d(CUtensorMap* out, CUtensorMapDataType type, const void* base, uint64_t rows, uint64_t cols,
                 uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(CRAG_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (driver too old?)");
  if (rows == 0 || cols == 0) return fail(CRAG_ERR_INVALID, "tensor map over an empty tensor");
  // The encode needs a current context.  A host thread whose first CUDA call this is (its tensors all came from the
  // allocator's cache) has none yet, and the encode fails with CUDA_ERROR_INVALID_CONTEXT: bind the primary context
  // of the thread's current device first, once per thread.
  thread_local bool bound = false;
  if (!bound) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaSetDevice(dev) != cudaSuccess)
      return fail(CRAG_ERR_CUDA, "no CUDA context for the tensor map: %s", cudaGetErrorString(cudaGetLastError()));
    bound = true;
  }
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {row_stride_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estride[2] = {1, 1};
  CUresult r = enc(out, type, 2, const_cast<void*>(base), gdim, gstride, box, estride,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(CRAG_ERR_CUDA, "cuTensorMapEncodeTiled failed (CUresult %d; rows=%llu cols=%llu stride=%llu box=%ux%u)",
                int(r), (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)row_stride_bytes,
                box_rows, box_cols);
  return CRAG_OK;
}
}  // namespace

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                      uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rows, cols, row_stride_bytes, box_rows, box_cols);
}

int make_tmap_u8_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                    uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rows, cols, row_stride_bytes, box_rows, box_cols);
}

int sm_count() {
  // cached per device; a handful of devices at most
  static int cached[64] = {0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess || dev < 0 || dev >= 64) {
    fail(CRAG_ERR_CUDA, "no usable CUDA device (%s)", e != cudaSuccess ? cudaGetErrorString(e) : "device ordinal out of range");
    return -1;
  }
  if (cached[dev] == 0) {
    int n = 0;
    e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) {
      fail(CRAG_ERR_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(e));
      return -1;
    }
    cached[dev] = n;
  }
  return cached[dev];
}

int check_workspace(const char* who, const void* ws, size_t bytes, size_t need) {
  if (!ws) return fail(CRAG_ERR_INVALID, "%s: null workspace pointer", who);
  if (reinterpret_cast<uintptr_t>(ws) % kWsAlign) return fail(CRAG_ERR_INVALID, "%s: workspace must be 256-byte aligned", who);
  if (bytes < need) return fail(CRAG_ERR_WORKSPACE, "%s: workspace %zu < %zu bytes", who, bytes, need);
  return CRAG_OK;
}

}  // namespace crag

extern "C" int crag_version(void) { return 1003; }
extern "C" const char* crag_last_error(void) { return crag::g_err; }
extern "C" int crag_sm_count(void) { return crag::sm_count(); }

// ---------------------------------------------------------------------------------------------------------------
// Growable device buffer: reserve virtual address space once, map physical memory as the corpus shard grows.
// The reference keeps its index as a Python list of rows it re-stacks on demand (embedding_store.py:96,147-157); a
// device shard that reallocates on growth needs old + new storage at once (a 20 GB shard: 50 GB transiently) and moves
// -- which invalidates every tensor map / captured graph that points at it.  With cuMemAddressReserve + cuMemMap the
// shard's address never changes and growth copies nothing.
namespace crag {
namespace {
struct VmemApi {
  CUresult (*reserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*addr_free)(CUdeviceptr, size_t) = nullptr;
  CUresult (*create)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*release)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*unmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*set_access)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*granularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  bool ok = false;
};

const VmemApi& vmem_api() {
  static VmemApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    auto get = [](const char* name, void** fn) {
      cudaDriverEntryPointQueryResult q;
      return cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess;
    };
    api.ok = get("cuMemAddressReserve", reinterpret_cast<void**>(&api.reserve)) &&
             get("cuMemAddressFree", reinterpret_cast<void**>(&api.addr_free)) &&
             get("cuMemCreate", reinterpret_cast<void**>(&api.create)) &&
             get("cuMemRelease", reinterpret_cast<void**>(&api.release)) &&
             get("cuMemMap", reinterpret_cast<void**>(&api.map)) &&
             get("cuMemUnmap", reinterpret_cast<void**>(&api.unmap)) &&
             get("cuMemSetAccess", reinterpret_cast<void**>(&api.set_access)) &&
             get("cuMemGetAllocationGranularity", reinterpret_cast<void**>(&api.granularity));
  });
  return api;
}

CUmemAllocationProp vmem_prop(int dev) {
  CUmemAllocationProp prop = {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = dev;
  return prop;
}
}  // namespace
}  // namespace crag

extern "C" int crag_vmem_reserve(size_t max_bytes, uint64_t* base_out, size_t* granularity_out) {
  using namespace crag;
  const VmemApi& api = vmem_api();
  if (!api.ok) return fail(CRAG_ERR_UNSUPPORTED, "virtual memory management entry points unavailable");
  if (!base_out || !granularity_out || max_bytes == 0) return fail(CRAG_ERR_INVALID, "crag_vmem_reserve: bad arguments");
  int dev = 0;
  CRAG_CUDA_OK(cudaGetDevice(&dev));
  CRAG_CUDA_OK(cudaFree(nullptr));   // make sure the primary context exists
  const CUmemAllocationProp prop = vmem_prop(dev);
  size_t gran = 0;
  CUresult r = api.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED);
  if (r != CUDA_SUCCESS || gran == 0) return fail(CRAG_ERR_CUDA, "cuMemGetAllocationGranularity failed (%d)", int(r));
  const size_t size = (max_bytes + gran - 1) / gran * gran;
  CUdeviceptr base = 0;
  r = api.reserve(&base, size, gran, 0, 0);
  if (r != CUDA_SUCCESS) return fail(CRAG_ERR_CUDA, "cuMemAddressReserve(%zu) failed (%d)", size, int(r));
  *base_out = uint64_t(base);
  *granularity_out = gran;
  return CRAG_OK;
}

extern "C" int crag_vmem_grow(uint64_t base, size_t mapped_bytes, size_t new_mapped_bytes) {
  using namespace crag;
  const VmemApi& api = vmem_api();
  if (!api.ok) return fail(CRAG_ERR_UNSUPPORTED, "virtual memory management entry points unavailable");
  if (new_mapped_bytes <= mapped_bytes) return CRAG_OK;
  int dev = 0;
  CRAG_CUDA_OK(cudaGetDevice(&dev));
  const CUmemAllocationProp prop = vmem_prop(dev);
  const size_t bytes = new_mapped_bytes - mapped_bytes;
  CUmemGenericAllocationHandle h;
  CUresult r = api.create(&h, bytes, &prop, 0);
  if (r != CUDA_SUCCESS) return fail(CRAG_ERR_CUDA, "cuMemCreate(%zu) failed (%d): out of device memory?", bytes, int(r));
  r = api.map(CUdeviceptr(base + mapped_bytes), bytes, 0, h, 0);
  if (r != CUDA_SUCCESS) {
    api.release(h);
    return fail(CRAG_ERR_CUDA, "cuMemMap failed (%d)", int(r));
  }
  api.release(h);   // the mapping keeps the memory alive until it is unmapped
  CUmemAccessDesc acc = {};
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = dev;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = api.set_access(CUdeviceptr(base + mapped_bytes), bytes, &acc, 1);
  if (r != CUDA_SUCCESS) return fail(CRAG_ERR_CUDA, "cuMemSetAccess failed (%d)", int(r));
  return CRAG_OK;
}

extern "C" int crag_vmem_release(uint64_t base, size_t mapped_bytes, size_t reserved_bytes) {
  using namespace crag;
  const VmemApi& api = vmem_api();
  if (!api.ok) return fail(CRAG_ERR_UNSUPPORTED, "virtual memory management entry points unavailable");
  if (mapped_bytes) {
    CUresult r = api.unmap(CUdeviceptr(base), mapped_bytes);
    if (r != CUDA_SUCCESS) return fail(CRAG_ERR_CUDA, "cuMemUnmap failed (%d)", int(r));
  }
  CUresult r = api.addr_free(CUdeviceptr(base), reserved_bytes);
  if (r != CUDA_SUCCESS) return fail(CRAG_ERR_CUDA, "cuMemAddressFree failed (%d)", int(r));
  return CRAG_OK;
}
