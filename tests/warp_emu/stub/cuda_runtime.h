// Host stand-in for <cuda_runtime.h>, seen ONLY by tests/warp_emu (g++ -I tests/warp_emu/stub): it lets the pure-SIMT
// headers of the search kernels (csrc/topk.cuh, pool_floor.cuh, merge_kernels.cuh, rank_kernels.cuh) compile for the
// CPU, with thread indices, shared memory, barriers, warp intrinsics and the few memory-model operations they use
// mapped onto the fiber emulator of warp_emu.h.  Test infrastructure, not product code.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <thread>

#include "../warp_emu.h"

#define CRAG_EMULATED_PTX 1     // csrc headers leave their inline-PTX wrappers to this file when it is defined

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __shared__ static thread_local   // blocks of one emulator run one after the other; one emulator per OS thread

#define threadIdx (warp_emu::thread_idx())
#define blockIdx (warp_emu::block_idx())
#define blockDim (warp_emu::block_dim())
#define gridDim (warp_emu::grid_dim())

struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(16) float4 { float x, y, z, w; };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
struct alignas(16) int4 { int x, y, z, w; };
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }   // the GPU's rsqrt.approx is within 2 ulp of this

// csrc/encoder_simt.cuh: dynamic shared memory and its one named barrier
#define CRAG_DYNAMIC_SHARED(type, name) type* name = static_cast<type*>(warp_emu::dynamic_shared())
namespace crag {
static inline void bar_sync_group0_128() { warp_emu::named_barrier(1, 128); }
// csrc/select_warps.cuh: the select warps' named barriers
static inline void named_bar_sync(uint32_t id, uint32_t n) { warp_emu::named_barrier(int(id), int(n)); }
static inline bool named_bar_or(uint32_t id, uint32_t n, bool p) { return warp_emu::named_barrier_or(int(id), int(n), p); }
}  // namespace crag

static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline int __popc(uint32_t x) { return __builtin_popcount(x); }
static inline int __ffs(uint32_t x) { return __builtin_ffs((int)x); }

template <class T> static inline T __ldcg(const T* p) { return *p; }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcv(const T* p) {
  if (warp_emu::nap_us() && warp_emu::nap_armed()) {       // fault injection, see warp_emu::nap_us()
    warp_emu::nap_armed() = false;
    std::this_thread::sleep_for(std::chrono::microseconds(warp_emu::nap_us()));
  }
  return *static_cast<const volatile T*>(p);
}

// fibers of one block never run at the same time, so a read-modify-write is atomic among them
template <class T> static inline T atomicAdd(T* p, T v) { ++warp_emu::census().atomics; T old = *p; *p = old + v; return old; }
template <class T> static inline T atomicOr(T* p, T v) { T old = *p; *p = old | v; return old; }

static inline void __syncthreads() { warp_emu::sync_block(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { warp_emu::barrier(); }
static inline void __threadfence_system() { std::atomic_thread_fence(std::memory_order_seq_cst); }
static inline void __nanosleep(unsigned) {
  ++warp_emu::spin_count();
  std::this_thread::yield();      // another rank (OS thread) has to make progress
  warp_emu::yield_thread();       // and so may the other threads of this block
}

template <class T> static inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
  ++warp_emu::census().shuffles;
  return warp_emu::exchange(v, [&](int lane) { return lane ^ lane_mask; });
}
template <class T> static inline T __shfl_sync(unsigned, T v, int src) {
  ++warp_emu::census().shuffles;
  return warp_emu::exchange(v, [&](int) { return src & 31; });
}
static inline unsigned __ballot_sync(unsigned, int pred) {
  ++warp_emu::census().ballots;
  return warp_emu::reduce<unsigned>(pred ? (1u << warp_emu::lane()) : 0u, [](unsigned a, unsigned b) { return a | b; });
}
static inline unsigned __match_any_sync(unsigned, unsigned v) {
  const int me = warp_emu::lane();
  return warp_emu::gather(v, [&](const unsigned* all) {
    unsigned m = 0;
    for (int l = 0; l < 32; ++l) m |= (all[l] == all[me]) ? (1u << l) : 0u;
    return m;
  });
}
static inline int __reduce_add_sync(unsigned, int v) { ++warp_emu::census().reductions; return warp_emu::reduce<int>(v, [](int a, int b) { return a + b; }); }
static inline unsigned __reduce_add_sync(unsigned, unsigned v) { ++warp_emu::census().reductions; return warp_emu::reduce<unsigned>(v, [](unsigned a, unsigned b) { return a + b; }); }
static inline unsigned __reduce_min_sync(unsigned, unsigned v) { ++warp_emu::census().reductions; return warp_emu::reduce<unsigned>(v, [](unsigned a, unsigned b) { return a < b ? a : b; }); }
static inline unsigned __reduce_max_sync(unsigned, unsigned v) { ++warp_emu::census().reductions; return warp_emu::reduce<unsigned>(v, [](unsigned a, unsigned b) { return a > b ? a : b; }); }
static inline unsigned __reduce_or_sync(unsigned, unsigned v) { ++warp_emu::census().reductions; return warp_emu::reduce<unsigned>(v, [](unsigned a, unsigned b) { return a | b; }); }

// the inline-PTX wrappers of csrc/merge_kernels.cuh (st.release.sys / ld.acquire.sys / %globaltimer)
namespace crag {
static inline void st_release_sys_u64(uint64_t* p, uint64_t v) {
  reinterpret_cast<std::atomic<uint64_t>*>(p)->store(v, std::memory_order_release);
}
static inline uint64_t ld_acquire_sys_u64(const uint64_t* p) {
  return reinterpret_cast<const std::atomic<uint64_t>*>(p)->load(std::memory_order_acquire);
}
static inline uint64_t global_timer_ns() {
  return uint64_t(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count());
}
}  // namespace crag
