// Device workspaces.  An entry point that takes a workspace lays it out as regions in a fixed order, each starting on
// a kWsAlign boundary of a kWsAlign-aligned buffer.  One layout function per workspace runs a WsCursor over its
// regions: with a null base it sizes the workspace (crag_*_workspace_bytes), with the caller's buffer it hands out the
// region pointers, so the size and the carve cannot disagree.  Host code only, no CUDA headers: tests/warp_emu
// compiles the kernel headers that include it.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace crag {

constexpr size_t kWsAlign = 256;

inline size_t ws_round(size_t bytes) { return (bytes + kWsAlign - 1) & ~(kWsAlign - 1); }

struct WsCursor {
  uintptr_t base;     // 0: size only, every region comes back null
  size_t bytes;       // taken so far
  // `at`: where the regions start, after those of the layout this one extends
  explicit WsCursor(const void* ws, size_t at = 0) : base(reinterpret_cast<uintptr_t>(ws)), bytes(at) {}
  // the next region, of `count` T
  template <class T>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += ws_round(sizeof(T) * count);
    return p;
  }
};

}  // namespace crag
