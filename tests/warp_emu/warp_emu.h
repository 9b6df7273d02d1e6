// CUDA thread blocks on the CPU, for the pure-SIMT parts of the search kernels.  Every CUDA thread of one block is a
// fiber (its own stack, switched in user space); fibers run one at a time and switch only at synchronisation points, so plain arrays behave like
// shared memory between barriers:
//   * a warp collective (shuffle, ballot, reduction, match, __syncwarp) is a barrier of the 32 lanes of one warp at
//     which values are handed over through a slot array;
//   * __syncthreads() is a barrier of the block's live threads (threads that returned no longer count, as on the GPU);
//   * a kernel "launch" runs its blocks one after the other (blockIdx 0, 1, ...).
// All state is thread_local: a test that needs several blocks to make progress TOGETHER (the cross-rank exchange
// kernel: block q of every rank waits for block q of every other rank) runs one OS thread per rank, each with its own
// emulator, and real atomics between them (stub/cuda_runtime.h).  A collective that can never complete -- lanes
// waiting for a lane that already returned -- is reported as a deadlock instead of hanging the test.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <algorithm>
#include <functional>
#include <memory>
#include <vector>

namespace warp_emu {

constexpr int kLanes = 32;
constexpr size_t kStackBytes = 512 << 10;

// Context switch between fibers.  x86-64: a dozen instructions that swap the callee-saved registers and the stack
// pointer (glibc's swapcontext makes two sigprocmask system calls per switch, and the kernels below switch millions of
// times); elsewhere: ucontext.
#if defined(__x86_64__) && !defined(WARP_EMU_USE_UCONTEXT)
#define WARP_EMU_FAST_SWITCH 1
extern "C" void warp_emu_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.weak warp_emu_switch
.type warp_emu_switch,@function
warp_emu_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size warp_emu_switch,.-warp_emu_switch
)");
#endif

struct Fiber {
#ifdef WARP_EMU_FAST_SWITCH
  void* sp = nullptr;
#else
  ucontext_t ctx;
#endif
  char* stack = nullptr;
  bool done = false;
};

struct WarpState {
  int live = 0, arrived = 0;
  uint64_t gen = 0;
  uint64_t slot[kLanes];
};

struct Block {
#ifdef WARP_EMU_FAST_SWITCH
  void* main_sp = nullptr;
#else
  ucontext_t main;
#endif
  std::vector<Fiber> fibers;
  std::vector<WarpState> warps;
  int n_threads = 0, live = 0;
  int bar_arrived = 0;
  uint64_t bar_gen = 0;
  int named_arrived[16] = {0};   // bar.sync <id>, <count>: barriers over a fixed number of threads
  uint64_t named_gen[16] = {0};
  bool named_or_acc[16] = {false}, named_or_result[16] = {false};
  std::vector<uint8_t> dyn_smem;  // the launch's dynamic shared memory (garbage-filled: CUDA does not zero it)
  uint64_t progress = 0;        // bumps whenever any barrier releases or a thread exits (deadlock detection)
  int stuck_sweeps = 0;
  uint64_t spinning_sweeps = 0;
  int cur = 0;
  unsigned block_idx = 0, grid_dim = 1;
  std::function<void()> body;
};

// How often each kind of warp-level operation ran on this OS thread (every lane counts its own call): lets a tool say
// what the select warps spend their instructions on (tests/warp_emu/select_census.cpp).
struct Census {
  uint64_t shuffles = 0, reductions = 0, ballots = 0, named_barriers = 0, atomics = 0;
};
inline Census& census() {
  static thread_local Census c;
  return c;
}

// bumped by the __nanosleep stand-in: a thread that sleeps is waiting for memory ANOTHER OS thread will write
inline uint64_t& spin_count() {
  static thread_local uint64_t n = 0;
  return n;
}

// Fault injection for protocol tests: when nap_us() is set on an OS thread, the FIRST volatile load (__ldcv) of every
// block it runs sleeps that long -- in the exchange kernel that is the moment a rank starts reading the records its
// peers pushed, i.e. the window in which a peer that ran ahead must not be able to overwrite them.
inline int& nap_us() {
  static thread_local int us = 0;
  return us;
}
inline bool& nap_armed() {
  static thread_local bool armed = false;
  return armed;
}

inline Block*& current() {
  static thread_local Block* b = nullptr;
  return b;
}

struct Dim3 { unsigned x, y, z; };
inline Dim3 thread_idx() { return Dim3{unsigned(current()->cur), 0u, 0u}; }
inline Dim3 block_idx() { return Dim3{current()->block_idx, 0u, 0u}; }
inline Dim3 block_dim() { return Dim3{unsigned(current()->n_threads), 1u, 1u}; }
inline Dim3 grid_dim() { return Dim3{current()->grid_dim, 1u, 1u}; }
inline int lane() { return current()->cur & (kLanes - 1); }

inline void yield_thread() {
  Block* b = current();
#ifdef WARP_EMU_FAST_SWITCH
  warp_emu_switch(&b->fibers[b->cur].sp, b->main_sp);
#else
  swapcontext(&b->fibers[b->cur].ctx, &b->main);
#endif
}

inline void barrier() {            // the 32 lanes of the calling thread's warp
  Block* b = current();
  WarpState& w = b->warps[b->cur / kLanes];
  const uint64_t my = w.gen;
  if (++w.arrived >= w.live) {
    w.arrived = 0;
    ++w.gen;
    ++b->progress;
  }
  while (w.gen == my) yield_thread();
}

inline void sync_block() {         // __syncthreads()
  Block* b = current();
  const uint64_t my = b->bar_gen;
  if (++b->bar_arrived >= b->live) {
    b->bar_arrived = 0;
    ++b->bar_gen;
    ++b->progress;
  }
  while (b->bar_gen == my) yield_thread();
}

inline void named_barrier(int id, int count) {     // bar.sync id, count
  Block* b = current();
  ++census().named_barriers;
  const uint64_t my = b->named_gen[id];
  if (++b->named_arrived[id] >= count) {
    b->named_arrived[id] = 0;
    ++b->named_gen[id];
    ++b->progress;
  }
  while (b->named_gen[id] == my) yield_thread();
}

// barrier.cta.red.or: named barrier whose threads also learn the OR of everybody's predicate
inline bool named_barrier_or(int id, int count, bool pred) {
  Block* b = current();
  ++census().named_barriers;
  const uint64_t my = b->named_gen[id];
  b->named_or_acc[id] = b->named_or_acc[id] || pred;
  if (++b->named_arrived[id] >= count) {
    b->named_or_result[id] = b->named_or_acc[id];
    b->named_or_acc[id] = false;
    b->named_arrived[id] = 0;
    ++b->named_gen[id];
    ++b->progress;
  }
  while (b->named_gen[id] == my) yield_thread();
  return b->named_or_result[id];   // stable until every participant has left: the next release needs all of them again
}

inline void* dynamic_shared() { return current()->dyn_smem.data(); }

// every lane deposits v; lane l receives the value of lane src_of(l)
template <class T, class F>
inline T exchange(T v, F src_of) {
  static_assert(sizeof(T) <= 8, "exchange moves at most 64 bits");
  Block* b = current();
  WarpState& w = b->warps[b->cur / kLanes];
  const int me = b->cur & (kLanes - 1);
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  w.slot[me] = bits;
  barrier();
  const uint64_t got = w.slot[src_of(me) & (kLanes - 1)];
  barrier();                       // nobody overwrites a slot before every lane has read
  T r;
  memcpy(&r, &got, sizeof(T));
  return r;
}

// every lane receives f(all 32 deposited values)
template <class T, class F>
inline auto gather(T v, F f) -> decltype(f(static_cast<const T*>(nullptr))) {
  static_assert(sizeof(T) <= 8, "gather moves at most 64 bits");
  Block* b = current();
  WarpState& w = b->warps[b->cur / kLanes];
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  w.slot[b->cur & (kLanes - 1)] = bits;
  barrier();
  T all[kLanes];
  for (int l = 0; l < kLanes; ++l) memcpy(&all[l], &w.slot[l], sizeof(T));
  auto r = f(static_cast<const T*>(all));
  barrier();
  return r;
}

template <class T, class F>
inline T reduce(T v, F op) {
  return gather(v, [&](const T* all) {
    T acc = all[0];
    for (int l = 1; l < kLanes; ++l) acc = op(acc, all[l]);
    return acc;
  });
}

inline void trampoline() {
  Block* b = current();
  b->body();
  Fiber& f = b->fibers[b->cur];
  f.done = true;
  // a thread that returns stops counting towards the barriers it might have been expected at
  --b->live;
  WarpState& w = b->warps[b->cur / kLanes];
  --w.live;
  ++b->progress;
  if (w.arrived > 0 && w.arrived >= w.live) { w.arrived = 0; ++w.gen; }
  if (b->bar_arrived > 0 && b->bar_arrived >= b->live) { b->bar_arrived = 0; ++b->bar_gen; }
#ifdef WARP_EMU_FAST_SWITCH
  for (;;) yield_thread();       // a finished fiber has no frame to return to; the scheduler never resumes it
#endif
}

// ---- a block's life: make_block(), sweep() until nothing is left alive, destroy_block()
inline Block* make_block(int n_threads, unsigned block_index, unsigned grid, const std::function<void()>& body,
                         size_t dynamic_smem_bytes, size_t stack_bytes) {
  if (n_threads % kLanes != 0) { fprintf(stderr, "warp_emu: block size must be a multiple of 32\n"); abort(); }
  Block* b = new Block;
  b->body = body;
  b->dyn_smem.assign(dynamic_smem_bytes + 16, 0xCD);
  b->n_threads = b->live = n_threads;
  b->block_idx = block_index;
  b->grid_dim = grid;
  b->fibers.resize(n_threads);
  b->warps.resize(n_threads / kLanes);
  for (auto& w : b->warps) w.live = kLanes;
  for (int t = 0; t < n_threads; ++t) {
    Fiber& f = b->fibers[t];
    f.stack = static_cast<char*>(malloc(stack_bytes));
#ifdef WARP_EMU_FAST_SWITCH
    // initial frame: six callee-saved registers, then the entry point as the address `ret` jumps to, then a dummy
    // return address so the entry function sees the stack alignment of an ordinary call
    uintptr_t top = (reinterpret_cast<uintptr_t>(f.stack) + stack_bytes) & ~uintptr_t(15);
    void** frame = reinterpret_cast<void**>(top) - 8;
    for (int i = 0; i < 6; ++i) frame[i] = nullptr;
    frame[6] = reinterpret_cast<void*>(&trampoline);
    frame[7] = nullptr;
    f.sp = frame;
#else
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack;
    f.ctx.uc_stack.ss_size = stack_bytes;
    f.ctx.uc_link = &b->main;
    makecontext(&f.ctx, reinterpret_cast<void (*)()>(trampoline), 0);
#endif
  }
  return b;
}

inline void destroy_block(Block* b) {
  for (auto& f : b->fibers) free(f.stack);
  delete b;
}

// every live thread of the block runs up to its next synchronisation point; false once the block has finished
inline bool sweep(Block* b) {
  Block* outer = current();
  current() = b;
  const uint64_t before = b->progress;
  const uint64_t spins_before = spin_count();
  const int arrived_before = b->bar_arrived;
  int warp_arrived_before = 0;
  for (auto& w : b->warps) warp_arrived_before += w.arrived;
  for (int i = 0; i < 16; ++i) warp_arrived_before += b->named_arrived[i];
  for (int t = 0; t < b->n_threads; ++t) {
    if (b->fibers[t].done) continue;
    b->cur = t;
#ifdef WARP_EMU_FAST_SWITCH
    warp_emu_switch(&b->main_sp, b->fibers[t].sp);
#else
    swapcontext(&b->main, &b->fibers[t].ctx);
#endif
  }
  int warp_arrived_after = 0;
  for (auto& w : b->warps) warp_arrived_after += w.arrived;
  for (int i = 0; i < 16; ++i) warp_arrived_after += b->named_arrived[i];
  if (b->progress == before && b->bar_arrived == arrived_before && warp_arrived_after == warp_arrived_before && b->live > 0) {
    // nothing moved in a whole sweep.  Threads sleeping in a spin-wait on memory another OS thread will write (the
    // exchange kernel's flag wait) are legitimate and get a long leash; anything else is a lost collective.
    const bool spinning = spin_count() != spins_before;
    if (spinning ? ++b->spinning_sweeps > (uint64_t(1) << 24) : ++b->stuck_sweeps > 4) {
      fprintf(stderr, "warp_emu: deadlock in block %u -- %d live threads, %d at __syncthreads, %d at warp collectives\n",
              b->block_idx, b->live, b->bar_arrived, warp_arrived_after);
      abort();
    }
  } else {
    b->stuck_sweeps = 0;
  }
  current() = outer;
  return b->live > 0;
}

inline void run_block(int n_threads, unsigned block_index, unsigned grid, const std::function<void()>& body,
                      size_t dynamic_smem_bytes = 0) {
  Block* b = make_block(n_threads, block_index, grid, body, dynamic_smem_bytes, kStackBytes);
  nap_armed() = true;
  while (sweep(b)) {}
  destroy_block(b);
}

// kernel<<<grid, block>>> with all blocks RESIDENT TOGETHER (a persistent kernel: one block per SM): the blocks advance
// in turns, in an order drawn afresh from `seed` every round and by a random number of steps each, so that what one
// block publishes in global memory reaches the others at arbitrary points of their own progress.  Block-local storage
// must come from dynamic shared memory (each block has its own); `static` storage would be shared by all of them.
inline void launch_concurrent(unsigned grid, int block, const std::function<void()>& kernel_call, size_t dynamic_smem_bytes,
                              uint64_t seed, size_t stack_bytes = 96 << 10) {
  std::vector<Block*> blocks(grid);
  for (unsigned i = 0; i < grid; ++i) blocks[i] = make_block(block, i, grid, kernel_call, dynamic_smem_bytes, stack_bytes);
  uint64_t x = seed * 0x9E3779B97F4A7C15ull + 1;
  auto next = [&]() { x ^= x >> 12; x ^= x << 25; x ^= x >> 27; return x * 0x2545F4914F6CDD1Dull; };
  std::vector<unsigned> alive(grid);
  for (unsigned i = 0; i < grid; ++i) alive[i] = i;
  while (!alive.empty()) {
    for (size_t i = alive.size(); i > 1; --i) std::swap(alive[i - 1], alive[next() % i]);
    for (size_t i = 0; i < alive.size();) {
      bool more = true;
      for (int steps = 1 + int(next() % 3); steps > 0 && more; --steps) more = sweep(blocks[alive[i]]);
      if (!more) { alive[i] = alive.back(); alive.pop_back(); } else { ++i; }
    }
  }
  for (Block* b : blocks) destroy_block(b);
}

// kernel<<<grid, block>>>: blocks run one after the other
// A host stand-in for a device workspace: `bytes` bytes from an `align` boundary, every byte `poison` (0xFF bytes
// are NaN), so a kernel that reads what it did not write sees garbage.
struct Workspace {
  std::vector<uint8_t> mem;
  uint8_t* base;
  Workspace(size_t bytes, size_t align, uint8_t poison) : mem(bytes + align, poison) {
    void* p = mem.data();
    size_t space = mem.size();
    base = static_cast<uint8_t*>(std::align(align, bytes, p, space));
  }
};

inline void launch(unsigned grid, int block, const std::function<void()>& kernel_call, size_t dynamic_smem_bytes = 0) {
  for (unsigned bidx = 0; bidx < grid; ++bidx) run_block(block, bidx, grid, kernel_call, dynamic_smem_bytes);
}

// one warp, body(lane): what the selector-primitive tests use
inline void run_warp(const std::function<void(int)>& body) {
  run_block(kLanes, 0, 1, [&]() { body(lane()); });
}

}  // namespace warp_emu
