// warp_emu.h — run CUDA kernel SOURCE on the CPU: one FIBER (ucontext) per CUDA thread, the fibers of a
// block scheduled round-robin on the calling OS thread, blocks one after another.  Just enough of the
// CUDA surface for kernels written in the warp-synchronous style of this repo: full-mask warp
// collectives, __syncwarp, __syncthreads, global and shared atomics, static __shared__ arrays.
// Collectives are real rendezvous: a lane that skips one, or lanes that disagree about how many they
// execute, leave the block with runnable-but-blocked fibers only, which the scheduler reports as a
// deadlock (abort) — the CPU-side picture of a mis-synchronised kernel.
//
// A harness defines KVG_HOST_EMU, includes this file, then includes the kernel headers of csrc/ whole:
// kvg_common.cuh skips its inline-PTX block, whose functions are defined here, and everything else is
// compiled from the same text nvcc compiles.
//
// Test infrastructure only (tests/test_*_emu.py); never part of the product.
#pragma once
#include <cassert>
#include <ucontext.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <vector>

struct uint4 {
  uint32_t x, y, z, w;
};
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct uint2 {
  uint32_t x, y;
};
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct EmuDim3 {
  unsigned x = 1, y = 1, z = 1;
};
static EmuDim3 threadIdx, blockIdx, blockDim, gridDim;  // restored by the scheduler on every resume

struct EmuFiber {
  ucontext_t ctx;
  bool done = false;
};
struct EmuBlock {
  unsigned n_threads, n_warps;
  unsigned block_expected, block_arrived = 0, block_gen = 0;
  std::vector<unsigned> warp_expected, warp_arrived, warp_gen;
  std::vector<uint64_t> xchg;  // [warp][lane]
  std::vector<EmuFiber> fibers;
  ucontext_t sched;
  unsigned current = 0;
  bool progressed = false;
  explicit EmuBlock(unsigned n)
      : n_threads(n), n_warps((n + 31) / 32), block_expected(n), warp_expected(n_warps), warp_arrived(n_warps, 0),
        warp_gen(n_warps, 0), xchg(n_warps * 32), fibers(n) {
    for (unsigned w = 0; w < n_warps; w++) warp_expected[w] = (w + 1) * 32 <= n ? 32 : n - w * 32;
  }
};
static EmuBlock* emu_block = nullptr;
static inline void emu_yield() {
  EmuBlock* b = emu_block;
  swapcontext(&b->fibers[b->current].ctx, &b->sched);
}

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define __restrict__ __restrict

static inline uint32_t emu_lane() { return threadIdx.x & 31u; }
static inline uint32_t emu_warp() { return threadIdx.x >> 5; }
static inline void __threadfence() {}
static inline void __threadfence_system() {}
static inline long long clock64() { return 0; }
template <class T>
static inline T __ldg(const T* p) { return *p; }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline int __ffs(uint32_t v) { return __builtin_ffs((int)v); }
static inline int __clz(uint32_t v) { return v ? __builtin_clz(v) : 32; }
static inline uint32_t min(uint32_t a, uint32_t b) { return a < b ? a : b; }
static inline uint32_t max(uint32_t a, uint32_t b) { return a > b ? a : b; }

static inline void __syncthreads() {
  EmuBlock* b = emu_block;
  const unsigned gen = b->block_gen;
  b->progressed = true;
  if (++b->block_arrived == b->block_expected) {
    b->block_arrived = 0;
    b->block_gen++;
    return;
  }
  while (b->block_gen == gen) emu_yield();
}
static inline void __syncwarp() {
  EmuBlock* b = emu_block;
  const unsigned w = threadIdx.x >> 5, gen = b->warp_gen[w];
  b->progressed = true;
  if (++b->warp_arrived[w] == b->warp_expected[w]) {
    b->warp_arrived[w] = 0;
    b->warp_gen[w]++;
    return;
  }
  while (b->warp_gen[w] == gen) emu_yield();
}
// every lane publishes, everybody reads, everybody leaves: two rendezvous per collective
static inline uint64_t emu_exchange(uint64_t mine, uint32_t src_lane) {
  uint64_t* slot = &emu_block->xchg[emu_warp() * 32];
  slot[emu_lane()] = mine;
  __syncwarp();
  uint64_t got = slot[src_lane & 31u];
  __syncwarp();
  return got;
}
static inline uint32_t __shfl_sync(uint32_t, uint32_t v, uint32_t src) { return (uint32_t)emu_exchange(v, src); }
static inline uint32_t __shfl_up_sync(uint32_t, uint32_t v, uint32_t d) {
  uint32_t l = emu_lane();
  return (uint32_t)emu_exchange(v, l >= d ? l - d : l);
}
static inline uint32_t __shfl_xor_sync(uint32_t, uint32_t v, uint32_t m) { return (uint32_t)emu_exchange(v, emu_lane() ^ m); }
static inline uint32_t __ballot_sync(uint32_t, bool p) {
  uint64_t* slot = &emu_block->xchg[emu_warp() * 32];
  slot[emu_lane()] = p ? 1 : 0;
  __syncwarp();
  uint32_t m = 0;
  for (uint32_t l = 0; l < 32; l++) m |= (uint32_t)(slot[l] & 1) << l;
  __syncwarp();
  return m;
}
static inline bool __any_sync(uint32_t mask, bool p) { return __ballot_sync(mask, p) != 0; }
static inline uint32_t __match_any_sync(uint32_t, uint32_t v) {
  uint64_t* slot = &emu_block->xchg[emu_warp() * 32];
  slot[emu_lane()] = v;
  __syncwarp();
  uint32_t m = 0;
  for (uint32_t l = 0; l < 32; l++) m |= (uint32_t)(slot[l] == v) << l;
  __syncwarp();
  return m;
}

// full-warp reductions (REDUX on the GPU), on top of the emulated shuffles
static inline uint32_t __reduce_add_sync(uint32_t, uint32_t v) {
  for (uint32_t o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
static inline uint32_t __reduce_min_sync(uint32_t, uint32_t v) {
  for (uint32_t o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
static inline uint32_t __reduce_max_sync(uint32_t, uint32_t v) {
  for (uint32_t o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// byte n of the result is byte (s >> 4n) & 7 of the eight bytes {y:x}
static inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) {
  const uint64_t v = ((uint64_t)y << 32) | x;
  uint32_t r = 0;
  for (int n = 0; n < 4; n++) r |= (uint32_t)((v >> (8 * ((s >> (4 * n)) & 7u))) & 0xffu) << (8 * n);
  return r;
}

static inline uint32_t atomicAdd(uint32_t* p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline uint32_t atomicOr(uint32_t* p, uint32_t v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline uint32_t atomicExch(uint32_t* p, uint32_t v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
static inline uint32_t atomicMax(uint32_t* p, uint32_t v) {
  uint32_t old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v > old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
  }
  return old;
}
static inline uint32_t atomicMin(uint32_t* p, uint32_t v) {
  uint32_t old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
  }
  return old;
}
static inline uint32_t atomicCAS(uint32_t* p, uint32_t cmp, uint32_t v) {
  __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return cmp;  // the old value either way
}
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return cmp;  // the old value either way
}
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  unsigned long long old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
  }
  return old;
}

// ---- the hardware layer: what kvg_common.cuh defines in inline PTX under #ifndef KVG_HOST_EMU ----------
static inline uint32_t lanemask_lt() { return (1u << emu_lane()) - 1u; }
static inline void pdl_enter() {}
static inline uint4 ld_stream(const uint4* p) { return *p; }
static inline void st_stream(uint4* p, const uint4& v) { *p = v; }
static inline uint64_t ld_relaxed_u64(const uint64_t* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
static inline void st_relaxed_u64(uint64_t* p, uint64_t v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
static inline void st_relaxed_u32(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
static inline uint4 ld_volatile_v4(const uint4* p) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p);
  return uint4{__atomic_load_n(w, __ATOMIC_RELAXED), __atomic_load_n(w + 1, __ATOMIC_RELAXED),
               __atomic_load_n(w + 2, __ATOMIC_RELAXED), __atomic_load_n(w + 3, __ATOMIC_RELAXED)};
}

// mbarrier + TMA 1-D bulk copy as used by the per-warp text ring of k_pciids_scan and the span re-reads of
// k_pciids_resolve_finalize (kvg_parse_k1.cuh): the copy completes at issue time, the barrier word counts
// completed phases, a wait on parity p returns once phase p has completed — the same observable protocol,
// minus the asynchrony
// (barrier word here: low half = completed phases, high half = bytes still expected by the current phase;
// one arriving thread per phase, which is how every kernel of this library uses its barriers)
static inline void mbar_init(uint64_t* bar, uint32_t) { *bar = 0; }
static inline void mbar_fence_init() {}
static inline void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) { *bar += (uint64_t)bytes << 32; }
static inline void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  memcpy(smem_dst, gmem_src, bytes);
  assert((*bar >> 32) >= bytes && "bulk copy without a matching expect_tx");
  *bar -= (uint64_t)bytes << 32;
  if ((*bar >> 32) == 0) (*bar)++;  // the phase's last byte has landed
  emu_block->progressed = true;
}
static inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (((*bar) & 1u) == parity) emu_yield();
}

// kernel<<<grid, block>>>(args)
static std::function<void()> emu_entry;
static void emu_trampoline() {
  EmuBlock* b = emu_block;
  const unsigned t = b->current;
  emu_entry();
  // the thread leaves the kernel: later rendezvous of its warp / block no longer wait for it
  b = emu_block;
  b->fibers[t].done = true;
  b->progressed = true;
  const unsigned w = t >> 5;
  if (--b->warp_expected[w] > 0 && b->warp_arrived[w] == b->warp_expected[w]) {
    b->warp_arrived[w] = 0;
    b->warp_gen[w]++;
  }
  if (--b->block_expected > 0 && b->block_arrived == b->block_expected) {
    b->block_arrived = 0;
    b->block_gen++;
  }
  swapcontext(&b->fibers[t].ctx, &b->sched);
}
template <class... KArgs, class... Args>
static void emu_launch(void (*kernel)(KArgs...), dim3 grid2, unsigned block, Args... args) {
  constexpr size_t STACK = 256 << 10;
  emu_entry = [=] { kernel(args...); };
  // fiber stacks are allocated once per process and reused by every block of every launch
  static std::vector<std::unique_ptr<char[]>> stacks;
  while (stacks.size() < block) stacks.emplace_back(new char[STACK]);
  for (unsigned by = 0; by < grid2.y; by++)
    for (unsigned bx = 0; bx < grid2.x; bx++) {
      EmuBlock blk(block);
      emu_block = &blk;
      for (unsigned t = 0; t < block; t++) {
        EmuFiber& f = blk.fibers[t];
        getcontext(&f.ctx);
        f.ctx.uc_stack.ss_sp = stacks[t].get();
        f.ctx.uc_stack.ss_size = STACK;
        f.ctx.uc_link = &blk.sched;
        makecontext(&f.ctx, emu_trampoline, 0);
      }
      for (unsigned live = block; live;) {
        blk.progressed = false;
        live = 0;
        for (unsigned t = 0; t < block; t++) {
          if (blk.fibers[t].done) continue;
          blk.current = t;
          threadIdx.x = t;
          blockIdx.x = bx;
          blockIdx.y = by;
          blockDim.x = block;
          gridDim.x = grid2.x;
          gridDim.y = grid2.y;
          swapcontext(&blk.sched, &blk.fibers[t].ctx);
          live += !blk.fibers[t].done;
        }
        if (live && !blk.progressed) {
          fprintf(stderr, "warp_emu: deadlock in block (%u,%u): %u threads blocked at a rendezvous that cannot complete\n",
                  bx, by, live);
          abort();
        }
      }
    }
  emu_block = nullptr;
}
