// kvg_common.cuh — device-side building blocks shared by every kernel of libkvgpu.so (sm_90a).
//
//   * streaming global loads/stores (ld.global.nc.L1::no_allocate / st.global.L1::no_allocate)
//   * mbarrier + 1-D TMA bulk copy (cp.async.bulk ... mbarrier::complete_tx::bytes -> SASS UBLKCP)
//   * warp / block scans
//   * epoch-tagged decoupled look-back (single-pass chained scan) used by the stable compactions
//     and by the vendor-context carry of the pci.ids parser
#pragma once
#include <stdint.h>

#define KVG_BLOCK 256
#define KVG_WARPS (KVG_BLOCK / 32)
#define KVG_FULL 0xffffffffu

// ---- the hardware layer -------------------------------------------------------------------------
// The inline PTX of the library lives in this one block.  The CPU emulator (tools/emu/warp_emu.h) defines
// KVG_HOST_EMU and supplies the same functions; everything outside the block, and every kernel header, is
// compiled from the same text for the GPU and for the emulator.
#ifndef KVG_HOST_EMU
#include <cuda_runtime.h>

namespace kvg {

__device__ __forceinline__ uint32_t lanemask_lt() {
  uint32_t m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// ---- streaming memory access --------------------------------------------------------------------
// Programmatic dependent launch (sm_90+): every kernel on the scan path opens with pdl_enter().
// launch_dependents lets the NEXT kernel of the stream be scheduled while this one still runs (its CTAs
// park in griddepcontrol.wait); wait returns once the PREVIOUS kernel has completed and its writes are
// visible.  Without the launch attribute both instructions are no-ops, so plain launches stay correct.
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// four words another CTA may be writing right now: never from L1, each word read whole
__device__ __forceinline__ uint4 ld_volatile_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}

// ---- mbarrier + TMA 1-D bulk copy ---------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// global -> shared bulk copy through the TMA unit; bytes % 16 == 0, both addresses 16-B aligned
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

}  // namespace kvg
#endif  // KVG_HOST_EMU

namespace kvg {

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t warp_id() { return threadIdx.x >> 5; }

// ---- scans --------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t warp_incl_sum(uint32_t v) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(KVG_FULL, v, d);
    if (lane_id() >= (uint32_t)d) v += t;
  }
  return v;
}
__device__ __forceinline__ uint32_t warp_incl_max(uint32_t v) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(KVG_FULL, v, d);
    if (lane_id() >= (uint32_t)d) v = max(v, t);
  }
  return v;
}
// full-warp reductions: one REDUX instruction each (sm_80+)
__device__ __forceinline__ uint32_t warp_sum(uint32_t v) { return __reduce_add_sync(KVG_FULL, v); }
__device__ __forceinline__ uint32_t warp_max(uint32_t v) { return __reduce_max_sync(KVG_FULL, v); }
__device__ __forceinline__ uint32_t warp_min(uint32_t v) { return __reduce_min_sync(KVG_FULL, v); }

// Block-wide exclusive sum over KVG_BLOCK threads; *total receives the block sum.
// `scratch` is KVG_WARPS+1 words of shared memory; contains two __syncthreads().
__device__ __forceinline__ uint32_t block_excl_sum(uint32_t v, uint32_t* scratch, uint32_t* total) {
  uint32_t incl = warp_incl_sum(v);
  if (lane_id() == 31) scratch[warp_id()] = incl;
  __syncthreads();
  if (warp_id() == 0) {
    uint32_t w = lane_id() < KVG_WARPS ? scratch[lane_id()] : 0;
    uint32_t wi = warp_incl_sum(w);
    if (lane_id() < KVG_WARPS) scratch[lane_id()] = wi - w;
    if (lane_id() == KVG_WARPS - 1) scratch[KVG_WARPS] = wi;
  }
  __syncthreads();
  uint32_t r = scratch[warp_id()] + incl - v;
  *total = scratch[KVG_WARPS];
  return r;
}
// ---- decoupled look-back ------------------------------------------------------------------------
// One 64-bit word per tile: [63:34] launch epoch, [33:32] status, [31:0] value.  The epoch makes a
// stale word from an earlier launch read as "not ready", so the array never needs clearing.
enum : uint32_t { LB_INVALID = 0, LB_AGGREGATE = 1, LB_INCLUSIVE = 2 };
__device__ __forceinline__ uint64_t lb_pack(uint32_t epoch, uint32_t status, uint32_t value) {
  return ((uint64_t)(epoch & 0x3fffffffu) << 34) | ((uint64_t)status << 32) | value;
}
__device__ __forceinline__ uint32_t lb_status(uint64_t w, uint32_t epoch) {
  return ((uint32_t)(w >> 34) == (epoch & 0x3fffffffu)) ? (uint32_t)((w >> 32) & 3) : LB_INVALID;
}

// Sum look-back, executed by one full warp.  Publishes this tile's aggregate, walks predecessors
// and returns the exclusive prefix (valid in every lane); publishes the inclusive.
// The walk reads LB_WIDE*32 predecessor states per step with INDEPENDENT loads: with ~1000 tiles
// in flight the nearest inclusive prefix is typically hundreds of tiles back, and a 32-wide
// window would turn that into a chain of ~15 dependent L2 round trips per tile.
constexpr int LB_WIDE = 1;  // measured: 8-wide windows were slower (more polling traffic), 1 = classic
__device__ __forceinline__ uint32_t lookback_sum(uint64_t* state, uint32_t tile, uint32_t aggregate,
                                                 uint32_t epoch) {
  const uint32_t lane = lane_id();
  if (tile == 0) {
    if (lane == 0) st_relaxed_u64(&state[0], lb_pack(epoch, LB_INCLUSIVE, aggregate));
    return 0;
  }
  if (lane == 0) st_relaxed_u64(&state[tile], lb_pack(epoch, LB_AGGREGATE, aggregate));
  uint32_t excl = 0;
  int look = (int)tile - 1;
  for (;;) {
    uint64_t w[LB_WIDE];
#pragma unroll
    for (int k = 0; k < LB_WIDE; k++) {
      int idx = look - (int)lane - 32 * k;
      w[k] = idx >= 0 ? ld_relaxed_u64(&state[idx]) : lb_pack(epoch, LB_INCLUSIVE, 0);
    }
    bool done = false;
#pragma unroll
    for (int k = 0; k < LB_WIDE; k++) {
      uint32_t st = lb_status(w[k], epoch);
      uint32_t incl_mask = __ballot_sync(KVG_FULL, st == LB_INCLUSIVE);
      uint32_t inv_mask = __ballot_sync(KVG_FULL, st == LB_INVALID);
      uint32_t first = incl_mask ? (uint32_t)__ffs(incl_mask) - 1 : 32;
      uint32_t need = first >= 31 ? KVG_FULL : ((2u << first) - 1);  // lanes 0..first
      if (inv_mask & need) break;  // a needed predecessor is not published yet: reload from here
      excl += warp_sum(lane <= first ? (uint32_t)w[k] : 0u);
      if (first < 32) {
        done = true;
        break;
      }
      look -= 32;
    }
    if (done) break;
  }
  if (lane == 0) st_relaxed_u64(&state[tile], lb_pack(epoch, LB_INCLUSIVE, excl + aggregate));
  return excl;
}

}  // namespace kvg
