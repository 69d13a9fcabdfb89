// kvg_common.cuh — device-side building blocks shared by every kernel of libkvgpu.so (sm_90a).
//
//   * streaming global loads/stores (ld.global.nc.L1::no_allocate / st.global.L1::no_allocate)
//   * mbarrier + 1-D TMA bulk copy (cp.async.bulk ... mbarrier::complete_tx::bytes -> SASS UBLKCP)
//   * warp / block scans
//   * epoch-tagged decoupled look-back (single-pass chained scan) used by the stable compactions
//     and by the vendor-context carry of the pci.ids parser
//   * the tile front-end of every compaction (ClassifyTile) and its look-back tile body (lookback_tile)
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

// Sum look-back, executed by one full warp.  Publishes this tile's aggregate, walks the predecessors 32 at a time
// (one state word per lane) and returns the exclusive prefix (valid in every lane); publishes the inclusive.
// (Measured: windows of 8 x 32 predecessors per step, all loads independent, were slower — more polling traffic.)
__device__ __forceinline__ uint32_t lookback_sum(uint64_t* state, uint32_t tile, uint32_t aggregate,
                                                 uint32_t epoch) {
  const uint32_t lane = lane_id();
  if (tile == 0) {
    if (lane == 0) st_relaxed_u64(&state[0], lb_pack(epoch, LB_INCLUSIVE, aggregate));
    return 0;
  }
  if (lane == 0) st_relaxed_u64(&state[tile], lb_pack(epoch, LB_AGGREGATE, aggregate));
  uint32_t excl = 0;
  for (int look = (int)tile - 1;;) {
    const int idx = look - (int)lane;
    const uint64_t w = idx >= 0 ? ld_relaxed_u64(&state[idx]) : lb_pack(epoch, LB_INCLUSIVE, 0);
    const uint32_t st = lb_status(w, epoch);
    const uint32_t incl_mask = __ballot_sync(KVG_FULL, st == LB_INCLUSIVE);
    const uint32_t inv_mask = __ballot_sync(KVG_FULL, st == LB_INVALID);
    const uint32_t first = incl_mask ? (uint32_t)__ffs(incl_mask) - 1 : 32;
    const uint32_t need = first >= 31 ? KVG_FULL : ((2u << first) - 1);  // lanes 0..first
    if (inv_mask & need) continue;  // a needed predecessor is not published yet: reload the same window
    excl += warp_sum(lane <= first ? (uint32_t)w : 0u);
    if (first < 32) break;
    look -= 32;
  }
  if (lane == 0) st_relaxed_u64(&state[tile], lb_pack(epoch, LB_INCLUSIVE, excl + aggregate));
  return excl;
}

// ------------------------------------------------------------------------------------------------
// The tile front-end of every compaction (classify, health, the ordering heads, the delta lists).  A warp owns 32 x ROWS consecutive records of the tile
// (THREADS x ROWS records); `classify` issues every load before the first ballot, votes Op::pred per row and
// calls Op::prepare for the survivors, whose dependent loads then overlap what the kernel does next.  `emit`
// hands each of the lane's survivors to f(pos, item, i, aux), numbered in record order from the warp's offset.
//   Op::Item                          what a thread holds per record
//   uint32_t n                        number of records
//   Item load(uint32_t i, bool ok)    ok == false -> any value that fails pred
//   bool pred(const Item&, i)
//   uint32_t prepare(const Item&)     per-survivor value handed to emit (name slot, canonical type)
// ------------------------------------------------------------------------------------------------
template <class Op, int THREADS, int ROWS>
struct ClassifyTile {
  static constexpr uint32_t TILE = THREADS * ROWS;
  static constexpr uint32_t NW = THREADS / 32;
  static constexpr uint32_t WARP_ITEMS = 32 * ROWS;
  typename Op::Item item[ROWS];
  uint32_t bal[ROWS], aux[ROWS];
  uint32_t base;  // the warp's first record
  uint32_t wtot;  // the warp's survivors

  __device__ __forceinline__ void classify(Op& op, uint32_t tile) {
    const uint32_t lane = lane_id(), n = op.n;
    base = tile * TILE + (threadIdx.x >> 5) * WARP_ITEMS;
#pragma unroll
    for (int k = 0; k < ROWS; k++) {
      const uint32_t i = base + k * 32 + lane;
      item[k] = op.load(i, i < n);
    }
    wtot = 0;
#pragma unroll
    for (int k = 0; k < ROWS; k++) {
      const uint32_t i = base + k * 32 + lane;
      const bool p = i < n && op.pred(item[k], i);
      bal[k] = __ballot_sync(KVG_FULL, p);
      wtot += __popc(bal[k]);
      aux[k] = p ? op.prepare(item[k]) : 0u;
    }
  }
  template <class F>
  __device__ __forceinline__ void emit(uint32_t off, F&& f) const {
    const uint32_t lane = lane_id();
#pragma unroll
    for (int k = 0; k < ROWS; k++) {
      if ((bal[k] >> lane) & 1u) f(off + __popc(bal[k] & lanemask_lt()), item[k], base + k * 32 + lane, aux[k]);
      off += __popc(bal[k]);
    }
  }
};

// One tile of the look-back compaction: classify it, place it behind all earlier tiles (decoupled look-back on
// the tile counts), write its survivors.  Besides the front-end, Op provides emit(pos, item, i, aux),
// tile_epilogue() (once per warp after its survivors) and finish(total) (one thread of the last tile).
// s_wtot / s_woff: a word per warp of shared memory.
template <class Op, int THREADS, int ROWS>
__device__ __forceinline__ void lookback_tile(Op& op, uint32_t tile, uint32_t n_tiles, uint64_t* tile_state, uint32_t epoch,
                                              uint32_t* s_wtot, uint32_t* s_woff, uint32_t& s_base) {
  constexpr uint32_t NW = THREADS / 32;
  const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
  ClassifyTile<Op, THREADS, ROWS> ct;
  ct.classify(op, tile);
  if (lane == 0) s_wtot[warp] = ct.wtot;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < NW ? s_wtot[lane] : 0;
    uint32_t wi = warp_incl_sum(w);
    if (lane < NW) s_woff[lane] = wi - w;
    uint32_t tile_total = __shfl_sync(KVG_FULL, wi, NW - 1);
    uint32_t excl = lookback_sum(tile_state, tile, tile_total, epoch);
    if (lane == 0) {
      s_base = excl;
      if (tile == n_tiles - 1) op.finish(excl + tile_total);
    }
  }
  __syncthreads();
  ct.emit(s_base + s_woff[warp], [&](uint32_t pos, const typename Op::Item& r, uint32_t i, uint32_t a) { op.emit(pos, r, i, a); });
  op.tile_epilogue();
}

// The whole look-back compaction of op.n records: tiles blockIdx.x, blockIdx.x + gridDim.x, ... (a grid of one CTA
// per tile runs the loop once; a smaller grid must be co-resident, since a tile waits for every lower one).  An empty
// list still finishes, with total 0.
template <class Op, int THREADS, int ROWS>
__device__ __forceinline__ void lookback_tiles(Op& op, uint64_t* tile_state, uint32_t epoch) {
  constexpr uint32_t TILE = THREADS * ROWS;
  __shared__ uint32_t s_wtot[THREADS / 32], s_woff[THREADS / 32];
  __shared__ uint32_t s_base;
  const uint32_t n_tiles = (op.n + TILE - 1) / TILE;
  if (n_tiles == 0 && blockIdx.x == 0 && threadIdx.x == 0) op.finish(0);
  for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)
    lookback_tile<Op, THREADS, ROWS>(op, tile, n_tiles, tile_state, epoch, s_wtot, s_woff, s_base);
}

}  // namespace kvg
