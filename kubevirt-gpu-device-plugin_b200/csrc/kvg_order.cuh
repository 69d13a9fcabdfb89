// kvg_order.cuh — K4: the two stable orderings of a survivor list (deviceMap / iommuMap of
// createIommuDeviceMap, device_plugin.go:240-242; vGpuMap / gpuVgpuMap of createVgpuIDMap, :287-288).
//
// Stable LSD radix sort of {key, survivor index} pairs over 2048-pair tiles; both orderings share every
// launch (blockIdx.y).  Per pass:
//   k_order_hist       per-tile digit histogram (shared-memory atomics, all loads of a tile in flight first)
//   k_order_tilescan   one WARP per digit row: exclusive scan over the tiles, in place; digit totals
//   k_order_scatter    every thread OWNS a run of consecutive digits (8 at 11-bit digits), so the digit bases
//                      and the tile-local starts are ONE block scan each; ranks by match + per-warp u16
//                      counters, stages the tile in shared memory in sorted order and writes bucket runs with
//                      consecutive threads on consecutive addresses
// then the final permutation and the segment heads (distinct keys + offsets, the bucket's joined name slot):
//   k_order_final      latency-bound sizes: ONE launch, chained scan of the per-tile head counts
//   k_order_heads<0/1> bandwidth-bound sizes: count -> k_tile_offsets -> emit (no CTA ever waits for another)
//
// Measured dead end (kept here so nobody repeats it): accumulating the histograms with global REDs from the
// producers (one per survivor from the classify / pack kernel for pass 0, one per element from the scatter for
// the next pass) removes the histogram launches but costs more than they do — in the 1 M-record classify, in
// its pass-0 scatter (hot rows) and in the 16.7 M-record pack.
//
// Second measured dead end: the whole step as ONE persistent launch (the same device functions in a grid that
// fits the GPU, 3 grid barriers per pass + 1 for the heads).  Correct (GPU suite green) but SLOWER at 1 M
// records: seven grid barriers cost more than the nine launch boundaries they replace once those launches
// overlap through programmatic dependent launch.
//
// Digit width is decided ON THE DEVICE from the largest key of the ordering: the fewest passes of at most
// `max_bits` bits, the key bits split evenly between them (19-bit keys: 2 passes of 10 bits; 16-bit keys:
// 2 x 8; 23-bit: 3 x 8).  Every CTA of every kernel of a pass derives the same plan from the same word, so
// nothing about it crosses the host; a pass above the largest key returns immediately and the ping-pong
// parity tells consumers which buffer is final.
#pragma once
#include "kvg_common.cuh"

namespace kvg {

constexpr uint32_t C_ROWS = 8;                      // items per thread
constexpr uint32_t C_TILE = KVG_BLOCK * C_ROWS;     // 2048 items per tile
constexpr uint32_t C_WARP_ITEMS = 32 * C_ROWS;      // 256 contiguous items per warp

enum : int { SRC_PAIRS = 0, SRC_PCI_GROUP = 1, SRC_PCI_DEVICE = 2, SRC_MDEV_PARENT = 3, SRC_MDEV_TYPE = 4 };

constexpr uint32_t RADIX_MAX_BITS = 11;
constexpr uint32_t RADIX_MAX_DIGITS = 1u << RADIX_MAX_BITS;  // 2048
struct RadixPlan {
  uint32_t npass, shift, bits;  // of the queried pass; bits == 0: the pass does not exist
};
__host__ __device__ __forceinline__ RadixPlan radix_plan(uint32_t max_key, uint32_t key_bits_max, uint32_t pass,
                                                         uint32_t max_bits) {
#ifdef __CUDA_ARCH__
  uint32_t kb = max_key ? 32u - (uint32_t)__clz((int)max_key) : 1u;
#else
  uint32_t kb = 1;
  while (kb < 32 && (max_key >> kb) != 0) kb++;
#endif
  if (kb > key_bits_max) kb = key_bits_max;
  RadixPlan r;
  r.npass = (kb + max_bits - 1) / max_bits;
  const uint32_t w = (kb + r.npass - 1) / r.npass;
  r.shift = pass * w;
  r.bits = pass < r.npass ? (kb - r.shift < w ? kb - r.shift : w) : 0;
  return r;
}

struct OrdArgs {
  const uint32_t* n_ptr;    // element count (device)
  const uint32_t* max_key;  // largest key (device): decides the plan
  const void* src_records;  // survivors (pass 0)
  const uint2* pairs_in;    // {key, index} (passes >= 1)
  uint2* pairs_out;
  uint32_t* tile_hist;      // tile_major = 0: [digit][T] (T = ceil(n / C_TILE)); 1: [T][D] (D = digits padded to 256)
  uint32_t tile_major;      // 1 at latency-bound sizes: the histogram kernel writes a tile's counts as ONE contiguous
                            // row and the scatter kernel reads its eight digits as ONE 32-byte load (digit-major,
                            // each was 1024-2048 scattered 4-byte accesses per CTA); the tile scan then walks columns
  uint32_t* bin_total;      // [RADIX_MAX_DIGITS] digit totals of this pass
  uint32_t pass;            // 0xff: this ordering has no such launch set
  uint32_t key_bits_max;    // 16 (device id / type) or 32 (iommu group / parent)
  uint32_t max_bits;        // widest digit: 11 (latency-bound sizes) or 8 (large inputs)
  int src;                  // where pass-0 keys come from
};
struct OrdArgs2 {
  OrdArgs o[2];
};
__device__ __forceinline__ RadixPlan ord_pass(const OrdArgs& a) {
  if (a.pass == 0xffu) {
    RadixPlan r = {0, 0, 0};
    return r;
  }
  return radix_plan(*a.max_key, a.key_bits_max, a.pass, a.max_bits);
}
__device__ __forceinline__ uint2 ord_load(const OrdArgs& a, uint32_t i) {
  // survivors are 16-byte (PCI) or 32-byte (mdev) records; see kvgpu.h
  const uint4* rec = reinterpret_cast<const uint4*>(a.src_records);
  switch (a.src) {
    case SRC_PCI_GROUP: return make_uint2(__ldg(&reinterpret_cast<const uint32_t*>(rec + i)[1]), i);
    case SRC_PCI_DEVICE: return make_uint2(__ldg(&reinterpret_cast<const uint32_t*>(rec + i)[2]) & 0xffffu, i);
    case SRC_MDEV_PARENT: return make_uint2(__ldg(&reinterpret_cast<const uint32_t*>(rec + 2 * (size_t)i + 1)[0]), i);
    case SRC_MDEV_TYPE: return make_uint2(__ldg(&reinterpret_cast<const uint32_t*>(rec + 2 * (size_t)i + 1)[1]) & 0xffffu, i);
    default: return a.pairs_in[i];
  }
}

// ---- histogram ----------------------------------------------------------------------------------
// tiles tile0, tile0 + tstride, ... of one ordering; h: RADIX_MAX_DIGITS words of shared memory
__device__ __forceinline__ void ord_hist_tiles(const OrdArgs& a, const RadixPlan pl, uint32_t tile0, uint32_t tstride,
                                               uint32_t* h) {
  const uint32_t n = *a.n_ptr;
  const uint32_t T = (n + C_TILE - 1) / C_TILE;
  const uint32_t dmask = (1u << pl.bits) - 1;
  const uint32_t nj = ((1u << pl.bits) + KVG_BLOCK - 1) / KVG_BLOCK;  // digit chunks in use
  const uint32_t lane = lane_id();
  for (uint32_t tile = tile0; tile < T; tile += tstride) {
    for (uint32_t j = 0; j < nj; j++) h[j * KVG_BLOCK + threadIdx.x] = 0;
    __syncthreads();
    const uint32_t base = tile * C_TILE + warp_id() * C_WARP_ITEMS;
    uint32_t d[C_ROWS];
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++) {  // all loads in flight before the first shared atomic
      uint32_t i = base + k * 32 + lane;
      d[k] = i < n ? ((ord_load(a, i).x >> pl.shift) & dmask) : 0xffffffffu;
    }
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++)
      if (d[k] != 0xffffffffu) atomicAdd(&h[d[k]], 1u);
    __syncthreads();
    for (uint32_t j = 0; j < nj; j++) {
      const uint32_t dg = j * KVG_BLOCK + threadIdx.x;
      if (a.tile_major)
        a.tile_hist[(size_t)tile * (nj * KVG_BLOCK) + dg] = h[dg];
      else
        a.tile_hist[(size_t)dg * T + tile] = h[dg];
    }
    __syncthreads();
  }
}
__global__ void __launch_bounds__(KVG_BLOCK) k_order_hist(OrdArgs2 aa) {
  pdl_enter();
  const OrdArgs a = blockIdx.y ? aa.o[1] : aa.o[0];  // static indices: parameters stay in the constant bank
  const RadixPlan pl = ord_pass(a);
  if (!pl.bits) return;
  __shared__ uint32_t h[RADIX_MAX_DIGITS];
  // tile loop: launched with one CTA per tile for the always-active passes, with a small grid for the
  // high passes that are usually ruled out by the device-side max key (they then cost ~nothing)
  ord_hist_tiles(a, pl, blockIdx.x, gridDim.x, h);
}

// ---- tile scan: one warp per digit row, in place; bin_total[digit] <- the row's total -----------------
constexpr uint32_t TS_WARPS = 8;  // digit rows per CTA
// digit rows row0, row0 + rstride, ... of one ordering, one warp per row
__device__ __forceinline__ void ord_tilescan_rows(const OrdArgs& a, const RadixPlan pl, uint32_t row0, uint32_t rstride) {
  const uint32_t n = *a.n_ptr;
  const uint32_t T = (n + C_TILE - 1) / C_TILE;
  if (T == 0) return;
  const uint32_t digits = (((1u << pl.bits) + KVG_BLOCK - 1) / KVG_BLOCK) * KVG_BLOCK;  // rows the histogram wrote
  const uint32_t lane = lane_id();
  for (uint32_t dg = row0; dg < digits; dg += rstride) {
    uint32_t* row = a.tile_hist + (size_t)dg * T;
    uint32_t carry = 0;
    for (uint32_t b = 0; b < T; b += 128) {  // four independent loads per lane and round
      uint32_t v[4], incl[4];
#pragma unroll
      for (uint32_t q = 0; q < 4; q++) {
        const uint32_t i = b + q * 32 + lane;
        v[q] = i < T ? row[i] : 0;
      }
#pragma unroll
      for (uint32_t q = 0; q < 4; q++) {
        const uint32_t i = b + q * 32 + lane;
        incl[q] = warp_incl_sum(v[q]);
        if (i < T) row[i] = carry + incl[q] - v[q];
        carry += __shfl_sync(KVG_FULL, incl[q], 31);
      }
    }
    if (lane == 0) a.bin_total[dg] = carry;
  }
}
__global__ void __launch_bounds__(TS_WARPS * 32) k_order_tilescan(OrdArgs2 aa) {
  pdl_enter();
  const OrdArgs a = blockIdx.y ? aa.o[1] : aa.o[0];  // static indices: parameters stay in the constant bank
  const RadixPlan pl = ord_pass(a);
  if (!pl.bits) return;
  ord_tilescan_rows(a, pl, blockIdx.x * TS_WARPS + (threadIdx.x >> 5), gridDim.x * TS_WARPS);
}

// the same for long rows (bandwidth-bound sizes: thousands of tiles): one CTA per digit row, every thread
// scans a contiguous slice, one block scan combines the slices
__global__ void __launch_bounds__(KVG_BLOCK) k_order_tilescan_long(OrdArgs2 aa) {
  pdl_enter();
  const OrdArgs a = blockIdx.y ? aa.o[1] : aa.o[0];
  const uint32_t n = *a.n_ptr;
  const uint32_t T = (n + C_TILE - 1) / C_TILE;
  const RadixPlan pl = ord_pass(a);
  if (T == 0 || !pl.bits) return;
  const uint32_t digits = (((1u << pl.bits) + KVG_BLOCK - 1) / KVG_BLOCK) * KVG_BLOCK;
  __shared__ uint32_t scratch[KVG_WARPS + 1];
  const uint32_t per = (T + KVG_BLOCK - 1) / KVG_BLOCK;
  for (uint32_t dg = blockIdx.x; dg < digits; dg += gridDim.x) {
    uint32_t* row = a.tile_hist + (size_t)dg * T;
    const uint32_t i0 = threadIdx.x * per, i1 = min(T, i0 + per);
    uint32_t sum = 0;
    for (uint32_t i = i0; i < i1; i++) sum += row[i];
    uint32_t total;
    uint32_t run = block_excl_sum(sum, scratch, &total);  // syncs inside
    for (uint32_t i = i0; i < i1; i++) {
      const uint32_t v = row[i];
      row[i] = run;
      run += v;
    }
    if (threadIdx.x == 0) a.bin_total[dg] = total;
    __syncthreads();
  }
}

// tile-major layout: one CTA per group of 32 digits (a lane per digit: coalesced rows), its 8 warps split the
// tiles; pass 1 sums a warp's slice per digit, the slices are combined in shared memory, pass 2 rewrites the
// slice as exclusive prefixes.  64 CTAs per ordering at 11-bit digits: one wave.
__global__ void __launch_bounds__(KVG_BLOCK) k_order_tilescan_cols(OrdArgs2 aa) {
  pdl_enter();
  const OrdArgs a = blockIdx.y ? aa.o[1] : aa.o[0];
  const RadixPlan pl = ord_pass(a);
  if (!pl.bits) return;
  const uint32_t n = *a.n_ptr;
  const uint32_t T = (n + C_TILE - 1) / C_TILE;
  if (T == 0) return;
  const uint32_t D = (((1u << pl.bits) + KVG_BLOCK - 1) / KVG_BLOCK) * KVG_BLOCK;
  __shared__ uint32_t s_part[KVG_WARPS][32];
  const uint32_t lane = lane_id(), warp = warp_id();
  const uint32_t per = (T + KVG_WARPS - 1) / KVG_WARPS;
  const uint32_t t0 = min(T, warp * per), t1 = min(T, t0 + per);
  for (uint32_t g = blockIdx.x; g * 32 < D; g += gridDim.x) {
    uint32_t* col = a.tile_hist + g * 32 + lane;
    if (per <= 32) {
      // the whole slice of a lane fits in registers (up to 256 tiles, i.e. 512 K elements): ONE read with every
      // load in flight, one write
      uint32_t v[32];
      uint32_t sum = 0;
#pragma unroll
      for (uint32_t k = 0; k < 32; k++) v[k] = t0 + k < t1 ? col[(size_t)(t0 + k) * D] : 0;
#pragma unroll
      for (uint32_t k = 0; k < 32; k++) sum += v[k];
      s_part[warp][lane] = sum;
      __syncthreads();
      uint32_t run = 0, total = 0;
#pragma unroll
      for (uint32_t w = 0; w < KVG_WARPS; w++) {
        const uint32_t c = s_part[w][lane];
        if (w < warp) run += c;
        total += c;
      }
      if (warp == 0) a.bin_total[g * 32 + lane] = total;
#pragma unroll
      for (uint32_t k = 0; k < 32; k++) {
        if (t0 + k < t1) col[(size_t)(t0 + k) * D] = run;
        run += v[k];
      }
      __syncthreads();  // s_part is rewritten by the next group
      continue;
    }
    uint32_t sum = 0;
    for (uint32_t t = t0; t < t1; t += 8) {  // eight independent loads per round
      uint32_t v[8];
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) v[k] = t + k < t1 ? col[(size_t)(t + k) * D] : 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) sum += v[k];
    }
    s_part[warp][lane] = sum;
    __syncthreads();
    uint32_t run = 0, total = 0;
#pragma unroll
    for (uint32_t w = 0; w < KVG_WARPS; w++) {
      const uint32_t c = s_part[w][lane];
      if (w < warp) run += c;
      total += c;
    }
    if (warp == 0) a.bin_total[g * 32 + lane] = total;
    for (uint32_t t = t0; t < t1; t += 8) {
      uint32_t v[8];
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) v[k] = t + k < t1 ? col[(size_t)(t + k) * D] : 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) {
        if (t + k < t1) col[(size_t)(t + k) * D] = run;
        run += v[k];
      }
    }
    __syncthreads();  // s_part is rewritten by the next group
  }
}

// ---- scatter ------------------------------------------------------------------------------------
// dynamic shared memory: per-warp digit counts (u16: a warp owns 256 items), tile-local digit starts,
// global run offsets, the staged tile
// (11-bit digits: 32 + 4 + 8 + 16 = 60 KiB, 3 CTAs/SM; 8-bit digits: 4 + 0.5 + 1 + 16 KiB, 5 CTAs/SM)
template <uint32_t MAXB>
struct OrdScatterCfg {
  static constexpr uint32_t DIGITS = 1u << MAXB;
  static constexpr uint32_t DPT = DIGITS / KVG_BLOCK;  // consecutive digits owned by a thread (8 or 1)
  static constexpr uint32_t CNT_BYTES = KVG_WARPS * DIGITS * 2;
  static constexpr uint32_t START_BYTES = DIGITS * 2;
  static constexpr uint32_t GOFF_BYTES = DIGITS * 4;
  static constexpr uint32_t STAGE_BYTES = C_TILE * 8;
  static constexpr uint32_t SMEM = CNT_BYTES + START_BYTES + GOFF_BYTES + STAGE_BYTES;
  static constexpr int MIN_CTAS = MAXB <= 8 ? 5 : 3;  // 6 would cap registers at 40 and spill
};

// tiles tile0, tile0 + tstride, ... of one ordering; rs_smem: Cfg::SMEM bytes, scratch: KVG_WARPS + 1 words
template <uint32_t MAXB>
__device__ __forceinline__ void ord_scatter_tiles(const OrdArgs& a, const RadixPlan pl, uint32_t tile0, uint32_t tstride,
                                                  uint8_t* rs_smem, uint32_t* scratch) {
  using Cfg = OrdScatterCfg<MAXB>;
  constexpr uint32_t DPT = Cfg::DPT;
  const uint32_t n = *a.n_ptr;
  const uint32_t T = (n + C_TILE - 1) / C_TILE;
  const uint32_t dmask = (1u << pl.bits) - 1;
  const uint32_t digits = 1u << pl.bits;
  const uint32_t lane = lane_id(), warp = warp_id(), tid = threadIdx.x;
  const uint32_t d0 = tid * DPT;  // my digits: d0 .. d0 + DPT - 1
  const bool mine = d0 < digits;
  const uint32_t DP = ((digits + KVG_BLOCK - 1) / KVG_BLOCK) * KVG_BLOCK;  // row pitch of the tile-major layout
  uint16_t (*s_cnt)[Cfg::DIGITS] = reinterpret_cast<uint16_t (*)[Cfg::DIGITS]>(rs_smem);
  uint16_t* s_start = reinterpret_cast<uint16_t*>(rs_smem + Cfg::CNT_BYTES);
  int32_t* s_goff = reinterpret_cast<int32_t*>(rs_smem + Cfg::CNT_BYTES + Cfg::START_BYTES);
  uint2* s_stage = reinterpret_cast<uint2*>(rs_smem + Cfg::CNT_BYTES + Cfg::START_BYTES + Cfg::GOFF_BYTES);
  uint32_t total;
  uint32_t bin_base[DPT];
  bool have_base = false;
  for (uint32_t tile = tile0; tile < T; tile += tstride) {
    const uint32_t base = tile * C_TILE + warp * C_WARP_ITEMS;
    // all global loads of the tile up front: the scanned tile counts of my digits, the pairs
    uint32_t tile_prefix[DPT];
#pragma unroll
    for (uint32_t q = 0; q < DPT; q++)
      tile_prefix[q] = (mine && d0 + q < digits)
                           ? (a.tile_major ? a.tile_hist[(size_t)tile * DP + d0 + q] : a.tile_hist[(size_t)(d0 + q) * T + tile])
                           : 0;
    uint2 kv[C_ROWS];
    uint32_t rank[C_ROWS];
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++) {
      uint32_t i = base + k * 32 + lane;
      kv[k] = i < n ? ord_load(a, i) : make_uint2(0, 0);
    }
    __syncthreads();  // previous tile's stage fully written out
    if (mine) {
#pragma unroll
      for (uint32_t w = 0; w < KVG_WARPS; w++) {
        if constexpr (DPT == 8)  // my eight u16 counters of a warp row are ONE 128-bit word
          *reinterpret_cast<uint4*>(&s_cnt[w][d0]) = make_uint4(0, 0, 0, 0);
        else
          s_cnt[w][d0] = 0;
      }
    }
    if (!have_base) {  // exclusive scan of the digit totals: local prefix over my digits + ONE block scan
      uint32_t loc[DPT], sum = 0;
#pragma unroll
      for (uint32_t q = 0; q < DPT; q++) {
        loc[q] = sum;
        sum += (mine && d0 + q < digits) ? a.bin_total[d0 + q] : 0;
      }
      const uint32_t excl = block_excl_sum(sum, scratch, &total);  // syncs inside
#pragma unroll
      for (uint32_t q = 0; q < DPT; q++) bin_base[q] = excl + loc[q];
      have_base = true;
    }
    __syncthreads();
    // stable rank inside the warp: rows in order, lanes in order within a row
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++) {
      uint32_t i = base + k * 32 + lane;
      bool ok = i < n;
      uint32_t d = ok ? ((kv[k].x >> pl.shift) & dmask) : (0x10000u + lane);  // inactive lanes: unique
      uint32_t peers = __match_any_sync(KVG_FULL, d);
      uint32_t leader = (uint32_t)__ffs(peers) - 1;
      uint32_t before = 0;
      if (ok && lane == leader) {
        before = s_cnt[warp][d];
        s_cnt[warp][d] = (uint16_t)(before + __popc(peers));
      }
      before = __shfl_sync(KVG_FULL, before, leader);
      rank[k] = before + __popc(peers & lanemask_lt());
      __syncwarp();
    }
    __syncthreads();
    {  // my digits: exclusive prefix over the warps, totals, then ONE block scan for the tile-local starts
      uint32_t dtot[DPT];
#pragma unroll
      for (uint32_t q = 0; q < DPT; q++) dtot[q] = 0;
      if (mine) {
#pragma unroll
        for (uint32_t w = 0; w < KVG_WARPS; w++) {
          if constexpr (DPT == 8) {  // conflict-free LDS.128 / STS.128 over my eight counters
            uint4* row = reinterpret_cast<uint4*>(&s_cnt[w][d0]);
            const uint4 c = *row;
            const uint32_t cw[4] = {c.x, c.y, c.z, c.w};
            uint32_t pw[4];
#pragma unroll
            for (uint32_t h = 0; h < 4; h++) {  // counters 2h (low half) and 2h + 1 (high half)
              pw[h] = (dtot[2 * h] & 0xffffu) | (dtot[2 * h + 1] << 16);
              dtot[2 * h] += cw[h] & 0xffffu;
              dtot[2 * h + 1] += cw[h] >> 16;
            }
            *row = make_uint4(pw[0], pw[1], pw[2], pw[3]);
          } else {
            const uint32_t c = s_cnt[w][d0];
            s_cnt[w][d0] = (uint16_t)dtot[0];
            dtot[0] += c;
          }
        }
      }
      uint32_t loc[DPT], sum = 0;
#pragma unroll
      for (uint32_t q = 0; q < DPT; q++) {
        loc[q] = sum;
        sum += dtot[q];
      }
      const uint32_t excl = block_excl_sum(sum, scratch, &total);  // syncs inside
      if (mine) {
#pragma unroll
        for (uint32_t q = 0; q < DPT; q++) {
          const uint32_t lstart = excl + loc[q];
          s_start[d0 + q] = (uint16_t)lstart;
          s_goff[d0 + q] = (int32_t)(bin_base[q] + tile_prefix[q]) - (int32_t)lstart;
        }
      }
      __syncthreads();
    }
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++) {
      uint32_t i = base + k * 32 + lane;
      if (i < n) {
        uint32_t d = (kv[k].x >> pl.shift) & dmask;
        s_stage[(uint32_t)s_start[d] + s_cnt[warp][d] + rank[k]] = kv[k];
      }
    }
    __syncthreads();
    const uint32_t cnt = min(C_TILE, n - tile * C_TILE);
    for (uint32_t j = tid; j < cnt; j += KVG_BLOCK) {
      uint2 e = s_stage[j];
      uint32_t d = (e.x >> pl.shift) & dmask;
      a.pairs_out[(uint32_t)(s_goff[d] + (int32_t)j)] = e;
    }
  }  // tile loop
}
template <uint32_t MAXB>
__global__ void __launch_bounds__(KVG_BLOCK, OrdScatterCfg<MAXB>::MIN_CTAS) k_order_scatter(OrdArgs2 aa) {
  pdl_enter();
  const OrdArgs a = blockIdx.y ? aa.o[1] : aa.o[0];  // static indices: parameters stay in the constant bank
  const RadixPlan pl = ord_pass(a);
  if (!pl.bits) return;
#ifndef KVG_HOST_EMU
  extern __shared__ __align__(16) uint8_t rs_smem[];
#else
  static __attribute__((aligned(16))) uint8_t rs_smem[OrdScatterCfg<MAXB>::SMEM];
#endif
  __shared__ uint32_t scratch[KVG_WARPS + 1];
  ord_scatter_tiles<MAXB>(a, pl, blockIdx.x, gridDim.x, rs_smem, scratch);
}

// ---- final permutation + distinct keys of both orderings ------------------------------------------
struct OrdFinalArgs {
  const uint2* p0;  // ping-pong buffers of the radix passes
  const uint2* p1;
  const uint32_t* max_key;
  uint32_t key_bits_max, max_bits;
  const uint32_t* n_ptr;
  uint32_t* perm;            // [n] survivor indices in key order (stable)
  uint64_t* state;           // k_order_final: [tiles] chained scan of the head counts (epoch-tagged)
  uint32_t* tile_heads;      // k_order_heads: [T] number of segment heads in each tile
  const uint32_t* tile_off;  // k_order_heads<true>: [T+1] exclusive scan of tile_heads
  uint32_t* seg_key;
  uint32_t* seg_off;         // [n_seg + 1]
  uint32_t* n_seg;           // total heads (written by k_order_final / k_tile_offsets)
  const uint4* head_surv;    // optional: survivors, to publish the joined name slot of each segment
  uint32_t* head_name;       // [n_seg] name slot of the segment's first member (NULL: skip)
  // deferred name join (the pci.ids parse ran beside the classification, on another stream): while the
  // permutation is written every record of the list gets its name slot — join 1: nv_index[key] (the ordering's
  // key IS the device id), join 2: nv_index[device id read from the record]; 0: names were joined at classify time
  const uint32_t* join_index;
  uint4* join_recs;
  uint32_t join;
};
struct OrdFinalArgs2 {
  OrdFinalArgs o[2];
};
__device__ __forceinline__ const uint2* ord_final_buf(const OrdFinalArgs& a) {
  const uint32_t np = radix_plan(*a.max_key, a.key_bits_max, 0, a.max_bits).npass;
  return ((np - 1) & 1) ? a.p1 : a.p0;
}
// The segment heads of the sorted pairs as a ClassifyTile operator: element i is a head iff i == 0 or its key differs
// from element i - 1's.  The previous key comes from the lane below, or for lane 0 (its predecessor lives in another
// row or tile) from memory; it is taken in load, which every lane runs, so the shuffle is convergent.
struct OrdHeadsOp {
  struct Item {
    uint32_t key, idx, prev;
  };
  OrdFinalArgs a;
  const uint2* pairs;  // the sorted pairs (the final radix buffer)
  uint32_t n;
  bool write_perm;     // the launch that owns the permutation (and the deferred name join)

  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    Item it = {0u, 0u, 0u};
    if (ok) {
      const uint2 e = pairs[i];
      it.key = e.x;
      it.idx = e.y;
      if (write_perm) {
        a.perm[i] = e.y;
        if (a.join == 1)
          reinterpret_cast<uint32_t*>(a.join_recs + e.y)[3] = __ldg(&a.join_index[e.x & 0xffffu]);
        else if (a.join == 2)
          reinterpret_cast<uint32_t*>(a.join_recs + e.y)[3] =
              __ldg(&a.join_index[reinterpret_cast<const uint32_t*>(a.join_recs + e.y)[2] & 0xffffu]);
      }
    }
    it.prev = __shfl_up_sync(KVG_FULL, it.key, 1);
    if (ok && lane_id() == 0 && i) it.prev = pairs[i - 1].x;  // overwrites the shuffled value: one register per row
    return it;
  }
  __device__ __forceinline__ bool pred(const Item& it, uint32_t i) const { return i == 0 || it.prev != it.key; }
  __device__ __forceinline__ uint32_t prepare(const Item&) const { return 0; }
  __device__ __forceinline__ void emit(uint32_t pos, const Item& it, uint32_t i, uint32_t) const {
    a.seg_key[pos] = it.key;
    a.seg_off[pos] = i;
    // all members of a device-id bucket share the name (same id): take the first member's slot
    if (a.head_name)  // deferred join: straight from the table (the record's slot may be written by another thread)
      a.head_name[pos] = a.join ? __ldg(&a.join_index[it.key & 0xffffu]) : __ldg(&a.head_surv[it.idx].w);
  }
  __device__ __forceinline__ void tile_epilogue() {}
  __device__ __forceinline__ void finish(uint32_t total) const {
    *a.n_seg = total;
    a.seg_off[total] = n;
  }
};
// the operator of ordering blockIdx.y
__device__ __forceinline__ OrdHeadsOp ord_heads_op(const OrdFinalArgs2& aa, bool write_perm) {
  OrdHeadsOp op;
  op.a = blockIdx.y ? aa.o[1] : aa.o[0];  // static indices: parameters stay in the constant bank
  op.n = *op.a.n_ptr;
  op.pairs = ord_final_buf(op.a);
  op.write_perm = write_perm;
  return op;
}

// latency-bound sizes: one launch; the per-tile head counts are combined by a chained scan (look-back).
// Tile loop: the grid may be smaller than the tile count (the sharded scan sizes it for the EXPECTED length of
// an owned list, not for its capacity) — it must then fit the GPU at once (a CTA waits for lower tiles, which
// must be running or done: enqueue_orderings bounds the grid by the occupancy).  6 CTAs per SM: 40 registers, which
// ptxas meets without spilling (left to itself it takes 48, i.e. 5 CTAs per SM and a smaller grid).
__global__ void __launch_bounds__(KVG_BLOCK, 6) k_order_final(OrdFinalArgs2 aa, uint32_t epoch) {
  pdl_enter();
  OrdHeadsOp op = ord_heads_op(aa, true);
  lookback_tiles<OrdHeadsOp, KVG_BLOCK, C_ROWS>(op, op.a.state, epoch);
}

// bandwidth-bound sizes: <false> writes the permutation and counts heads per tile, k_tile_offsets scans the
// counts (and writes n_seg), <true> emits the heads at known offsets
template <bool EMIT>
__global__ void __launch_bounds__(KVG_BLOCK) k_order_heads(OrdFinalArgs2 aa) {
  pdl_enter();
  using Tile = ClassifyTile<OrdHeadsOp, KVG_BLOCK, C_ROWS>;
  OrdHeadsOp op = ord_heads_op(aa, !EMIT);
  const uint32_t T = (op.n + C_TILE - 1) / C_TILE;
  const uint32_t lane = lane_id(), warp = warp_id();
  // n_seg came from k_tile_offsets; finishing ends the last segment (of an empty list too)
  if (EMIT && blockIdx.x == 0 && threadIdx.x == 0) op.finish(*op.a.n_seg);
  __shared__ uint32_t s_w[KVG_WARPS];
  for (uint32_t tile = blockIdx.x; tile < T; tile += gridDim.x) {
    Tile ct;
    ct.classify(op, tile);
    if (lane == 0) s_w[warp] = ct.wtot;
    __syncthreads();
    if (!EMIT) {
      if (threadIdx.x == 0) {
        uint32_t t = 0;
#pragma unroll
        for (uint32_t w = 0; w < KVG_WARPS; w++) t += s_w[w];
        op.a.tile_heads[tile] = t;
      }
    } else {
      uint32_t off = op.a.tile_off[tile];
#pragma unroll
      for (uint32_t w = 0; w < KVG_WARPS; w++)
        if (w < warp) off += s_w[w];
      ct.emit(off, [&](uint32_t pos, const OrdHeadsOp::Item& it, uint32_t i, uint32_t x) { op.emit(pos, it, i, x); });
    }
    __syncthreads();  // s_w is rewritten by the next tile
  }
}

}  // namespace kvg
