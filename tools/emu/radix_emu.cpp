// radix_emu.cpp — K4, the stable orderings (csrc/kvg_order.cuh: k_order_hist, k_order_tilescan,
// k_order_scatter<8|11>, k_order_final and k_order_heads<0/1>), compiled for the CPU from their real source
// on top of warp_emu.h.  The launch sequence is the one of enqueue_orderings (kvg_api.cu).
#define KVG_HOST_EMU 1
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_scan.cuh"

using namespace kvg;

namespace {
struct Ordering {
  uint32_t n, max_key, key_bits_max, max_bits;
  uint32_t tile_major = 0;  // histogram layout (OrdArgs::tile_major)
  size_t T;
  std::vector<uint2> p0, p1;
  std::vector<uint32_t> hist, bins;
  Ordering(const uint2* pairs, uint32_t n_, uint32_t kbm, uint32_t mb) : n(n_), max_key(0), key_bits_max(kbm), max_bits(mb) {
    T = n ? (n + C_TILE - 1) / C_TILE : 1;
    p0.assign(n + 1, make_uint2(0xdeadbeefu, 0xdeadbeefu));
    p1.assign(n + 1, make_uint2(0xdeadbeefu, 0xdeadbeefu));
    memcpy(p1.data(), pairs, sizeof(uint2) * n);  // pass 0 reads p1 (SRC_PAIRS), like the owned-pairs path
    hist.assign((size_t)RADIX_MAX_DIGITS * T, 0xdeadbeefu);  // poisoned: nothing relies on zero-fill
    bins.assign(RADIX_MAX_DIGITS, 0xdeadbeefu);
    for (uint32_t i = 0; i < n; i++) max_key = pairs[i].x > max_key ? pairs[i].x : max_key;
  }
  int sort() {
    const int nsets = (int)((key_bits_max + max_bits - 1) / max_bits);
    for (int p = 0; p < nsets; p++) {
      OrdArgs a;
      a.n_ptr = &n;
      a.max_key = &max_key;
      a.src_records = nullptr;
      a.pairs_in = (p & 1) ? p0.data() : p1.data();
      a.pairs_out = (p & 1) ? p1.data() : p0.data();
      a.tile_hist = hist.data();
      a.bin_total = bins.data();
      a.pass = (uint32_t)p;
      a.key_bits_max = key_bits_max;
      a.max_bits = max_bits;
      a.src = SRC_PAIRS;
      a.tile_major = tile_major;
      OrdArgs2 aa;
      aa.o[0] = a;
      aa.o[1] = a;
      emu_launch(k_order_hist, dim3((unsigned)T, 1), KVG_BLOCK, aa);
      if (tile_major)
        emu_launch(k_order_tilescan_cols, dim3((1u << max_bits) / 32, 1), KVG_BLOCK, aa);
      else
        emu_launch(k_order_tilescan, dim3((1u << max_bits) / TS_WARPS, 1), TS_WARPS * 32, aa);
      if (max_bits == 8)
        emu_launch(k_order_scatter<8>, dim3((unsigned)T, 1), KVG_BLOCK, aa);
      else
        emu_launch(k_order_scatter<RADIX_MAX_BITS>, dim3((unsigned)T, 1), KVG_BLOCK, aa);
    }
    return (int)radix_plan(max_key, key_bits_max, 0, max_bits).npass;
  }
};
}  // namespace

extern "C" {

// Stable sort of {key, index} pairs the way the device does it.  pairs_io: n x {key, index}; on return the
// sorted pairs.  Returns the pass count the device-side plan chose, or a negative number.
int emu_radix_sort(uint2* pairs_io, uint32_t n, uint32_t key_bits_max, uint32_t max_bits, int variant) {
  if (max_bits != 8 && max_bits != RADIX_MAX_BITS) return -1;
  Ordering o(pairs_io, n, key_bits_max, max_bits);
  o.tile_major = variant == 1 && max_bits == RADIX_MAX_BITS ? 1u : 0u;  // variant 1: the tile-major histogram layout
  const int np = o.sort();
  memcpy(pairs_io, (((np - 1) & 1) ? o.p1 : o.p0).data(), sizeof(uint2) * n);
  return np;
}

// One whole ordering the way enqueue_orderings runs it: radix passes, then the final kernels — fused = 1:
// k_order_final (one launch, chained scan), fused = 0: k_order_heads<false> -> k_tile_offsets ->
// k_order_heads<true>.  surv: the survivor records the pairs index (head_name gathers surv[idx].w).
// Outputs: perm[n], seg_key / seg_off / seg_name [n_seg (+1 for seg_off)]; returns n_seg.
int emu_ordering(uint2* pairs_io, uint32_t n, const uint4* surv, uint32_t key_bits_max, uint32_t max_bits, uint32_t* perm,
                 uint32_t* seg_key, uint32_t* seg_off, uint32_t* seg_name, int fused, const uint32_t* join_table, int join_mode) {
  if (max_bits != 8 && max_bits != RADIX_MAX_BITS) return -1;
  Ordering o(pairs_io, n, key_bits_max, max_bits);
  o.tile_major = fused && max_bits == RADIX_MAX_BITS ? 1u : 0u;  // the latency-bound form uses the tile-major layout
  o.sort();
  const size_t T = o.T;
  std::vector<uint64_t> state(T + 2, 0);
  std::vector<uint32_t> tile_heads(T + 1, 0xdeadbeefu), tile_off(T + 2, 0xdeadbeefu);
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  ctrl.n_surv = n;
  ctrl.n_groups = 0xdeadbeefu;
  OrdFinalArgs a;
  a.p0 = o.p0.data();
  a.p1 = o.p1.data();
  a.max_key = &o.max_key;
  a.key_bits_max = key_bits_max;
  a.max_bits = max_bits;
  a.n_ptr = &o.n;
  a.perm = perm;
  a.state = state.data();
  a.tile_heads = tile_heads.data();
  a.tile_off = tile_off.data();
  a.seg_key = seg_key;
  a.seg_off = seg_off;
  a.n_seg = &ctrl.n_groups;
  a.head_surv = surv;
  a.head_name = seg_name;
  // join_mode 1 / 2: the deferred name join — `join_table` is the 65,536-entry device-id -> name-slot table and
  // every record of `surv` gets its slot (word 3) while the permutation is written; 0: names already joined
  a.join_index = join_table;
  a.join_recs = const_cast<uint4*>(surv);
  a.join = join_table ? (uint32_t)join_mode : 0u;
  OrdFinalArgs2 ff;
  ff.o[0] = a;
  ff.o[1] = a;
  if (fused) {
    emu_launch(k_order_final, dim3((unsigned)T, 1), KVG_BLOCK, ff, 9u);
  } else {
    TileOffsetsArgs2 tt;
    tt.o[0] = {tile_heads.data(), nullptr, &o.n, 0, tile_off.data(), &ctrl.n_groups, state.data()};
    tt.o[1] = tt.o[0];
    emu_launch(k_order_heads<false>, dim3((unsigned)T, 1), KVG_BLOCK, ff);
    emu_launch(k_tile_offsets, dim3((unsigned)((T + C_TILE - 1) / C_TILE), 1), KVG_BLOCK, tt, &ctrl, 9u);
    emu_launch(k_order_heads<true>, dim3((unsigned)T, 1), KVG_BLOCK, ff);
  }
  const uint32_t np = radix_plan(o.max_key, key_bits_max, 0, max_bits).npass;
  memcpy(pairs_io, (((np - 1) & 1) ? o.p1 : o.p0).data(), sizeof(uint2) * n);
  return (int)ctrl.n_groups;
}

}  // extern "C"
