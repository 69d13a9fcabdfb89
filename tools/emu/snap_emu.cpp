// snap_emu.cpp — the raw-read decode of csrc/kvg_snap.cuh compiled for the CPU from its real source on top of
// warp_emu.h: k_raw_decode, then per column in index mode k_raw_probe and k_compact<RawInternOp>, then k_raw_pack, with
// the launch shapes and the order of kvg_scan_pci_raw (kvg_api_snap.inc); and k_mraw_decode, the type column's (and in
// index mode the parent column's) probe and compaction, then k_mraw_pack, in the order of kvg_scan_mdev_raw.
#define KVG_HOST_EMU 1
#include <vector>
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_snap.cuh"
using namespace kvg;

extern "C" {

// off [n * KVG_RAW_FIELDS + 1], state [n], bytes; recs_out [n]; tab_out [2][n] (the handle spans of the group and
// device columns); hdr_out: {miss, panic, range} as u64, then {broken, n_group_names, n_device_names} as u32.  The
// intern and pack run only when the decode found no missing read and no panic, as in the library.
int emu_scan_pci_raw(const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n, uint4* recs_out,
                     uint2* tab_out, uint64_t* hdr_out) {
  RawCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  ctrl.miss = ctrl.panic = ctrl.range = ~0ull;
  std::vector<uint2> span(2 * (size_t)n + 1);
  const RawIn in = {off, state, bytes, n};
  const unsigned grid = (n + RAW_THREADS - 1) / RAW_THREADS;
  if (n) emu_launch(k_raw_decode, dim3(grid), RAW_THREADS, in, recs_out, span.data(), &ctrl);
  if (n && ctrl.miss == ~0ull && ctrl.panic == ~0ull) {
    size_t slots = 64;
    while (slots < 2 * (size_t)n) slots <<= 1;
    std::vector<uint64_t> table(2 * slots, 0);
    std::vector<uint32_t> slot_of(2 * (size_t)n), hnd(2 * (size_t)n, 0xdeadbeefu);
    const size_t tiles = (n + 1023) / 1024;
    std::vector<uint64_t> tile_state(tiles + 2, 0);
    const bool idx[2] = {(ctrl.broken & RAW_BAD_GROUP) != 0, (ctrl.broken & RAW_BAD_DEVICE) != 0};
    RawPackArgs a = {};
    a.n = n;
    a.index_addr = (ctrl.broken & RAW_BAD_ADDR) ? 1u : 0u;
    for (uint32_t c = 0; c < 2; c++) {
      if (!idx[c]) continue;
      emu_launch(k_raw_probe, dim3(grid), RAW_THREADS, bytes, (const uint2*)span.data(), n, c, table.data() + c * slots,
                 (uint32_t)(slots - 1), 1u, slot_of.data() + (size_t)c * n);
      RawInternOp op;
      op.table = table.data() + c * slots;
      op.slot_of = slot_of.data() + (size_t)c * n;
      op.span = span.data();
      op.n = n;
      op.col = c;
      op.max_hnd = c == RAW_COL_DEVICE ? 0xffffu : 0xffffffffu;
      op.range_field = KVG_RAW_DEVICE;
      op.hnd = hnd.data() + (size_t)c * n;
      op.tab = tab_out + (size_t)c * n;
      op.ctrl = &ctrl;
      emu_launch(k_compact<RawInternOp, 128, 8>, dim3((unsigned)tiles), 128, op, tile_state.data(), 1u + c);
      a.table[c] = table.data() + c * slots;
      a.slot_of[c] = slot_of.data() + (size_t)c * n;
      a.hnd[c] = hnd.data() + (size_t)c * n;
    }
    if (ctrl.broken) emu_launch(k_raw_pack, dim3(grid), RAW_THREADS, a, recs_out);
  }
  hdr_out[0] = ctrl.miss;
  hdr_out[1] = ctrl.panic;
  hdr_out[2] = ctrl.range;
  uint32_t* w = (uint32_t*)(hdr_out + 3);
  w[0] = ctrl.broken;
  w[1] = ctrl.n_names[0];
  w[2] = ctrl.n_names[1];
  return 0;
}

// off [n * KVG_MRAW_FIELDS + 1], state [n], bytes; recs_out [2 n] uint4 (the 32-byte records); tab_out [2][n] (the
// handle spans of the type and parent columns); hdr_out as emu_scan_pci_raw's: {miss, panic, range} as u64, then
// {broken, n_types, n_parent_names} as u32.  The intern and pack run only when the decode found no missing read and no
// panic, as in the library.
int emu_scan_mdev_raw(const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n, uint4* recs_out,
                      uint2* tab_out, uint64_t* hdr_out) {
  RawCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  ctrl.miss = ctrl.panic = ctrl.range = ~0ull;
  std::vector<uint2> span(2 * (size_t)n + 1);
  const RawIn in = {off, state, bytes, n};
  const unsigned grid = (n + RAW_THREADS - 1) / RAW_THREADS;
  if (n) emu_launch(k_mraw_decode, dim3(grid), RAW_THREADS, in, recs_out, span.data(), &ctrl);
  if (n && ctrl.miss == ~0ull && ctrl.panic == ~0ull) {
    size_t slots = 64;
    while (slots < 2 * (size_t)n) slots <<= 1;
    std::vector<uint64_t> table(2 * slots, 0);
    std::vector<uint32_t> slot_of(2 * (size_t)n), hnd(2 * (size_t)n, 0xdeadbeefu);
    const size_t tiles = (n + 1023) / 1024;
    std::vector<uint64_t> tile_state(tiles + 2, 0);
    const bool idx[2] = {true, (ctrl.broken & MRAW_BAD_PARENT) != 0};
    RawPackArgs a = {};
    a.n = n;
    a.index_addr = (ctrl.broken & MRAW_BAD_UUID) ? 1u : 0u;
    for (uint32_t c = 0; c < 2; c++) {
      if (!idx[c]) continue;
      emu_launch(k_raw_probe, dim3(grid), RAW_THREADS, bytes, (const uint2*)span.data(), n, c, table.data() + c * slots,
                 (uint32_t)(slots - 1), 1u, slot_of.data() + (size_t)c * n);
      RawInternOp op;
      op.table = table.data() + c * slots;
      op.slot_of = slot_of.data() + (size_t)c * n;
      op.span = span.data();
      op.n = n;
      op.col = c;
      op.max_hnd = c == MRAW_COL_TYPE ? 65534u : 0xffffffffu;
      op.range_field = c == MRAW_COL_TYPE ? (uint32_t)KVG_MRAW_TYPE : (uint32_t)KVG_MRAW_LINK;
      op.hnd = hnd.data() + (size_t)c * n;
      op.tab = tab_out + (size_t)c * n;
      op.ctrl = &ctrl;
      emu_launch(k_compact<RawInternOp, 128, 8>, dim3((unsigned)tiles), 128, op, tile_state.data(), 1u + c);
      a.table[c] = table.data() + c * slots;
      a.slot_of[c] = slot_of.data() + (size_t)c * n;
      a.hnd[c] = hnd.data() + (size_t)c * n;
    }
    emu_launch(k_mraw_pack, dim3(grid), RAW_THREADS, a, recs_out);
  }
  hdr_out[0] = ctrl.miss;
  hdr_out[1] = ctrl.panic;
  hdr_out[2] = ctrl.range;
  uint32_t* w = (uint32_t*)(hdr_out + 3);
  w[0] = ctrl.broken;
  w[1] = ctrl.n_names[0];
  w[2] = ctrl.n_names[1];
  return 0;
}

}  // extern "C"
