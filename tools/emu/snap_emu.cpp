// snap_emu.cpp — the raw-read decode of csrc/kvg_snap.cuh compiled for the CPU from its real source on top of
// warp_emu.h, run by the launch plan kvg_scan_pci_raw and kvg_scan_mdev_raw run it by (kvg_api_snap.inc): the decode,
// then per interned column k_raw_probe and k_compact<RawInternOp>, then the pack, with the walk's traits
// (PciWalk / MdevWalk) and the argument builders of kvg_snap.cuh (raw_column, raw_intern_op, raw_pack_needed,
// raw_pack_args).  The harness keeps only its buffers and the launches.
#define KVG_HOST_EMU 1
#include <vector>
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_snap.cuh"
using namespace kvg;

template <class W>
static int emu_scan_raw(const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n, uint4* recs_out,
                        uint2* tab_out, uint64_t* hdr_out) {
  RawCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  ctrl.miss = ctrl.panic = ctrl.range = ~0ull;
  std::vector<uint2> span(2 * (size_t)n + 1);
  const RawIn in = {off, state, bytes, n};
  const unsigned grid = (n + RAW_THREADS - 1) / RAW_THREADS;
  if (n) emu_launch(W::decode, dim3(grid), RAW_THREADS, in, recs_out, span.data(), &ctrl);
  if (n && ctrl.miss == ~0ull && ctrl.panic == ~0ull) {
    std::vector<uint64_t> table(2 * raw_slots(n), 0);
    std::vector<uint32_t> slot_of(2 * (size_t)n), hnd(2 * (size_t)n, 0xdeadbeefu);
    const size_t tiles = (n + 1023) / 1024;
    std::vector<uint64_t> tile_state(tiles + 2, 0);
    const RawWork w = {table.data(), slot_of.data(), hnd.data(), tab_out};
    for (uint32_t c = 0; c < 2; c++) {
      if (!W::interned(ctrl.broken, c)) continue;
      const RawColumn col = raw_column(w, n, c);
      emu_launch(k_raw_probe, dim3(grid), RAW_THREADS, bytes, (const uint2*)span.data(), n, c, col.table, col.mask, 1u,
                 col.slot_of);
      emu_launch(k_compact<RawInternOp, 128, 8>, dim3((unsigned)tiles), 128,
                 raw_intern_op<W>(col, span.data(), n, c, &ctrl), tile_state.data(), 1u + c);
    }
    if (raw_pack_needed<W>(ctrl.broken))
      emu_launch(W::pack, dim3(grid), RAW_THREADS, raw_pack_args<W>(w, n, ctrl.broken), recs_out);
  }
  hdr_out[0] = ctrl.miss;
  hdr_out[1] = ctrl.panic;
  hdr_out[2] = ctrl.range;
  uint32_t* h = (uint32_t*)(hdr_out + 3);
  h[0] = ctrl.broken;
  h[1] = ctrl.n_names[0];
  h[2] = ctrl.n_names[1];
  return 0;
}

extern "C" {

// off [n * KVG_RAW_FIELDS + 1], state [n], bytes; recs_out [n]; tab_out [2][n] (the handle spans of the group and
// device columns); hdr_out: {miss, panic, range} as u64, then {broken, n_group_names, n_device_names} as u32.  The
// intern and pack run only when the decode found no missing read and no panic, as in the library.
int emu_scan_pci_raw(const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n, uint4* recs_out,
                     uint2* tab_out, uint64_t* hdr_out) {
  return emu_scan_raw<PciWalk>(off, state, bytes, n, recs_out, tab_out, hdr_out);
}

// off [n * KVG_MRAW_FIELDS + 1], state [n], bytes; recs_out [2 n] uint4 (the 32-byte records); tab_out [2][n] (the
// handle spans of the type and parent columns); hdr_out as emu_scan_pci_raw's: {miss, panic, range} as u64, then
// {broken, n_types, n_parent_names} as u32.
int emu_scan_mdev_raw(const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n, uint4* recs_out,
                      uint2* tab_out, uint64_t* hdr_out) {
  return emu_scan_raw<MdevWalk>(off, state, bytes, n, recs_out, tab_out, hdr_out);
}

}  // extern "C"
