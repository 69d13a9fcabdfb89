// delta_emu.cpp — K7, the re-scan delta of csrc/kvg_delta.cuh, compiled for the CPU from its real source on top of
// warp_emu.h: k_delta_merge then k_delta_lists, with the launch shapes of kvg_scan_pci_delta (kvg_api_delta.inc).
#define KVG_HOST_EMU 1
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_delta.cuh"
using namespace kvg;

extern "C" {

// prev / now: survivor lists (16-byte kvg_pci_surv).  keys: the distinct device ids now, before, the distinct groups
// now, before (u32 each, ascending) with their lengths in n_keys[4].  flags: four arrays of flag_cap tag words in the
// same order, kept by the caller across calls; tag: this call's tag (never repeated, never 0).
// changes: room for n_prev + n_now entries (2 x uint4); lists: dev_dirty, dev_gone (u16), grp_dirty, grp_gone.
// counts: {n_changes, error, the four list lengths}.
int emu_delta(const uint4* prev, uint32_t n_prev, const uint4* now, uint32_t n_now, const uint32_t* const* keys,
              const uint32_t* n_keys, uint32_t* flags, uint32_t flag_cap, uint32_t tag, uint4* changes, uint32_t* dev_dirty,
              uint16_t* dev_gone, uint32_t* grp_dirty, uint32_t* grp_gone, uint32_t* counts) {
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  const uint32_t M = n_prev + n_now;
  const uint32_t merge_tiles = M ? (M + DELTA_TILE - 1) / DELTA_TILE : 1;
  uint32_t list_tiles = 1;
  for (int k = 0; k < 4; k++) list_tiles = max(list_tiles, (n_keys[k] + C_TILE - 1) / C_TILE);
  std::vector<uint64_t> state(merge_tiles + 1 + 4 * (list_tiles + 1), 0);
  uint32_t* f[4];
  for (int k = 0; k < 4; k++) f[k] = flags + (size_t)k * flag_cap;
  DeltaMergeOp op = {};
  op.prev = prev;
  op.n_prev = n_prev;
  op.now = now;
  op.n_now = n_now;
  op.n = M;
  op.out = changes;
  op.ctrl = &ctrl;
  op.dev = {keys[0], n_keys[0], f[0], keys[1], n_keys[1], f[1]};
  op.grp = {keys[2], n_keys[2], f[2], keys[3], n_keys[3], f[3]};
  op.tag = tag;
  emu_launch(k_delta_merge, dim3(merge_tiles), DELTA_THREADS, op, state.data());
  DeltaListArgs la;
  uint32_t* cnt = &ctrl.reserved2[DELTA_W_LISTS];
  la.o[0] = {f[0], n_keys[0], tag, nullptr, dev_dirty, nullptr, cnt + 0};
  la.o[1] = {f[1], n_keys[1], tag, keys[1], nullptr, dev_gone, cnt + 1};
  la.o[2] = {f[2], n_keys[2], tag, nullptr, grp_dirty, nullptr, cnt + 2};
  la.o[3] = {f[3], n_keys[3], tag, keys[3], grp_gone, nullptr, cnt + 3};
  emu_launch(k_delta_lists, dim3(list_tiles, 4), KVG_BLOCK, la, state.data() + merge_tiles + 1, list_tiles + 1, tag + 1);
  counts[0] = ctrl.reserved2[DELTA_W_CHANGES];
  counts[1] = ctrl.reserved2[DELTA_W_ERROR];
  for (int k = 0; k < 4; k++) counts[2 + k] = cnt[k];
  return 0;
}

}  // extern "C"
