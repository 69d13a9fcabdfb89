// delta_emu.cpp — K7, the re-scan deltas of csrc/kvg_delta.cuh, compiled for the CPU from their real source on top
// of warp_emu.h, with the launch shapes of kvg_api_delta.inc: k_delta_merge<PciDeltaRec> then k_delta_lists
// (kvg_scan_pci_delta), k_mdev_delta_types, k_delta_merge<MdevDeltaRec>, k_delta_lists (kvg_scan_mdev_delta), and the
// sharded forms through k_delta_merge_shard<PciDeltaRec> / <MdevDeltaRec>.
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
  DeltaMergeOp<PciDeltaRec> op = {};
  op.prev = prev;
  op.n_prev = n_prev;
  op.now = now;
  op.n_now = n_now;
  op.n = M;
  op.out = changes;
  op.ctrl = &ctrl;
  op.k0 = {keys[0], n_keys[0], f[0], keys[1], n_keys[1], f[1], nullptr};
  op.k1 = {keys[2], n_keys[2], f[2], keys[3], n_keys[3], f[3], nullptr};
  op.tag = tag;
  emu_launch(k_delta_merge<PciDeltaRec>, dim3(merge_tiles), DELTA_THREADS, op, state.data());
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

// One rank of the sharded delta.  prev[y] / now[y] with n_prev[y] / n_now[y] entries (16-byte kvg_pci_surv, Walk
// order): y = 0 the local survivors, 1 the members of the owned device ids, 2 the members of the owned groups.  keys:
// the owned device ids now, before, the owned groups now, before.  flags, tag, changes (room for n_prev[0] +
// n_now[0] entries), the four lists and counts as for emu_delta.
int emu_shard_delta(const uint4* const* prev, const uint32_t* n_prev, const uint4* const* now, const uint32_t* n_now,
                    const uint32_t* const* keys, const uint32_t* n_keys, uint32_t* flags, uint32_t flag_cap,
                    uint32_t tag, uint4* changes, uint32_t* dev_dirty, uint16_t* dev_gone, uint32_t* grp_dirty,
                    uint32_t* grp_gone, uint32_t* counts) {
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  const uint32_t M = n_prev[0] + n_now[0];
  const uint32_t merge_tiles = M ? (M + DELTA_TILE - 1) / DELTA_TILE : 1;
  uint32_t list_tiles = 1;
  for (int k = 0; k < 4; k++) list_tiles = max(list_tiles, (n_keys[k] + C_TILE - 1) / C_TILE);
  std::vector<uint64_t> state(merge_tiles + 1 + 4 * (list_tiles + 1), 0);
  uint32_t* f[4];
  for (int k = 0; k < 4; k++) f[k] = flags + (size_t)k * flag_cap;
  DeltaShardArgs<PciDeltaRec> a;
  uint32_t cols = merge_tiles;
  for (int y = 0; y < 3; y++) {
    DeltaMergeOp<PciDeltaRec>& o = a.o[y];
    o = {};
    o.prev = prev[y];
    o.n_prev = n_prev[y];
    o.now = now[y];
    o.n_now = n_now[y];
    o.n = n_prev[y] + n_now[y];
    o.out = y == 0 ? changes : nullptr;
    o.ctrl = &ctrl;
    if (y == 1) o.k0 = {keys[0], n_keys[0], f[0], keys[1], n_keys[1], f[1], nullptr};
    if (y == 2) o.k1 = {keys[2], n_keys[2], f[2], keys[3], n_keys[3], f[3], nullptr};
    o.tag = tag;
    cols = max(cols, (o.n + DELTA_TILE - 1) / DELTA_TILE);
  }
  emu_launch(k_delta_merge_shard<PciDeltaRec>, dim3(cols, 3), DELTA_THREADS, a, state.data());
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

// prev / now: survivor lists (32-byte kvg_mdev_surv).  keys: the distinct type ids now, before, the distinct parents
// now, before (u32 each, ascending) with their lengths in n_keys[4].  labels[0] / [1]: the new / previous dictionary
// (label bytes, offsets, lengths, FNV-1a hashes, indexed by canonical id).  table: XMAP_SLOTS words and xlate: 65,536
// words kept by the caller across calls, like flags.  changes: room for n_prev + n_now entries (3 x uint4); lists:
// type_dirty, type_gone (previous canonical ids), par_dirty, par_gone.  counts: as for emu_delta.
struct EmuLabels {
  const uint8_t* bytes;
  const uint32_t* off;
  const uint32_t* len;
  const uint64_t* hash;
};
int emu_mdev_delta(const uint4* prev, uint32_t n_prev, const uint4* now, uint32_t n_now, const uint32_t* const* keys,
                   const uint32_t* n_keys, const EmuLabels* labels, uint64_t* table, uint32_t* xlate, uint32_t* flags,
                   uint32_t flag_cap, uint32_t tag, uint4* changes, uint32_t* type_dirty, uint32_t* type_gone,
                   uint32_t* par_dirty, uint32_t* par_gone, uint32_t* counts) {
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  uint32_t slots = 64;
  while (slots < 2 * n_keys[0]) slots <<= 1;
  const MdevTypeLabels ln = {keys[0], n_keys[0], labels[0].bytes, labels[0].off, labels[0].len, labels[0].hash};
  const MdevTypeLabels lp = {keys[1], n_keys[1], labels[1].bytes, labels[1].off, labels[1].len, labels[1].hash};
  emu_launch(k_mdev_delta_types, dim3(1), XMAP_THREADS, ln, lp, table, slots - 1, tag, xlate);
  const uint32_t M = n_prev + n_now;
  const uint32_t merge_tiles = M ? (M + DELTA_TILE - 1) / DELTA_TILE : 1;
  uint32_t list_tiles = 1;
  for (int k = 0; k < 4; k++) list_tiles = max(list_tiles, (n_keys[k] + C_TILE - 1) / C_TILE);
  std::vector<uint64_t> state(merge_tiles + 1 + 4 * (list_tiles + 1), 0);
  uint32_t* f[4];
  for (int k = 0; k < 4; k++) f[k] = flags + (size_t)k * flag_cap;
  DeltaMergeOp<MdevDeltaRec> op = {};
  op.prev = reinterpret_cast<const MdevItem*>(prev);
  op.n_prev = n_prev;
  op.now = reinterpret_cast<const MdevItem*>(now);
  op.n_now = n_now;
  op.n = M;
  op.out = changes;
  op.ctrl = &ctrl;
  op.k0 = {keys[0], n_keys[0], f[0], keys[1], n_keys[1], f[1], xlate};
  op.k1 = {keys[2], n_keys[2], f[2], keys[3], n_keys[3], f[3], nullptr};
  op.tag = tag;
  emu_launch(k_delta_merge<MdevDeltaRec>, dim3(merge_tiles), DELTA_THREADS, op, state.data());
  DeltaListArgs la;
  uint32_t* cnt = &ctrl.reserved2[DELTA_W_LISTS];
  la.o[0] = {f[0], n_keys[0], tag, nullptr, type_dirty, nullptr, cnt + 0};
  la.o[1] = {f[1], n_keys[1], tag, keys[1], type_gone, nullptr, cnt + 1};
  la.o[2] = {f[2], n_keys[2], tag, nullptr, par_dirty, nullptr, cnt + 2};
  la.o[3] = {f[3], n_keys[3], tag, keys[3], par_gone, nullptr, cnt + 3};
  emu_launch(k_delta_lists, dim3(list_tiles, 4), KVG_BLOCK, la, state.data() + merge_tiles + 1, list_tiles + 1, tag + 1);
  counts[0] = ctrl.reserved2[DELTA_W_CHANGES];
  counts[1] = ctrl.reserved2[DELTA_W_ERROR];
  for (int k = 0; k < 4; k++) counts[2 + k] = cnt[k];
  return 0;
}

// One rank of the sharded mdev delta (kvg_dev_scan_mdev_shard_fetch_delta).  prev[y] / now[y] with n_prev[y] /
// n_now[y] entries (32-byte kvg_mdev_surv, Walk order): y = 0 the local survivors, 1 the members of the owned type ids,
// 2 the members of the owned parents.  keys: the owned type ids now, before, the owned parents now, before.  canon[0] /
// [1] with n_canon[2]: every canonical id of the new / previous dictionary (what k_mdev_delta_types translates).
// labels, table, xlate, flags, tag, changes (room for n_prev[0] + n_now[0] entries), the four lists and counts as for
// emu_mdev_delta.
int emu_mdev_shard_delta(const uint4* const* prev, const uint32_t* n_prev, const uint4* const* now,
                         const uint32_t* n_now, const uint32_t* const* keys, const uint32_t* n_keys,
                         const uint32_t* const* canon, const uint32_t* n_canon, const EmuLabels* labels,
                         uint64_t* table, uint32_t* xlate, uint32_t* flags, uint32_t flag_cap, uint32_t tag,
                         uint4* changes, uint32_t* type_dirty, uint32_t* type_gone, uint32_t* par_dirty,
                         uint32_t* par_gone, uint32_t* counts) {
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  uint32_t slots = 64;
  while (slots < 2 * n_canon[0]) slots <<= 1;
  const MdevTypeLabels ln = {canon[0], n_canon[0], labels[0].bytes, labels[0].off, labels[0].len, labels[0].hash};
  const MdevTypeLabels lp = {canon[1], n_canon[1], labels[1].bytes, labels[1].off, labels[1].len, labels[1].hash};
  emu_launch(k_mdev_delta_types, dim3(1), XMAP_THREADS, ln, lp, table, slots - 1, tag, xlate);
  const uint32_t M = n_prev[0] + n_now[0];
  const uint32_t merge_tiles = M ? (M + DELTA_TILE - 1) / DELTA_TILE : 1;
  uint32_t list_tiles = 1;
  for (int k = 0; k < 4; k++) list_tiles = max(list_tiles, (n_keys[k] + C_TILE - 1) / C_TILE);
  std::vector<uint64_t> state(merge_tiles + 1 + 4 * (list_tiles + 1), 0);
  uint32_t* f[4];
  for (int k = 0; k < 4; k++) f[k] = flags + (size_t)k * flag_cap;
  const DeltaKeys xlate_only = {nullptr, 0, nullptr, nullptr, 0, nullptr, xlate};
  DeltaShardArgs<MdevDeltaRec> a;
  uint32_t cols = merge_tiles;
  for (int y = 0; y < 3; y++) {
    DeltaMergeOp<MdevDeltaRec>& o = a.o[y];
    o = {};
    o.prev = reinterpret_cast<const MdevItem*>(prev[y]);
    o.n_prev = n_prev[y];
    o.now = reinterpret_cast<const MdevItem*>(now[y]);
    o.n_now = n_now[y];
    o.n = n_prev[y] + n_now[y];
    o.out = y == 0 ? changes : nullptr;
    o.ctrl = &ctrl;
    o.k0 = y == 1 ? DeltaKeys{keys[0], n_keys[0], f[0], keys[1], n_keys[1], f[1], xlate} : xlate_only;
    if (y == 2) o.k1 = {keys[2], n_keys[2], f[2], keys[3], n_keys[3], f[3], nullptr};
    o.tag = tag;
    cols = max(cols, (o.n + DELTA_TILE - 1) / DELTA_TILE);
  }
  emu_launch(k_delta_merge_shard<MdevDeltaRec>, dim3(cols, 3), DELTA_THREADS, a, state.data());
  DeltaListArgs la;
  uint32_t* cnt = &ctrl.reserved2[DELTA_W_LISTS];
  la.o[0] = {f[0], n_keys[0], tag, nullptr, type_dirty, nullptr, cnt + 0};
  la.o[1] = {f[1], n_keys[1], tag, keys[1], type_gone, nullptr, cnt + 1};
  la.o[2] = {f[2], n_keys[2], tag, nullptr, par_dirty, nullptr, cnt + 2};
  la.o[3] = {f[3], n_keys[3], tag, keys[3], par_gone, nullptr, cnt + 3};
  emu_launch(k_delta_lists, dim3(list_tiles, 4), KVG_BLOCK, la, state.data() + merge_tiles + 1, list_tiles + 1, tag + 1);
  counts[0] = ctrl.reserved2[DELTA_W_CHANGES];
  counts[1] = ctrl.reserved2[DELTA_W_ERROR];
  for (int k = 0; k < 4; k++) counts[2 + k] = cnt[k];
  return 0;
}

}  // extern "C"
