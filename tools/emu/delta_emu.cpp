// delta_emu.cpp — K7, the re-scan deltas of csrc/kvg_delta.cuh, compiled for the CPU from their real source on top
// of warp_emu.h.  The launch arguments come from the builders of kvg_delta.cuh that kvg_api_delta.inc uses, in its
// launch order: k_delta_merge<PciDeltaRec> then k_delta_lists (kvg_scan_pci_delta), k_mdev_delta_types,
// k_delta_merge<MdevDeltaRec>, k_delta_lists (kvg_scan_mdev_delta), the sharded forms through
// k_delta_merge_shard<PciDeltaRec> / <MdevDeltaRec>, and kvg_scan_pci_raw_delta's k_raw_rekey, k_raw_xlate,
// k_delta_merge<PciRawDeltaRec>, k_delta_lists.
#define KVG_HOST_EMU 1
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_delta.cuh"
using namespace kvg;

namespace {
// one call: its control block and the caller's four arrays of tag words
struct Call {
  ScanCtrl ctrl{};
  uint32_t* flag[4];
  Call(uint32_t* flags, uint32_t flag_cap) {
    for (int k = 0; k < 4; k++) flag[k] = flags + (size_t)k * flag_cap;
  }
  // the merge (merge(tile_state) launches it), the lists behind it, then counts: {n_changes, error, the list lengths}
  template <class Tr, class Merge>
  void run(const DeltaMergeOp<Tr>& op, void* const (&lists)[4], bool gone0_u16, uint32_t* counts, Merge&& merge) {
    DeltaListArgs la;
    const uint32_t merge_tiles = delta_merge_tiles(op.n), list_tiles = delta_list_args(la, op, lists, gone0_u16);
    std::vector<uint64_t> state(merge_tiles + 1 + 4 * (list_tiles + 1), 0);
    merge(state.data());
    emu_launch(k_delta_lists, dim3(list_tiles, 4), KVG_BLOCK, la, state.data() + merge_tiles + 1, list_tiles + 1,
               op.tag + 1);
    counts[0] = ctrl.reserved2[DELTA_W_CHANGES];
    counts[1] = ctrl.reserved2[DELTA_W_ERROR];
    for (int k = 0; k < 4; k++) counts[2 + k] = ctrl.reserved2[DELTA_W_LISTS + k];
  }
};
}  // namespace

extern "C" {

// prev / now: survivor lists (16-byte kvg_pci_surv).  keys: the distinct device ids now, before, the distinct groups
// now, before (u32 each, ascending) with their lengths in n_keys[4].  flags: four arrays of flag_cap tag words in the
// same order, kept by the caller across calls; tag: this call's tag (never repeated, never 0).
// changes: room for n_prev + n_now entries (2 x uint4); lists: dev_dirty, dev_gone (u16), grp_dirty, grp_gone.
// counts: {n_changes, error, the four list lengths}.
int emu_delta(const uint4* prev, uint32_t n_prev, const uint4* now, uint32_t n_now, const uint32_t* const* keys,
              const uint32_t* n_keys, uint32_t* flags, uint32_t flag_cap, uint32_t tag, uint4* changes, uint32_t* dev_dirty,
              uint16_t* dev_gone, uint32_t* grp_dirty, uint32_t* grp_gone, uint32_t* counts) {
  Call c(flags, flag_cap);
  const auto op = delta_merge_op<PciDeltaRec>(prev, n_prev, now, n_now, changes, &c.ctrl, keys, n_keys, c.flag, nullptr,
                                              tag);
  c.run(op, {dev_dirty, dev_gone, grp_dirty, grp_gone}, true, counts, [&](uint64_t* state) {
    emu_launch(k_delta_merge<PciDeltaRec>, dim3(delta_merge_tiles(op.n)), DELTA_THREADS, op, state);
  });
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
  Call c(flags, flag_cap);
  const auto op = delta_merge_op<PciDeltaRec>(prev[0], n_prev[0], now[0], n_now[0], changes, &c.ctrl, keys, n_keys,
                                              c.flag, nullptr, tag);
  c.run(op, {dev_dirty, dev_gone, grp_dirty, grp_gone}, true, counts, [&](uint64_t* state) {
    DeltaShardArgs<PciDeltaRec> a;
    const uint32_t cols = delta_shard_args(a, op, {prev[1], prev[2]}, {n_prev[1], n_prev[2]}, {now[1], now[2]},
                                           {n_now[1], n_now[2]});
    emu_launch(k_delta_merge_shard<PciDeltaRec>, dim3(cols, 3), DELTA_THREADS, a, state);
  });
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
  Call c(flags, flag_cap);
  const MdevTypeLabels ln = {keys[0], n_keys[0], labels[0].bytes, labels[0].off, labels[0].len, labels[0].hash};
  const MdevTypeLabels lp = {keys[1], n_keys[1], labels[1].bytes, labels[1].off, labels[1].len, labels[1].hash};
  emu_launch(k_mdev_delta_types, dim3(1), XMAP_THREADS, ln, lp, table, delta_xmap_mask(n_keys[0]), tag, xlate);
  const auto op = delta_merge_op<MdevDeltaRec>(prev, n_prev, now, n_now, changes, &c.ctrl, keys, n_keys, c.flag, xlate,
                                               tag);
  c.run(op, {type_dirty, type_gone, par_dirty, par_gone}, false, counts, [&](uint64_t* state) {
    emu_launch(k_delta_merge<MdevDeltaRec>, dim3(delta_merge_tiles(op.n)), DELTA_THREADS, op, state);
  });
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
  Call c(flags, flag_cap);
  const MdevTypeLabels ln = {canon[0], n_canon[0], labels[0].bytes, labels[0].off, labels[0].len, labels[0].hash};
  const MdevTypeLabels lp = {canon[1], n_canon[1], labels[1].bytes, labels[1].off, labels[1].len, labels[1].hash};
  emu_launch(k_mdev_delta_types, dim3(1), XMAP_THREADS, ln, lp, table, delta_xmap_mask(n_canon[0]), tag, xlate);
  const auto op = delta_merge_op<MdevDeltaRec>(prev[0], n_prev[0], now[0], n_now[0], changes, &c.ctrl, keys, n_keys,
                                               c.flag, xlate, tag);
  c.run(op, {type_dirty, type_gone, par_dirty, par_gone}, false, counts, [&](uint64_t* state) {
    DeltaShardArgs<MdevDeltaRec> a;
    const uint32_t cols = delta_shard_args(a, op, {prev[1], prev[2]}, {n_prev[1], n_prev[2]}, {now[1], now[2]},
                                           {n_now[1], n_now[2]});
    emu_launch(k_delta_merge_shard<MdevDeltaRec>, dim3(cols, 3), DELTA_THREADS, a, state);
  });
  return 0;
}

// kvg_scan_pci_raw_delta's delta of two snapshots, chosen by raw_rekey_needed as run_raw_delta chooses: both sides
// fully numeric, the merge of emu_delta on the survivors; otherwise the re-key first, its arguments from
// raw_rekey_args as the library builds them.  sides[0] / [1]: the previous and the new side (kvg_delta.cuh
// RawDeltaSide).  table: raw_rekey_table_words of the new keys, zero before the first call; xlate: RAW_XLATE_GROUP + the previous group keys; rekeyed: room for both sides' survivors.  flags,
// tag, changes, the four lists and counts as for emu_delta; *launches: the kernels run.
int emu_pci_raw_delta(const RawDeltaSide* sides, uint64_t* table, uint32_t* xlate, uint4* rekeyed, uint32_t* flags,
                      uint32_t flag_cap, uint32_t tag, uint4* changes, uint32_t* dev_dirty, uint16_t* dev_gone,
                      uint32_t* grp_dirty, uint32_t* grp_gone, uint32_t* counts, uint32_t* launches) {
  Call c(flags, flag_cap);
  const RawDeltaSide &pv = sides[0], &nw = sides[1];
  const uint32_t* keys[4] = {nw.keys[0], pv.keys[0], nw.keys[1], pv.keys[1]};
  const uint32_t n_keys[4] = {nw.n_keys[0], pv.n_keys[0], nw.n_keys[1], pv.n_keys[1]};
  if (!raw_rekey_needed(pv.numeric, nw.numeric, RAW_NUM_ADDR | RAW_NUM_DEVICE | RAW_NUM_GROUP)) {
    const auto op = delta_merge_op<PciDeltaRec>(pv.surv, pv.n, nw.surv, nw.n, changes, &c.ctrl, keys, n_keys, c.flag,
                                                nullptr, tag);
    c.run(op, {dev_dirty, dev_gone, grp_dirty, grp_gone}, true, counts, [&](uint64_t* state) {
      emu_launch(k_delta_merge<PciDeltaRec>, dim3(delta_merge_tiles(op.n)), DELTA_THREADS, op, state);
    });
    *launches = 2;
    return 0;
  }
  uint32_t g_rekey, g_xlate;
  const RawRekeyArgs a = raw_rekey_args<false>(pv, nw, rekeyed, table, xlate, tag, &c.ctrl, &g_rekey, &g_xlate);
  emu_launch(k_raw_rekey<false>, dim3(g_rekey), REKEY_THREADS, a);
  emu_launch(k_raw_xlate<false>, dim3(g_xlate), REKEY_THREADS, a);
  auto op = delta_merge_op<PciRawDeltaRec>(a.out[0], pv.n, a.out[1], nw.n, changes, &c.ctrl, keys, n_keys, c.flag,
                                           xlate, tag);
  op.k1.xlate = xlate + RAW_XLATE_GROUP;
  c.run(op, {dev_dirty, dev_gone, grp_dirty, grp_gone}, true, counts, [&](uint64_t* state) {
    emu_launch(k_delta_merge<PciRawDeltaRec>, dim3(delta_merge_tiles(op.n)), DELTA_THREADS, op, state);
  });
  *launches = 4;
  return 0;
}

}  // extern "C"
