// classify_emu.cpp — the record-classification pipeline of csrc/kvg_scan.cuh compiled for the CPU from
// its real source on top of warp_emu.h: the split form the large inputs and the pipelined host entry
// point use (k_classify_ragged -> k_tile_offsets -> k_pack_survivors) and the one-launch look-back form
// used below 2 M records (k_compact).  Launch shapes are those of enqueue_classify (kvg_api.cu).
#define KVG_HOST_EMU 1
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_scan.cuh"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_alloc.cuh"
using namespace kvg;

// K6, both forms of every health rule (kvg_scan.cuh) on the caller's state bytes, transitions in record order (a keyed
// rule writes its state bytes to `state`, its keys to the rule's key array).
// Small form (n <= 32,768): one CTA, transitions + counters written where the host reads them; hdr_out {n_alive,
// n_changed, seq}.  Look-back form: changed_out has room for n words; ctrl_out {n_changed, n_alive}.  Its grid is one
// CTA per tile — what compact_grid() picks whenever the tiles fit the GPU, and the only shape a sequential emulation of
// a look-back kernel can run.
template <class Rule>
static int health_small(Rule rule, const uint4* recs, uint32_t n, uint8_t* state, uint32_t* changed_out,
                        uint32_t* hdr_out, uint32_t seq) {
  if (n == 0 || n > HEALTH_SMALL_MAX) return -1;
  emu_launch(k_health_small<Rule>, dim3(1), HEALTH_SMALL_THREADS, rule, recs, n, state, changed_out, hdr_out, seq);
  return 0;
}

template <class Rule>
static int health_compact(Rule rule, const uint4* recs, uint32_t n, uint8_t* state, uint32_t* changed_out,
                          uint32_t* ctrl_out, uint32_t epoch) {
  const size_t tiles = (n + C_TILE - 1) / C_TILE;
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  std::vector<uint64_t> st(tiles + 4, 0);
  HealthOp<Rule> op;
  op.rule = rule;
  op.recs = recs;
  op.n = n;
  op.state = state;
  op.changed = changed_out;
  op.ctrl = &ctrl;
  op.set = nullptr;
  op.local_alive = 0;
  if constexpr (KEYED_RULE<Rule>) op.rule.err = &ctrl.key_err;
  emu_launch(k_compact<HealthOp<Rule>, KVG_BLOCK, C_ROWS>, dim3((unsigned)(tiles ? tiles : 1)), KVG_BLOCK, op, st.data(),
             epoch);
  ctrl_out[0] = ctrl.n_changed;
  ctrl_out[1] = ctrl.n_alive;
  if constexpr (KEYED_RULE<Rule>) ctrl_out[2] = ctrl.key_err;
  return 0;
}

// Keyed<Rule> over the previous list (prev_key, prev_state)[0..n_prev): this call's keys and state bytes go to key_out /
// state_out [n]; the caller adopts them as the next previous list only when the ascent flag (hdr_out[3] of the small
// form, ctrl_out[2] of the look-back form) is 0.
template <class Rule>
static Keyed<Rule> keyed(const Rule& base, const void* prev_key, const uint8_t* prev_state, uint32_t n_prev,
                         void* key_out) {
  Keyed<Rule> k{};
  static_cast<Rule&>(k) = base;
  k.prev_key = (const typename Keyed<Rule>::Key*)prev_key;
  k.prev_state = prev_state;
  k.n_prev = n_prev;
  k.key = (typename Keyed<Rule>::Key*)key_out;
  k.err = nullptr;
  return k;
}

extern "C" {

// recs: n x 16 B records; nv_index: 65536 name slots; surv_out: room for n survivors.
// variant 0 = ragged / offsets / pack, 1 = one-launch look-back.  ctrl_out: {n_surv, max_group, max_devkey}.
int emu_classify_pci(const uint4* recs, uint32_t n, const uint32_t* nv_index, int variant, uint4* surv_out,
                     uint32_t* ctrl_out) {
  constexpr int T = 128, R = 8;
  const size_t tiles = (n + (size_t)T * R - 1) / ((size_t)T * R);
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  std::vector<uint4> ragged((tiles + 1) * T * R, uint4{0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu});
  std::vector<uint32_t> tile_count(tiles + 2, 0xdeadbeefu), tile_off(tiles + 3, 0xdeadbeefu);
  std::vector<uint2> tile_max(tiles + 2);
  std::vector<uint64_t> state(tiles + 4, 0);
  PciClassifyOp op;
  op.recs = recs;
  op.n = n;
  op.ctrl = &ctrl;
  op.nv_index = nv_index;
  const uint32_t epoch = 7;
  if (variant == 1) {
    op.out = surv_out;
    emu_launch(k_compact<PciClassifyOp, T, R>, dim3((unsigned)(tiles ? tiles : 1)), T, op, state.data(), epoch);
  } else if (tiles) {
    op.out = ragged.data();
    emu_launch(k_classify_ragged<PciClassifyOp, T, R>, dim3((unsigned)tiles), T, op, tile_count.data(), tile_max.data());
    TileOffsetsArgs2 tt;
    tt.o[0] = {tile_count.data(), tile_max.data(), nullptr, (uint32_t)tiles, tile_off.data(), &ctrl.n_surv, state.data()};
    tt.o[1] = tt.o[0];
    emu_launch(k_tile_offsets, dim3((unsigned)((tiles + C_TILE - 1) / C_TILE)), KVG_BLOCK, tt, &ctrl, epoch);
    emu_launch(k_pack_survivors<1>, dim3((unsigned)tiles), 128, (const uint4*)ragged.data(),
               (const uint32_t*)tile_off.data(), (uint32_t)(T * R), surv_out);
  }
  ctrl_out[0] = ctrl.n_surv;
  ctrl_out[1] = ctrl.max_group;
  ctrl_out[2] = ctrl.max_devkey;
  return 0;
}

// K6 (kvg_health_rescan): alive-set diff against the previous scan.  recs: n x 16 B records.
int emu_health_rescan(const uint4* recs, uint32_t n, uint8_t* alive_prev, uint32_t* changed_out, uint32_t* ctrl_out) {
  return health_compact(PciHealthRule{}, recs, n, alive_prev, changed_out, ctrl_out, 11u);
}

int emu_health_small(const uint4* recs, uint32_t n, uint8_t* alive_prev, uint32_t* changed_out, uint32_t* hdr_out) {
  return health_small(PciHealthRule{}, recs, n, alive_prev, changed_out, hdr_out, 7u);
}

// K6 for vGPUs (kvg_health_rescan_mdev): state bit 0 healthy, bit 1 marked.  recs: n x 32 B records; xid: the sorted,
// deduplicated parent handles.
int emu_health_mdev_small(const uint4* recs, uint32_t n, uint32_t n_types, const uint32_t* xid, uint32_t n_xid,
                          uint8_t* state, uint32_t* changed_out, uint32_t* hdr_out) {
  if (n_xid > KVG_HEALTH_MAX_XID) return -1;
  return health_small(MdevHealthRule{xid, n_xid, n_types}, recs, n, state, changed_out, hdr_out, 9u);
}

int emu_health_mdev_compact(const uint4* recs, uint32_t n, uint32_t n_types, const uint32_t* xid, uint32_t n_xid,
                            uint8_t* state, uint32_t* changed_out, uint32_t* ctrl_out) {
  if (n_xid > KVG_HEALTH_MAX_XID) return -1;
  return health_compact(MdevHealthRule{xid, n_xid, n_types}, recs, n, state, changed_out, ctrl_out, 13u);
}

// The keyed vGPU re-scan (kvg_health_rescan_mdev_keyed): keys = the UUIDs (16 bytes each).  small: hdr_out {n_alive,
// n_changed, seq, ascent flag}; compact: ctrl_out {n_changed, n_alive, ascent flag}.
int emu_health_mdev_keyed_small(const uint4* recs, uint32_t n, uint32_t n_types, const uint32_t* xid, uint32_t n_xid,
                                const uint4* prev_key, const uint8_t* prev_state, uint32_t n_prev, uint4* key_out,
                                uint8_t* state_out, uint32_t* changed_out, uint32_t* hdr_out) {
  if (n_xid > KVG_HEALTH_MAX_XID) return -1;
  return health_small(keyed(MdevHealthRule{xid, n_xid, n_types}, prev_key, prev_state, n_prev, key_out), recs, n,
                      state_out, changed_out, hdr_out, 19u);
}

int emu_health_mdev_keyed_compact(const uint4* recs, uint32_t n, uint32_t n_types, const uint32_t* xid, uint32_t n_xid,
                                  const uint4* prev_key, const uint8_t* prev_state, uint32_t n_prev, uint4* key_out,
                                  uint8_t* state_out, uint32_t* changed_out, uint32_t* ctrl_out) {
  if (n_xid > KVG_HEALTH_MAX_XID) return -1;
  return health_compact(keyed(MdevHealthRule{xid, n_xid, n_types}, prev_key, prev_state, n_prev, key_out), recs, n,
                        state_out, changed_out, ctrl_out, 23u);
}

// K6 for passthrough GPUs by IOMMU group (kvg_health_rescan_groups): state = healthy bit.  recs: n x 16 B records;
// groups: the sorted, deduplicated handles of the groups whose node exists.
int emu_health_groups_small(const uint4* recs, uint32_t n, const uint32_t* groups, uint32_t n_groups, uint8_t* state,
                            uint32_t* changed_out, uint32_t* hdr_out) {
  if (n_groups > KVG_HEALTH_MAX_GROUPS) return -1;
  return health_small(GroupHealthRule{groups, n_groups}, recs, n, state, changed_out, hdr_out, 5u);
}

int emu_health_groups_compact(const uint4* recs, uint32_t n, const uint32_t* groups, uint32_t n_groups, uint8_t* state,
                              uint32_t* changed_out, uint32_t* ctrl_out) {
  if (n_groups > KVG_HEALTH_MAX_GROUPS) return -1;
  return health_compact(GroupHealthRule{groups, n_groups}, recs, n, state, changed_out, ctrl_out, 17u);
}

// The keyed group re-scan (kvg_health_rescan_groups_keyed): keys = the addresses.  Outputs as the keyed vGPU form's.
int emu_health_groups_keyed_small(const uint4* recs, uint32_t n, const uint32_t* groups, uint32_t n_groups,
                                  const uint32_t* prev_key, const uint8_t* prev_state, uint32_t n_prev, uint32_t* key_out,
                                  uint8_t* state_out, uint32_t* changed_out, uint32_t* hdr_out) {
  if (n_groups > KVG_HEALTH_MAX_GROUPS) return -1;
  return health_small(keyed(GroupHealthRule{groups, n_groups}, prev_key, prev_state, n_prev, key_out), recs, n,
                      state_out, changed_out, hdr_out, 29u);
}

int emu_health_groups_keyed_compact(const uint4* recs, uint32_t n, const uint32_t* groups, uint32_t n_groups,
                                    const uint32_t* prev_key, const uint8_t* prev_state, uint32_t n_prev,
                                    uint32_t* key_out, uint8_t* state_out, uint32_t* changed_out, uint32_t* ctrl_out) {
  if (n_groups > KVG_HEALTH_MAX_GROUPS) return -1;
  return health_compact(keyed(GroupHealthRule{groups, n_groups}, prev_key, prev_state, n_prev, key_out), recs, n,
                        state_out, changed_out, ctrl_out, 31u);
}

// K5 (kvg_dev_scan_mdev up to the survivor list): type dictionary -> labels -> canonical ids, then the
// 32-byte mdev records through k_classify_ragged<MdevClassifyOp,128,4> -> k_tile_offsets -> k_pack_survivors<2>.
// raw / raw_off: the dictionary blob with n_types+1 offsets.  Outputs: label bytes per entry (at raw_off),
// label_len, canon; surv_out: 2 x uint4 per survivor; ctrl_out: {n_surv, max_parent, max_type}.
int emu_scan_mdev(const uint4* recs, uint32_t n, const uint8_t* raw, const uint32_t* raw_off, uint32_t n_types, uint8_t* label,
                  uint32_t* label_len, uint16_t* canon, uint4* surv_out, uint32_t* ctrl_out) {
  std::vector<uint64_t> label_hash(n_types + 1);
  if (n_types) {
    emu_launch(k_mdev_labels, dim3((n_types + 127) / 128), 128, raw, raw_off, n_types, label, label_len, label_hash.data());
    emu_launch(k_mdev_canon, dim3((n_types + 127) / 128), 128, (const uint8_t*)label, raw_off, (const uint32_t*)label_len,
               (const uint64_t*)label_hash.data(), n_types, canon);
  }
  constexpr int T = 128, R = 4;
  const size_t tiles = (n + (size_t)T * R - 1) / ((size_t)T * R);
  ScanCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  std::vector<uint4> ragged(2 * (tiles + 1) * T * R);
  std::vector<uint32_t> tile_count(tiles + 2), tile_off(tiles + 3);
  std::vector<uint2> tile_max(tiles + 2);
  std::vector<uint64_t> state(tiles + 4, 0);
  MdevClassifyOp op;
  op.recs = recs;
  op.n = n;
  op.out = ragged.data();
  op.ctrl = &ctrl;
  op.type_canon = canon;
  op.n_types = n_types;
  if (tiles) {
    emu_launch(k_classify_ragged<MdevClassifyOp, T, R>, dim3((unsigned)tiles), T, op, tile_count.data(), tile_max.data());
    TileOffsetsArgs2 tt;
    tt.o[0] = {tile_count.data(), tile_max.data(), nullptr, (uint32_t)tiles, tile_off.data(), &ctrl.n_surv, state.data()};
    tt.o[1] = tt.o[0];
    emu_launch(k_tile_offsets, dim3((unsigned)((tiles + C_TILE - 1) / C_TILE)), KVG_BLOCK, tt, &ctrl, 13u);
    emu_launch(k_pack_survivors<2>, dim3((unsigned)tiles), 128, (const uint4*)ragged.data(),
               (const uint32_t*)tile_off.data(), (uint32_t)(T * R), surv_out);
  }
  ctrl_out[0] = ctrl.n_surv;
  ctrl_out[1] = ctrl.max_group;
  ctrl_out[2] = ctrl.max_devkey;
  return 0;
}

// kvg_mdev_label_match's kernel in its launch shape (one CTA of LABEL_MATCH_THREADS): raw / raw_off: n files with n+1
// offsets; name: min(name_len, raw_off[n]) bytes.  match_out: n bytes; seq_out: the sequence word (7 when done).
int emu_mdev_label_match(const uint8_t* raw, const uint32_t* raw_off, uint32_t n, const uint8_t* name, uint64_t name_len,
                         uint8_t* match_out, uint32_t* seq_out) {
  if (n == 0) return -1;
  emu_launch(k_mdev_label_match, dim3(1), LABEL_MATCH_THREADS, raw, raw_off, n, name, name_len, match_out, seq_out, 7u);
  return 0;
}

// kvg_pci_allocate_check's kernel in its launch shape (min(n_reqs, ALLOC_CHECK_MAX_GRID) CTAs of GROUP_CHECK_THREADS):
// reqs: n_reqs x {n_members, n_ids}; recs / want: the requests' members one after another; ids: their EGM handles;
// egm_off: n_egm + 1 offsets into egm_gpu.  first_bad_out: n_reqs words; take_out: n_reqs x n_egm bytes; seq_out: the
// sequence word (7 when done).  The request table comes from allocate_check_reqs (kvg_scan.cuh), as in the library;
// the CTA counter is the harness's.
int emu_pci_allocate_check(const uint32_t* reqs, uint32_t n_reqs, const uint4* recs, const uint32_t* want,
                           const uint32_t* ids, const uint32_t* egm_off, const uint32_t* egm_gpu, uint32_t n_egm,
                           uint32_t n_egm_gpus, uint32_t* first_bad_out, uint8_t* take_out, uint32_t* seq_out) {
  if (n_reqs == 0) return -1;
  std::vector<uint4> req(n_reqs);
  allocate_check_reqs((const kvg_alloc_req*)reqs, n_reqs, req.data());
  uint32_t done = 0;
  const uint32_t grid = std::min(n_reqs, ALLOC_CHECK_MAX_GRID);
  emu_launch(k_pci_allocate_check, dim3(grid), GROUP_CHECK_THREADS, (const uint4*)req.data(), recs, want, ids, egm_off,
             egm_gpu, n_reqs, n_egm, n_egm_gpus, &done, first_bad_out, take_out, seq_out, 7u);
  return done == grid ? 0 : -2;
}

// kvg_pci_group_check's launch: k_pci_allocate_check with one request and no EGM device.  recs: n x 16 B records;
// want: n group handles.  first_bad_out: the smallest failing index, or n; seq_out: the sequence word (7 when done).
int emu_pci_group_check(const uint4* recs, const uint32_t* want, uint32_t n, uint32_t* first_bad_out,
                        uint32_t* seq_out) {
  if (n == 0) return -1;
  const uint32_t req[2] = {n, 0};
  return emu_pci_allocate_check(req, 1, recs, want, nullptr, nullptr, nullptr, 0, 0, first_bad_out, nullptr, seq_out);
}

// kvg_preferred_allocation's kernel in its launch shape (min(n_reqs, PREF_MAX_GRID) CTAs of PREF_THREADS): reqs: n_reqs x
// {n_must, n_avail, size, pad}; ids: n_ids x {handle, node}, the requests' entries one after another.  res_out: n_out,
// P per request; pos_out: room for n_ids picks, request r's from its first entry; seq_out: the sequence word (7 when
// done).  The scratch, the CTA counter and the request offsets are the harness's, as the library's are its own.
int emu_preferred_allocation(const uint4* reqs, uint32_t n_reqs, const uint2* ids, uint32_t n_ids, uint32_t* res_out,
                             uint32_t* pos_out, uint32_t* seq_out) {
  if (n_reqs == 0) return -1;
  std::vector<uint32_t> off(n_reqs);
  for (uint32_t r = 0, a = 0; r < n_reqs; r++) {
    off[r] = a;
    a += reqs[r].x + reqs[r].y;
  }
  std::vector<uint32_t> scratch(pref_scratch_words(n_ids, n_reqs), 0xa5a5a5a5u);  // every CTA initialises its slice
  uint32_t done = 0;
  emu_launch(k_preferred_alloc, dim3(std::min(n_reqs, PREF_MAX_GRID)), PREF_THREADS, reqs, (const uint32_t*)off.data(),
             ids, n_reqs, n_ids, scratch.data(), &done, res_out, pos_out, seq_out, 7u);
  return done == std::min(n_reqs, PREF_MAX_GRID) ? 0 : -2;
}

}  // extern "C"
