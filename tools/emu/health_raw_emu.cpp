// health_raw_emu.cpp — the health re-scans from raw reads of csrc/kvg_snap.cuh (kvg_health_rescan_groups_raw /
// kvg_health_rescan_mdev_raw) compiled for the CPU from their real source on top of warp_emu.h, in both launch
// shapes: k_health_raw_small<Rule> (one CTA of HEALTH_SMALL_THREADS) and k_compact<RawHealthOp<Rule>, KVG_BLOCK,
// C_ROWS> (one CTA per tile, what compact_grid() picks whenever the tiles fit the GPU).  The harness stages the set's
// strings behind the entries' bytes as the library's image does (set_off rebased onto them); the caller keeps the
// previous list (its offsets, bytes and state bytes) and adopts this call's only when nothing is refused.
#define KVG_HOST_EMU 1
#include <vector>
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_snap.cuh"
using namespace kvg;

// off [n * Rule::FIELDS + 1], state [n], bytes: this call's entries; set_off [n_set + 1], set_bytes: the set;
// prev_off / prev_bytes / prev_state [n_prev]: the previous list.  state_out [n]: this call's bytes; changed_out: room
// for n words; hdr_out (u32 x 10): {n_alive, n_changed, seq (small form; 0 otherwise), name_err} then {miss, panic,
// range} as u64.
template <class Rule>
static int health_raw(int form, const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n,
                      const uint32_t* set_off, const uint8_t* set_bytes, uint32_t n_set, const uint32_t* prev_off,
                      const uint8_t* prev_bytes, const uint8_t* prev_state, uint32_t n_prev, uint8_t* state_out,
                      uint32_t* changed_out, uint32_t* hdr_out) {
  if (n == 0 || n_set > Rule::SET_CAP || (form == 0 && n > HEALTH_SMALL_MAX)) return -1;
  const uint32_t nb = off[(size_t)n * Rule::FIELDS], set_nb = n_set ? set_off[n_set] : 0;
  std::vector<uint8_t> all(nb + set_nb + 1);
  memcpy(all.data(), bytes, nb);
  if (set_nb) memcpy(all.data() + nb, set_bytes, set_nb);
  std::vector<uint32_t> so(n_set + 1);
  for (uint32_t k = 0; k <= n_set; k++) so[k] = nb + (n_set ? set_off[k] : 0);
  RawHealthArgs a;
  a.in = {off, state, all.data(), n};
  a.set_off = so.data();
  a.n_set = n_set;
  a.prev = {prev_off, prev_bytes, prev_state, n_prev, Rule::FIELDS};
  a.state = state_out;
  if (form == 0) {
    emu_launch(k_health_raw_small<Rule>, dim3(1), HEALTH_SMALL_THREADS, a, changed_out, hdr_out, 7u);
    return 0;
  }
  const size_t tiles = (n + C_TILE - 1) / C_TILE;
  ScanCtrl sc;
  memset(&sc, 0, sizeof sc);
  RawCtrl ctrl;
  memset(&ctrl, 0, sizeof ctrl);
  ctrl.miss = ctrl.panic = ctrl.range = ~0ull;
  std::vector<uint64_t> st(tiles + 4, 0);
  emu_launch(k_compact<RawHealthOp<Rule>, KVG_BLOCK, C_ROWS>, dim3((unsigned)tiles), KVG_BLOCK,
             raw_health_op<Rule>(a, &ctrl, &sc, changed_out), st.data(), 11u);
  hdr_out[0] = sc.n_alive;
  hdr_out[1] = sc.n_changed;
  hdr_out[2] = 0;
  hdr_out[3] = sc.key_err;
  unsigned long long* v = reinterpret_cast<unsigned long long*>(hdr_out + 4);
  v[0] = ctrl.miss;
  v[1] = ctrl.panic;
  v[2] = ctrl.range;
  return 0;
}

extern "C" {

// form 0: k_health_raw_small, 1: k_compact<RawHealthOp>.  Entries in the kvg_pci_raw layout; the set = node names.
int emu_health_groups_raw(int form, const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n,
                          const uint32_t* set_off, const uint8_t* set_bytes, uint32_t n_set, const uint32_t* prev_off,
                          const uint8_t* prev_bytes, const uint8_t* prev_state, uint32_t n_prev, uint8_t* state_out,
                          uint32_t* changed_out, uint32_t* hdr_out) {
  return health_raw<GroupRawRule>(form, off, state, bytes, n, set_off, set_bytes, n_set, prev_off, prev_bytes,
                                  prev_state, n_prev, state_out, changed_out, hdr_out);
}

// Entries in the kvg_mdev_raw layout; the set = XID bus ids.
int emu_health_mdev_raw(int form, const uint32_t* off, const uint16_t* state, const uint8_t* bytes, uint32_t n,
                        const uint32_t* set_off, const uint8_t* set_bytes, uint32_t n_set, const uint32_t* prev_off,
                        const uint8_t* prev_bytes, const uint8_t* prev_state, uint32_t n_prev, uint8_t* state_out,
                        uint32_t* changed_out, uint32_t* hdr_out) {
  return health_raw<MdevRawRule>(form, off, state, bytes, n, set_off, set_bytes, n_set, prev_off, prev_bytes,
                                 prev_state, n_prev, state_out, changed_out, hdr_out);
}

}  // extern "C"
