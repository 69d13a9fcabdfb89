// names_emu.cpp — getDeviceName end to end from kernel source on the CPU: K1 (csrc/kvg_parse_k1.cuh:
// scan with the per-warp TMA ring -> resolve + finalize -> names) followed by the lookup path of
// csrc/kvg_parse.cuh exactly as the library sequences it (kvg_api.cu: parse_enqueue, table_publish,
// kvg_name_lookup, lookup_general):
//   table path     nv_index[id] -> pool[slot] = u16 length + bytes        (4-lower-hex keys)
//   general path   k_section_lines -> k_lookup_general -> k_sanitise_matches   (every other key)
#define KVG_HOST_EMU 1
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_parse_k1.cuh"
using namespace kvg;

// K1 sequenced as parse_enqueue does (no clearing launch: dev_off all NONE and info all zero is the state a fresh
// allocation is given once, and the state every parse leaves behind).  scan_ctas = grid of the persistent scan kernel (0: one warp per
// span).  nv_index / pool may be NULL (then the names kernel is skipped).
static void run_k1(const uint8_t* text, uint64_t stride, uint32_t len, uint32_t n_files, uint32_t scan_ctas,
                   uint32_t* dev_off, PciIdsInfo* info, uint32_t* nv_index, uint8_t* pool, uint32_t pool16) {
  const uint32_t spf = (len + K1_SPAN - 1) / K1_SPAN, n_spans = spf * n_files;
  std::vector<uint4> sums(n_spans + 1, make_uint4(0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu));  // poisoned
  K1Args A;
  A.text = text;
  A.stride = stride;
  A.len = len;
  A.n_files = n_files;
  A.spans_per_file = spf;
  A.n_spans = n_spans;
  A.dev_off = dev_off;
  A.info = info;
  A.span_sum = sums.data();
  A.pool = (uint4*)pool;
  A.pool16 = pool16;
  unsigned grid = (n_spans + K1_WARPS - 1) / K1_WARPS;
  if (scan_ctas && scan_ctas < grid) grid = scan_ctas;
  if (n_spans) emu_launch(k_pciids_scan, dim3(grid), K1_WARPS * 32, A);
  emu_launch(k_pciids_resolve_finalize, dim3(n_files + (n_spans + K1_RWARPS - 1) / K1_RWARPS), KVG_BLOCK, A);
  if (nv_index)
    emu_launch(k_pciids_names, dim3(K1_NAME_CTAS + (n_files > 1 ? 3 : 0)), KVG_BLOCK, dev_off, n_files, text, len, info, nv_index, pool);
}

static bool canonical_key(const uint8_t* k, uint32_t n, uint32_t* v) {  // kvg_api.cu: 4 lower-case hex digits
  if (n != 4) return false;
  uint32_t x = 0;
  for (int i = 0; i < 4; i++) {
    uint32_t h = hexval(k[i]);
    if (h > 15) return false;
    x = (x << 4) | h;
  }
  *v = x;
  return true;
}

extern "C" {

// K1 alone: n_files images (text + f*stride); outputs per image info[8 words] and the device-id table
int emu_parse_k1(const uint8_t* text, uint64_t stride, uint32_t len, uint32_t n_files, uint32_t scan_ctas,
                 uint32_t* info_out, uint32_t* dev_off_out) {
  std::vector<uint32_t> dev_off((size_t)K1_IDS * n_files, P_NONE);  // the state of a fresh allocation
  std::vector<PciIdsInfo> info(n_files);
  memset(info.data(), 0, sizeof(PciIdsInfo) * n_files);
  run_k1(text, stride, len, n_files, scan_ctas, dev_off.data(), info.data(), nullptr, nullptr, 0);
  memcpy(info_out, info.data(), sizeof(PciIdsInfo) * n_files);
  memcpy(dev_off_out, dev_off.data(), sizeof(uint32_t) * dev_off.size());
  // the names kernel leaves EVERY image's table clean for the next parse (image 0 by the name CTAs, the others
  // by the cleaning CTAs)
  std::vector<uint32_t> nv_index(K1_IDS, 0x77777777u);
  std::vector<uint8_t> pool(((size_t)len + 16 + 15) & ~(size_t)15, 0);
  emu_launch(k_pciids_names, dim3(K1_NAME_CTAS + (n_files > 1 ? 3 : 0)), KVG_BLOCK, dev_off.data(), n_files, text, len, info.data(),
             nv_index.data(), pool.data());
  for (uint32_t v : dev_off)
    if (v != P_NONE) return 10;
  return 0;
}

// text: one image padded like kvg_text_pad.  keys: blob + n_keys+1 offsets.  names_out: n_keys x name_cap
// bytes, names_len: n_keys.  Returns 0.
int emu_get_device_names(const uint8_t* text, uint32_t len, const uint8_t* keys, const uint32_t* key_off, uint32_t n_keys,
                         uint8_t* names_out, uint32_t name_cap, uint32_t* names_len, uint32_t* info_out,
                         uint32_t* nv_index_out, uint8_t* pool_out, uint32_t pool_cap, uint32_t* pool_len) {
  PciIdsInfo info;
  memset(&info, 0, sizeof info);
  const uint32_t pool_bytes = (len + 16 + 15) & ~15u;
  std::vector<uint32_t> dev_off(K1_IDS, P_NONE), nv_index(K1_IDS, 0x77777777u);  // nv_index / pool: poisoned, K1 writes them whole
  std::vector<uint8_t> k1_pool(pool_bytes, 0xee);
  // twice on the same buffers: the second parse starts from what the first one left behind (self-cleaning table,
  // accumulators consumed by the finalize CTA) and must produce the same table
  std::vector<uint32_t> nv_first;
  std::vector<uint8_t> pool_first;
  PciIdsInfo info_first;
  for (int rep = 0; rep < 2; rep++) {
    run_k1(text, 0, len, 1, 3, dev_off.data(), &info, nv_index.data(), k1_pool.data(), pool_bytes / 16);
    for (uint32_t v : dev_off)
      if (v != P_NONE) return 10;  // a slot survived k_pciids_names
    if (info.pad[0] || info.pad[1]) return 11;
    if (rep == 0) {
      nv_first = nv_index;
      pool_first = k1_pool;
      info_first = info;
      std::fill(nv_index.begin(), nv_index.end(), 0x77777777u);
      std::fill(k1_pool.begin(), k1_pool.end(), 0xee);
    } else if (nv_first != nv_index || pool_first != k1_pool || memcmp(&info_first, &info, sizeof info)) {
      return 12;
    }
  }
  memcpy(info_out, &info, sizeof info);
  // ---- table_publish: the host mirrors sec + 16 bytes of the pool; the general lookup's candidate lines
  const size_t sec = info.v_off == P_NONE ? 0 : (size_t)info.sec_end - info.v_off;
  std::vector<uint8_t> pool(sec + 16, 0);
  memcpy(pool.data(), k1_pool.data(), std::min(pool.size(), k1_pool.size()));
  const uint32_t sec_cap = (uint32_t)(sec / 2 + 8);
  std::vector<uint32_t> sec_lines(sec_cap + 1, 0);
  if (sec)
    emu_launch(k_section_lines, dim3(8), KVG_BLOCK, text, (const PciIdsInfo*)&info, sec_lines.data(), sec_lines.data() + sec_cap,
               sec_cap);
  if (nv_index_out) {   // table export for the end-to-end scan test: what the scans join against
    memcpy(nv_index_out, nv_index.data(), sizeof(uint32_t) * 65536);
    if (pool.size() > pool_cap) return 3;
    memcpy(pool_out, pool.data(), pool.size());
    *pool_len = (uint32_t)pool.size();
  }
  // ---- kvg_name_lookup per key
  for (uint32_t k = 0; k < n_keys; k++) {
    const uint8_t* key = keys + key_off[k];
    const uint32_t klen = key_off[k + 1] - key_off[k];
    uint8_t* out = names_out + (size_t)k * name_cap;
    names_len[k] = 0;
    uint32_t v;
    if (canonical_key(key, klen, &v)) {
      const uint32_t slot = nv_index[v];
      if (slot == P_NONE) continue;
      const uint32_t n = pool[slot] | ((uint32_t)pool[slot + 1] << 8);
      if (n > name_cap) return 2;
      memcpy(out, &pool[slot + 2], n);
      names_len[k] = n;
      continue;
    }
    uint32_t match = P_NONE, off2[2] = {0, klen}, n = 0;
    if (sec)
      emu_launch(k_lookup_general, dim3(4, 1), KVG_BLOCK, text, len, (const uint32_t*)sec_lines.data(),
                 (const uint32_t*)(sec_lines.data() + sec_cap), key, (const uint32_t*)off2, &match);
    emu_launch(k_sanitise_matches, dim3(1), 64, text, len, (const uint32_t*)off2, (const uint32_t*)&match, 1u, out, name_cap, &n, (const uint64_t*)nullptr);
    if (n > name_cap) return 2;
    names_len[k] = n;
  }
  return 0;
}

}  // extern "C"
