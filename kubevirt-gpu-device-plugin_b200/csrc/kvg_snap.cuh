// kvg_snap.cuh — the readers of createIommuDeviceMap's walk callback, decoded on the GPU from the raw bytes the host
// read (kvg_scan_pci_raw), into the 16-byte records kvg_scan_pci takes.
//
//   k_raw_decode   one thread per Walk entry: the reference's short-circuit order (device_plugin.go:203-238), touching
//                  only the reads it reaches; writes the record as the all-numeric snapshot has it, the group and
//                  device spans, and the call's verdicts (RawCtrl): modes, lowest missing read, panic and range entry
//   k_raw_probe    index mode of one column: FNV-1a open-addressed table of the column's strings, one 64-bit word
//                  per slot = [call tag][lowest entry with that string], placed by CAS and lowered by atomicMin
//   k_compact<RawInternOp>  first appearances in Walk order -> handles 0, 1, ... (stable look-back compaction) and
//                  the handle -> span table the host copies the string tables from
//   k_raw_pack     addresses (index mode), groups and device ids (interned) into the records
//
// and the readers of createVgpuIDMap's walk callback (kvg_scan_mdev_raw), into the 32-byte records kvg_scan_mdev takes:
//
//   k_mraw_decode  one thread per Walk entry of the mdev bus: the short-circuit order of device_plugin.go:269-284;
//                  writes the record as the numeric snapshot has it, the type and parent spans, and the verdicts
//   k_raw_probe, k_compact<RawInternOp>  as above: column 0 = the type contents (always), 1 = the parent (index mode)
//   k_mraw_pack    type handles, parent handles (index mode) and the Walk index (names not canonical) into the records
//
// and the health re-scans from raw reads (kvg_health_rescan_groups_raw / kvg_health_rescan_mdev_raw): the entries
// decoded as above, the state joined by entry name, groups and parents matched as strings:
//
//   k_health_raw_small<Rule>                        poll-loop sizes: one CTA, the list into mapped host memory
//   k_compact<RawHealthOp<Rule>, KVG_BLOCK, C_ROWS>  above them
#pragma once
#include "../../include/kvgpu.h"
#include "kvg_common.cuh"
#include "kvg_scan.cuh"

namespace kvg {

constexpr uint32_t RAW_THREADS = 256;
constexpr uint32_t RAW_NONE = 0xffffffffu;
// RawCtrl::broken: the column is not in numeric mode
enum : uint32_t { RAW_BAD_ADDR = 1u, RAW_BAD_GROUP = 2u, RAW_BAD_DEVICE = 4u };
enum : uint32_t { RAW_COL_GROUP = 0, RAW_COL_DEVICE = 1 };

// The call's verdicts.  The three entry words hold (entry << 8) | field, lowest first; ~0 = none.  The host sets them
// to ~0 and the rest to 0 before the decode.
struct RawCtrl {
  unsigned long long miss;   // a read the reference reaches was not made
  unsigned long long panic;  // data[2:] on a file shorter than 2 bytes (vendor, device)
  unsigned long long range;  // numa_node outside int16, or the 65,537th distinct device string
  uint32_t broken;           // RAW_BAD_*
  uint32_t n_names[2];       // handles of the interned group / device strings
  uint32_t pad[7];
};

struct RawIn {
  const uint32_t* off;    // [n * KVG_RAW_FIELDS + 1] (the mdev walk: KVG_MRAW_FIELDS)
  const uint16_t* state;  // [n]
  const uint8_t* bytes;
  uint32_t n;
};

__device__ __forceinline__ bool raw_hex(uint8_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f'); }
__device__ __forceinline__ uint32_t raw_hexval(uint8_t c) { return c <= '9' ? c - '0' : c - 'a' + 10; }

// k hex digits at s as a number, or RAW_NONE
__device__ __forceinline__ uint32_t raw_hexn(const uint8_t* s, uint32_t k) {
  uint32_t v = 0;
  for (uint32_t j = 0; j < k; j++) {
    if (!raw_hex(s[j])) return RAW_NONE;
    v = v * 16 + raw_hexval(s[j]);
  }
  return v;
}
// 'dddd:bb:dd.f' -> packed BDF, or RAW_NONE (plugin.parse_bdf)
__device__ __forceinline__ uint32_t raw_bdf(const uint8_t* s, uint32_t len) {
  if (len != 12 || s[4] != ':' || s[7] != ':' || s[10] != '.') return RAW_NONE;
  const uint32_t dom = raw_hexn(s, 4), bus = raw_hexn(s + 5, 2), dev = raw_hexn(s + 8, 2), fn = raw_hexn(s + 11, 1);
  if (dom == RAW_NONE || bus == RAW_NONE || dev > 31 || fn > 7) return RAW_NONE;
  return (dom << 16) | (bus << 8) | (dev << 3) | fn;
}

// strings.Trim(string(data[2:]), "\n") (readIDFromFileFunc :300); the caller has checked len >= 2
__device__ __forceinline__ uint2 raw_id_span(const uint8_t* b, uint32_t a, uint32_t e) {
  a += 2;
  while (a < e && b[a] == '\n') a++;
  while (e > a && b[e - 1] == '\n') e--;
  return make_uint2(a, e);
}
// filepath.Split(os.Readlink(...)): the part after the last '/' (readLinkFunc :329)
__device__ __forceinline__ uint2 raw_base_span(const uint8_t* b, uint32_t a, uint32_t e) {
  uint32_t s = e;
  while (s > a && b[s - 1] != '/') s--;
  return make_uint2(s, e);
}

// utf8.DecodeRune; *w = bytes taken (1 for RuneError on bad input)
__device__ __forceinline__ uint32_t raw_decode_rune(const uint8_t* p, uint32_t n, uint32_t* w) {
  constexpr uint32_t ERR = 0xFFFD;
  *w = 1;
  if (n == 0) { *w = 0; return ERR; }
  const uint8_t b0 = p[0];
  if (b0 < 0x80) return b0;
  uint32_t need, lo = 0x80, hi = 0xBF, r;
  if (b0 >= 0xC2 && b0 <= 0xDF) { need = 1; r = b0 & 0x1F; }
  else if (b0 >= 0xE0 && b0 <= 0xEF) { need = 2; r = b0 & 0x0F; if (b0 == 0xE0) lo = 0xA0; if (b0 == 0xED) hi = 0x9F; }
  else if (b0 >= 0xF0 && b0 <= 0xF4) { need = 3; r = b0 & 0x07; if (b0 == 0xF0) lo = 0x90; if (b0 == 0xF4) hi = 0x8F; }
  else return ERR;
  if (n < need + 1) return ERR;
  if (p[1] < lo || p[1] > hi) return ERR;
  r = (r << 6) | (p[1] & 0x3F);
  for (uint32_t k = 2; k <= need; k++) {
    if ((p[k] & 0xC0) != 0x80) return ERR;
    r = (r << 6) | (p[k] & 0x3F);
  }
  *w = need + 1;
  return r;
}
// utf8.DecodeLastRune
__device__ __forceinline__ uint32_t raw_decode_last_rune(const uint8_t* p, uint32_t n, uint32_t* w) {
  if (n == 0) { *w = 0; return 0xFFFD; }
  if (p[n - 1] < 0x80) { *w = 1; return p[n - 1]; }
  const uint32_t lim = n >= 4 ? n - 4 : 0;
  uint32_t s = n - 1;
  while (s > lim && (p[s] & 0xC0) == 0x80) s--;
  uint32_t ww;
  const uint32_t r = raw_decode_rune(p + s, n - s, &ww);
  if (s + ww != n) { *w = 1; return 0xFFFD; }
  *w = ww;
  return r;
}
// unicode.IsSpace
__device__ __forceinline__ bool raw_space(uint32_t r) {
  return (r >= '\t' && r <= '\r') || r == ' ' || r == 0x85 || r == 0xA0 || r == 0x1680 || (r >= 0x2000 && r <= 0x200A) ||
         r == 0x2028 || r == 0x2029 || r == 0x202F || r == 0x205F || r == 0x3000;
}
// readNUMANodeFunc :310-315: strings.TrimSpace, then strconv.ParseInt(s, 10, 64).  False on a parse or range error.
// TrimSpace decodes runes on either side (its ASCII fast path trims the same bytes).
__device__ __forceinline__ bool raw_numa(const uint8_t* b, uint32_t a, uint32_t e, long long* out) {
  uint32_t w;
  while (a < e && raw_space(raw_decode_rune(b + a, e - a, &w))) a += w;
  while (e > a && raw_space(raw_decode_last_rune(b + a, e - a, &w))) e -= w;
  if (a == e) return false;
  bool neg = false;
  if (b[a] == '+' || b[a] == '-') {
    neg = b[a] == '-';
    if (++a == e) return false;
  }
  const unsigned long long cut = neg ? (1ull << 63) : (1ull << 63) - 1;
  unsigned long long v = 0;
  for (; a < e; a++) {
    const uint32_t d = (uint32_t)b[a] - '0';
    if (d > 9 || v > (cut - d) / 10) return false;
    v = v * 10 + d;
  }
  *out = neg ? (long long)(0ull - v) : (long long)v;
  return true;
}

// One Walk entry.  rec: the record in numeric mode (addr = packed BDF, group and device as numbers); span: the group
// basename when non-empty and the device id string when read ({1, 0} = none); bad: RAW_BAD_* of this entry.
struct RawEntry {
  uint4 rec;
  uint2 span[2];
  uint32_t bad;
};

__device__ __forceinline__ void raw_note(unsigned long long* word, uint32_t i, uint32_t field) {
  atomicMin(word, ((unsigned long long)i << 8) | field);
}

__device__ __forceinline__ RawEntry raw_decode_entry(const RawIn& in, uint32_t i, RawCtrl* ctrl) {
  const uint8_t* b = in.bytes;
  const uint32_t* o = in.off + (size_t)i * KVG_RAW_FIELDS;
  const uint32_t st = __ldg(&in.state[i]);
  RawEntry r;
  r.span[0] = r.span[1] = make_uint2(1, 0);
  r.bad = 0;
  const uint32_t addr = raw_bdf(b + o[KVG_RAW_NAME], o[KVG_RAW_NAME + 1] - o[KVG_RAW_NAME]);
  if (addr == RAW_NONE) r.bad |= RAW_BAD_ADDR;
  if (i > 0) {
    const uint32_t* p = o - KVG_RAW_FIELDS;
    const uint32_t prev = raw_bdf(b + p[KVG_RAW_NAME], p[KVG_RAW_NAME + 1] - p[KVG_RAW_NAME]);
    if (prev != RAW_NONE && addr != RAW_NONE && prev >= addr) r.bad |= RAW_BAD_ADDR;
  }
  uint32_t vendor = 0xffffu, device = 0, group = 0, driver = KVG_DRV_NONE, flags = 0;
  long long numa = 0;
  // a reached read: made?  failed?
  auto reach = [&](uint32_t f, uint32_t err_flag) -> bool {
    if (!((st >> f) & 1u)) {
      raw_note(&ctrl->miss, i, f);
      return false;
    }
    if ((st >> (8 + f)) & 1u) {
      flags |= err_flag;
      return false;
    }
    return true;
  };
  auto len_of = [&](uint32_t f) { return o[f + 1] - o[f]; };
  bool go = reach(KVG_RAW_VENDOR, KVG_PF_VENDOR_ERR);  // :202-206
  if (go && len_of(KVG_RAW_VENDOR) < 2) {
    raw_note(&ctrl->panic, i, KVG_RAW_VENDOR);
    go = false;
  }
  if (go) {
    const uint2 v = raw_id_span(b, o[KVG_RAW_VENDOR], o[KVG_RAW_VENDOR + 1]);
    const uint32_t x = v.y - v.x == 4 ? raw_hexn(b + v.x, 4) : RAW_NONE;
    if (x != RAW_NONE) vendor = x;
    go = vendor == 0x10deu;  // :209 the string equals "10de" exactly when it is these four digits
  }
  if (go && (go = reach(KVG_RAW_DRIVER, KVG_PF_DRIVER_ERR))) {  // :212-220, isSupportedVfioDriver :249-252
    const uint2 d = raw_base_span(b, o[KVG_RAW_DRIVER], o[KVG_RAW_DRIVER + 1]);
    const uint8_t* s = b + d.x;
    const uint32_t dl = d.y - d.x;
    const char* vfio = "vfio-pci";
    const char* grace = "nvgrace_gpu_vfio_pci";
    bool is_vfio = dl == 8, is_grace = dl == 20;
    for (uint32_t k = 0; k < dl && (is_vfio || is_grace); k++) {
      is_vfio = is_vfio && s[k] == (uint8_t)vfio[k];
      is_grace = is_grace && s[k] == (uint8_t)grace[k];
    }
    driver = is_vfio ? KVG_DRV_VFIO_PCI : is_grace ? KVG_DRV_NVGRACE : KVG_DRV_OTHER;
    go = driver != KVG_DRV_OTHER;
  }
  if (go && (go = reach(KVG_RAW_GROUP, KVG_PF_IOMMU_ERR))) {  // :221-225
    const uint2 g = raw_base_span(b, o[KVG_RAW_GROUP], o[KVG_RAW_GROUP + 1]);
    if (g.y > g.x) {
      r.span[RAW_COL_GROUP] = g;
      // numeric mode: canonical decimal below 2^32
      const uint32_t gl = g.y - g.x;
      bool ok = gl <= 10 && (gl == 1 || b[g.x] != '0');
      unsigned long long v = 0;
      for (uint32_t k = g.x; k < g.y && ok; k++) {
        const uint32_t dd = (uint32_t)b[k] - '0';
        ok = dd <= 9;
        v = v * 10 + dd;
      }
      if (ok && v <= 0xffffffffull) group = (uint32_t)v;
      else r.bad |= RAW_BAD_GROUP;
    }
  }
  if (go) {
    if (reach(KVG_RAW_NUMA, KVG_PF_NUMA_ERR)) {  // :226-230 (an error keeps the entry with node 0)
      if (!raw_numa(b, o[KVG_RAW_NUMA], o[KVG_RAW_NUMA + 1], &numa)) {
        flags |= KVG_PF_NUMA_ERR;
        numa = 0;
      } else if (numa < -32768 || numa > 32767) {
        raw_note(&ctrl->range, i, KVG_RAW_NUMA);
      }
    }
    if (reach(KVG_RAW_DEVICE, KVG_PF_DEVICE_ERR)) {  // :234-238
      if (len_of(KVG_RAW_DEVICE) < 2) {
        raw_note(&ctrl->panic, i, KVG_RAW_DEVICE);
      } else {
        const uint2 d = raw_id_span(b, o[KVG_RAW_DEVICE], o[KVG_RAW_DEVICE + 1]);
        r.span[RAW_COL_DEVICE] = d;
        const uint32_t x = d.y - d.x == 4 ? raw_hexn(b + d.x, 4) : RAW_NONE;
        if (x != RAW_NONE) device = x;
        else r.bad |= RAW_BAD_DEVICE;
      }
    }
  }
  r.rec = make_uint4(addr, vendor | device << 16, group, driver | flags << 8 | ((uint32_t)numa & 0xffffu) << 16);
  return r;
}

__global__ void __launch_bounds__(RAW_THREADS) k_raw_decode(RawIn in, uint4* __restrict__ recs, uint2* __restrict__ span,
                                                            RawCtrl* ctrl) {
  pdl_enter();
  const uint32_t i = blockIdx.x * RAW_THREADS + threadIdx.x;
  uint32_t bad = 0;
  if (i < in.n) {
    const RawEntry e = raw_decode_entry(in, i, ctrl);
    recs[i] = e.rec;
    span[2 * (size_t)i] = e.span[0];
    span[2 * (size_t)i + 1] = e.span[1];
    bad = e.bad;
  }
  // the modes: one atomic per warp that saw a non-numeric value
  const uint32_t m = __ballot_sync(KVG_FULL, bad & RAW_BAD_ADDR) ? RAW_BAD_ADDR : 0u;
  const uint32_t g = __ballot_sync(KVG_FULL, bad & RAW_BAD_GROUP) ? RAW_BAD_GROUP : 0u;
  const uint32_t d = __ballot_sync(KVG_FULL, bad & RAW_BAD_DEVICE) ? RAW_BAD_DEVICE : 0u;
  if (lane_id() == 0 && (m | g | d)) atomicOr(&ctrl->broken, m | g | d);
}

__device__ __forceinline__ uint64_t raw_fnv(const uint8_t* b, uint2 s) {
  uint64_t h = 1469598103934665603ull;
  for (uint32_t k = s.x; k < s.y; k++) h = (h ^ b[k]) * 1099511628211ull;
  return h;
}
__device__ __forceinline__ bool raw_same(const uint8_t* b, uint2 x, uint2 y) {
  if (x.y - x.x != y.y - y.x) return false;
  for (uint32_t k = 0; k < x.y - x.x; k++)
    if (b[x.x + k] != b[y.x + k]) return false;
  return true;
}

// Index mode of column `col`: every entry with a string finds the slot of that string (slot_of[i]; RAW_NONE without
// one), and the slot's word ends as [tag][the lowest such entry].  A slot of an earlier call's tag is free, so the
// table is never cleared; the table has at least twice as many slots as entries.
__global__ void __launch_bounds__(RAW_THREADS) k_raw_probe(const uint8_t* __restrict__ bytes, const uint2* __restrict__ span,
                                                           uint32_t n, uint32_t col, uint64_t* table, uint32_t mask,
                                                           uint32_t tag, uint32_t* __restrict__ slot_of) {
  pdl_enter();
  const uint32_t i = blockIdx.x * RAW_THREADS + threadIdx.x;
  if (i >= n) return;
  const uint2 s = span[2 * (size_t)i + col];
  if (s.y < s.x) {
    slot_of[i] = RAW_NONE;
    return;
  }
  const unsigned long long mine = ((unsigned long long)tag << 32) | i;
  unsigned long long* cas = reinterpret_cast<unsigned long long*>(table);
  for (uint32_t slot = (uint32_t)raw_fnv(bytes, s) & mask;; slot = (slot + 1) & mask) {
    unsigned long long w = ld_relaxed_u64(table + slot);
    if ((uint32_t)(w >> 32) != tag) {
      const unsigned long long seen = atomicCAS(cas + slot, w, mine);
      if (seen == w) {
        slot_of[i] = slot;
        return;
      }
      w = seen;  // another entry of this call took the slot first
    }
    if (raw_same(bytes, s, __ldg(&span[2 * (size_t)(uint32_t)w + col]))) {
      atomicMin(cas + slot, mine);
      slot_of[i] = slot;
      return;
    }
  }
}

// The first appearances of column `col` in Walk order, compacted by k_compact: handle h goes to the h-th first
// appearance.  hnd[i] = the handle of first appearance i, tab[h] = its span; a handle above max_hnd is the range error
// of its entry, noted on field range_field (the PCI device column: 0xffff, the 65,537th distinct string; the mdev
// types: 65534, the 65,536th; ~0 where every handle fits).
struct RawInternOp {
  using Item = uint32_t;
  const uint64_t* table;
  const uint32_t* slot_of;
  const uint2* span;
  uint32_t n, col;
  uint32_t max_hnd, range_field;
  uint32_t* hnd;
  uint2* tab;
  RawCtrl* ctrl;

  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    const uint32_t s = ok ? __ldg(&slot_of[i]) : RAW_NONE;
    return s == RAW_NONE ? RAW_NONE : (uint32_t)ld_relaxed_u64(table + s);
  }
  __device__ __forceinline__ bool pred(const Item& first, uint32_t i) const { return first == i; }
  __device__ __forceinline__ uint32_t prepare(const Item&) const { return 0; }
  __device__ __forceinline__ void emit(uint32_t pos, const Item&, uint32_t i, uint32_t) {
    hnd[i] = pos;
    tab[pos] = __ldg(&span[2 * (size_t)i + col]);
    if (pos > max_hnd) raw_note(&ctrl->range, i, range_field);
  }
  __device__ __forceinline__ void tile_epilogue() {}
  __device__ __forceinline__ void finish(uint32_t total) { ctrl->n_names[col] = total; }
};

// The modes the decode found, applied: the Walk index for addresses that are not all canonical and ascending, the
// handles of interned columns (an entry without the string: 0).
struct RawPackArgs {
  uint32_t n;
  uint32_t index_addr;
  const uint64_t* table[2];   // NULL: the column is numeric
  const uint32_t* slot_of[2];
  const uint32_t* hnd[2];
};
__global__ void __launch_bounds__(RAW_THREADS) k_raw_pack(RawPackArgs a, uint4* __restrict__ recs) {
  pdl_enter();
  const uint32_t i = blockIdx.x * RAW_THREADS + threadIdx.x;
  if (i >= a.n) return;
  uint4 r = recs[i];
  if (a.index_addr) r.x = i;
  uint32_t h[2] = {0, 0};
  for (int c = 0; c < 2; c++) {
    if (!a.table[c]) continue;
    const uint32_t s = __ldg(&a.slot_of[c][i]);
    if (s != RAW_NONE) h[c] = __ldg(&a.hnd[c][(uint32_t)ld_relaxed_u64(a.table[c] + s)]);
  }
  if (a.table[RAW_COL_GROUP]) r.z = h[RAW_COL_GROUP];
  if (a.table[RAW_COL_DEVICE]) r.y = (r.y & 0xffffu) | (h[RAW_COL_DEVICE] & 0xffffu) << 16;
  recs[i] = r;
}

// ---- the mdev bus (kvg_scan_mdev_raw) --------------------------------------------------------------------------
// RawCtrl::broken of the mdev walk: the names are not canonical ascending UUIDs / a parent is not a canonical BDF
enum : uint32_t { MRAW_BAD_UUID = 1u, MRAW_BAD_PARENT = 2u };
enum : uint32_t { MRAW_COL_TYPE = 0, MRAW_COL_PARENT = 1 };

__device__ __forceinline__ uint32_t raw_bswap(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// a canonical lower-case 'xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx' -> its 16 bytes as two big-endian halves; false else
__device__ __forceinline__ bool raw_uuid(const uint8_t* s, uint32_t len, unsigned long long* hi, unsigned long long* lo) {
  if (len != 36) return false;
  unsigned long long h = 0, l = 0;
  for (uint32_t j = 0, k = 0; j < 36; j++) {
    const uint8_t c = s[j];
    if (j == 8 || j == 13 || j == 18 || j == 23) {
      if (c != '-') return false;
      continue;
    }
    if (!raw_hex(c)) return false;
    if (k++ < 16) h = h << 4 | raw_hexval(c);
    else l = l << 4 | raw_hexval(c);
  }
  *hi = h;
  *lo = l;
  return true;
}

// One mdev Walk entry: rec[0] = the UUID words (numeric mode), rec[1] = parent (packed BDF or 0), flags << 16,
// parent_numa; span: the type contents when read and the parent when decoded ({1, 0} = none); bad: MRAW_BAD_*.
struct MRawEntry {
  uint4 rec[2];
  uint2 span[2];
  uint32_t bad;
};

__device__ __forceinline__ MRawEntry mraw_decode_entry(const RawIn& in, uint32_t i, RawCtrl* ctrl) {
  const uint8_t* b = in.bytes;
  const uint32_t* o = in.off + (size_t)i * KVG_MRAW_FIELDS;
  const uint32_t st = __ldg(&in.state[i]);
  MRawEntry r;
  r.span[0] = r.span[1] = make_uint2(1, 0);
  r.bad = 0;
  unsigned long long hi = 0, lo = 0;
  if (!raw_uuid(b + o[KVG_MRAW_NAME], o[KVG_MRAW_NAME + 1] - o[KVG_MRAW_NAME], &hi, &lo)) {
    r.bad |= MRAW_BAD_UUID;
    hi = lo = 0;
  } else if (i > 0) {  // strictly ascending, as 16 big-endian bytes
    const uint32_t* p = o - KVG_MRAW_FIELDS;
    unsigned long long ph, pl;
    if (raw_uuid(b + p[KVG_MRAW_NAME], p[KVG_MRAW_NAME + 1] - p[KVG_MRAW_NAME], &ph, &pl) &&
        (ph > hi || (ph == hi && pl >= lo)))
      r.bad |= MRAW_BAD_UUID;
  }
  uint32_t parent = 0, flags = 0;
  long long numa = 0;
  auto reach = [&](uint32_t f, uint32_t err_flag) -> bool {
    if (!((st >> f) & 1u)) {
      raw_note(&ctrl->miss, i, f);
      return false;
    }
    if ((st >> (8 + f)) & 1u) {
      flags |= err_flag;
      return false;
    }
    return true;
  };
  if (reach(KVG_MRAW_TYPE, KVG_MF_TYPE_ERR)) {  // :269-273
    r.span[MRAW_COL_TYPE] = make_uint2(o[KVG_MRAW_TYPE], o[KVG_MRAW_TYPE + 1]);
    if (reach(KVG_MRAW_LINK, KVG_MF_PARENT_ERR)) {  // :275-279, readGpuIDForVgpuFunc :347-357
      const uint32_t a = o[KVG_MRAW_LINK];
      uint32_t e = o[KVG_MRAW_LINK + 1];
      while (e > a && b[e - 1] != '/') e--;
      if (e == a) {
        raw_note(&ctrl->panic, i, KVG_MRAW_LINK);  // splitStr[len(splitStr)-2] of a single component
      } else {
        e--;  // the last '/'
        uint32_t s = e;
        while (s > a && b[s - 1] != '/') s--;
        while (s < e && b[s] == '\n') s++;  // strings.Trim(.., "\n")
        while (e > s && b[e - 1] == '\n') e--;
        r.span[MRAW_COL_PARENT] = make_uint2(s, e);
        parent = raw_bdf(b + s, e - s);
        if (parent == RAW_NONE) {
          r.bad |= MRAW_BAD_PARENT;
          parent = 0;
        }
        if (reach(KVG_MRAW_NUMA, KVG_MF_NUMA_ERR)) {  // :280-284 (an error keeps the entry with node 0)
          if (!raw_numa(b, o[KVG_MRAW_NUMA], o[KVG_MRAW_NUMA + 1], &numa)) {
            flags |= KVG_MF_NUMA_ERR;
            numa = 0;
          } else if (numa < -32768 || numa > 32767) {
            raw_note(&ctrl->range, i, KVG_MRAW_NUMA);
          }
        }
      }
    }
  }
  r.rec[0] = make_uint4(raw_bswap((uint32_t)(hi >> 32)), raw_bswap((uint32_t)hi), raw_bswap((uint32_t)(lo >> 32)),
                        raw_bswap((uint32_t)lo));
  r.rec[1] = make_uint4(parent, flags << 16, (uint32_t)numa & 0xffffu, 0);
  return r;
}

__global__ void __launch_bounds__(RAW_THREADS) k_mraw_decode(RawIn in, uint4* __restrict__ recs, uint2* __restrict__ span,
                                                             RawCtrl* ctrl) {
  pdl_enter();
  const uint32_t i = blockIdx.x * RAW_THREADS + threadIdx.x;
  uint32_t bad = 0;
  if (i < in.n) {
    const MRawEntry e = mraw_decode_entry(in, i, ctrl);
    recs[2 * (size_t)i] = e.rec[0];
    recs[2 * (size_t)i + 1] = e.rec[1];
    span[2 * (size_t)i] = e.span[0];
    span[2 * (size_t)i + 1] = e.span[1];
    bad = e.bad;
  }
  const uint32_t u = __ballot_sync(KVG_FULL, bad & MRAW_BAD_UUID) ? MRAW_BAD_UUID : 0u;
  const uint32_t p = __ballot_sync(KVG_FULL, bad & MRAW_BAD_PARENT) ? MRAW_BAD_PARENT : 0u;
  if (lane_id() == 0 && (u | p)) atomicOr(&ctrl->broken, u | p);
}

// The modes applied to the 32-byte records: type_idx from the type handles (always interned; 0 without a type),
// parent from the parent handles when a.table[MRAW_COL_PARENT] is set (0 without a parent), and the Walk index,
// big-endian, in bytes 0..3 of the UUID when a.index_addr is set.
__global__ void __launch_bounds__(RAW_THREADS) k_mraw_pack(RawPackArgs a, uint4* __restrict__ recs) {
  pdl_enter();
  const uint32_t i = blockIdx.x * RAW_THREADS + threadIdx.x;
  if (i >= a.n) return;
  if (a.index_addr) recs[2 * (size_t)i] = make_uint4(raw_bswap(i), 0, 0, 0);
  uint4 r = recs[2 * (size_t)i + 1];
  uint32_t h[2] = {0, 0};
  for (int c = 0; c < 2; c++) {
    if (!a.table[c]) continue;
    const uint32_t s = __ldg(&a.slot_of[c][i]);
    if (s != RAW_NONE) h[c] = __ldg(&a.hnd[c][(uint32_t)ld_relaxed_u64(a.table[c] + s)]);
  }
  r.y = (r.y & 0xffff0000u) | (h[MRAW_COL_TYPE] & 0xffffu);
  if (a.table[MRAW_COL_PARENT]) r.x = h[MRAW_COL_PARENT];
  recs[2 * (size_t)i + 1] = r;
}

// ---- K6 from raw reads (kvg_health_rescan_groups_raw / kvg_health_rescan_mdev_raw) ------------------------------
// The health rules of kvg_scan.cuh on entries decoded by the scans' own decoders (raw_decode_entry,
// mraw_decode_entry), with every identity a string compared byte for byte: an entry is its name, a group or parent
// is its string, the tick's set is a list of strings.
//   RawNameSet<CAP>   the set (VFIO node names / XID bus ids) as a per-CTA open-addressed table in shared memory, built
//                     once per call: one word per slot, tag (19 hash bits) << 13 | index + 1; the strings stay in
//                     global memory, behind the entries' bytes
//   RawNameJoin       the prior state byte of a name: the same position of the previous list first, then a binary
//                     search of its names (Keyed<Rule>::find with a byte-wise compare)
//   raw_health_step   one entry: the name-ascent check, the join, the rule, this call's byte
//   k_health_raw_small<Rule>             poll-loop sizes: one CTA, the transition list into mapped host memory
//   k_compact<RawHealthOp<Rule>, KVG_BLOCK, C_ROWS>  above them (or with kernel timing on)

// byte-wise order of a[x.x, x.y) and c[y.x, y.y): <0, 0, >0
__device__ __forceinline__ int raw_cmp(const uint8_t* a, uint2 x, const uint8_t* c, uint2 y) {
  const uint32_t la = x.y - x.x, lc = y.y - y.x, m = min(la, lc);
  for (uint32_t k = 0; k < m; k++) {
    const uint32_t p = a[x.x + k], q = c[y.x + k];
    if (p != q) return p < q ? -1 : 1;
  }
  return la < lc ? -1 : la > lc ? 1 : 0;
}

constexpr uint32_t RAW_SET_IDX_BITS = 13;
static_assert(KVG_HEALTH_MAX_GROUPS < (1u << RAW_SET_IDX_BITS) && KVG_HEALTH_MAX_XID < (1u << RAW_SET_IDX_BITS),
              "index + 1 of every set string fits the slot word");
template <uint32_t CAP>
struct RawNameSet {
  static constexpr uint32_t SLOTS = 2 * CAP, MASK = SLOTS - 1;  // at most half full
  uint32_t* slot;                                               // shared memory, [SLOTS]
  const uint8_t* bytes;                                         // string k = bytes[off[k], off[k + 1])
  const uint32_t* off;
  __device__ __forceinline__ static uint32_t tag(uint64_t h) { return (uint32_t)(h >> 45); }
  // every thread of the CTA: clear the table, then place its share of the n strings (duplicates take a slot each)
  __device__ __forceinline__ void build(uint32_t n) {
    for (uint32_t k = threadIdx.x; k < SLOTS; k += blockDim.x) slot[k] = 0;
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) {
      const uint64_t h = raw_fnv(bytes, make_uint2(__ldg(&off[k]), __ldg(&off[k + 1])));
      const uint32_t w = tag(h) << RAW_SET_IDX_BITS | (k + 1);
      for (uint32_t s = (uint32_t)h & MASK;; s = (s + 1) & MASK)
        if (atomicCAS(&slot[s], 0u, w) == 0u) break;
    }
    __syncthreads();
  }
  // is bytes[x) one of the strings?
  __device__ __forceinline__ bool has(uint2 x) const {
    const uint64_t h = raw_fnv(bytes, x);
    const uint32_t t = tag(h);
    for (uint32_t s = (uint32_t)h & MASK;; s = (s + 1) & MASK) {
      const uint32_t w = slot[s];
      if (!w) return false;
      const uint32_t k = (w & ((1u << RAW_SET_IDX_BITS) - 1)) - 1;
      if ((w >> RAW_SET_IDX_BITS) == t && raw_same(bytes, x, make_uint2(__ldg(&off[k]), __ldg(&off[k + 1]))))
        return true;
    }
  }
};

// The previous call's list: its names (field 0 of each entry of its staged walk, `fields` offsets per entry) ascending
// byte-wise, and its state bytes.
struct RawNameJoin {
  const uint32_t* off;
  const uint8_t* bytes;
  const uint8_t* state;
  uint32_t n, fields;
  __device__ __forceinline__ uint2 name(uint32_t j) const {
    return make_uint2(__ldg(&off[(size_t)j * fields]), __ldg(&off[(size_t)j * fields + 1]));
  }
  // the prior byte of the name b[k), entry i of this call; 0 for a name the previous list lacks
  __device__ __forceinline__ uint32_t find(const uint8_t* b, uint2 k, uint32_t i) const {
    if (i < n && raw_cmp(bytes, name(i), b, k) == 0) return __ldg(&state[i]);
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (raw_cmp(bytes, name(mid), b, k) < 0)
        lo = mid + 1;
      else
        hi = mid;
    }
    return lo < n && raw_cmp(bytes, name(lo), b, k) == 0 ? (uint32_t)__ldg(&state[lo]) : 0u;
  }
};

// passthrough GPUs by IOMMU group: h' = pci_record_alive(decoded record) && the iommu_group link basename is one of
// the node names.  An alive record has read its link; a basename left without a span is the empty string.
struct GroupRawRule {
  static constexpr uint32_t FIELDS = KVG_RAW_FIELDS, SET_CAP = KVG_HEALTH_MAX_GROUPS, STATE_BITS = 1;
  __device__ __forceinline__ static uint32_t next(const RawIn& in, uint32_t i, uint32_t, RawCtrl* ctrl,
                                                  const RawNameSet<SET_CAP>& set) {
    const RawEntry e = raw_decode_entry(in, i, ctrl);
    const uint2 g = e.span[RAW_COL_GROUP];
    return health_group_next(e.rec, [&] { return set.has(g.y >= g.x ? g : make_uint2(0, 0)); });
  }
};
// vGPUs: present = the type and link reads succeeded (the raw dictionary always holds the type: one entry, index 0),
// marked by a non-empty decoded parent that is one of the XID bus ids.
struct MdevRawRule {
  static constexpr uint32_t FIELDS = KVG_MRAW_FIELDS, SET_CAP = KVG_HEALTH_MAX_XID, STATE_BITS = 2;
  __device__ __forceinline__ static uint32_t next(const RawIn& in, uint32_t i, uint32_t s, RawCtrl* ctrl,
                                                  const RawNameSet<SET_CAP>& set) {
    const MRawEntry e = mraw_decode_entry(in, i, ctrl);
    const uint2 p = e.span[MRAW_COL_PARENT];
    return health_mdev_next(e.rec[1], s, 1u, [&] { return p.y > p.x && set.has(p); });
  }
};

// One call: this call's entries (the set's strings behind their bytes: set_off indexes in.bytes), the previous list,
// and where this call's state bytes go.
struct RawHealthArgs {
  RawIn in;
  const uint32_t* set_off;  // [n_set + 1]
  uint32_t n_set;
  RawNameJoin prev;
  uint8_t* state;  // [in.n]
};

// Entry i: its name must exceed entry i - 1's (else *name_err = 1), its prior byte comes from the previous list by
// name, the rule gives its new byte, which goes to this call's slot.  Returns the new byte; *was = the prior one.
template <class Rule>
__device__ __forceinline__ uint32_t raw_health_step(const RawHealthArgs& a, const RawNameSet<Rule::SET_CAP>& set,
                                                    uint32_t i, RawCtrl* ctrl, uint32_t* name_err, uint32_t* was) {
  const uint8_t* b = a.in.bytes;
  const uint32_t* o = a.in.off + (size_t)i * Rule::FIELDS;
  const uint2 nm = make_uint2(o[0], o[1]);
  if (i > 0 && raw_cmp(b, make_uint2(o[-(int)Rule::FIELDS], o[1 - (int)Rule::FIELDS]), b, nm) >= 0) *name_err = 1u;
  *was = a.prev.find(b, nm, i);
  const uint32_t s = Rule::next(a.in, i, *was, ctrl, set);
  a.state[i] = (uint8_t)s;
  return s;
}

// Poll-loop sizes (n <= HEALTH_SMALL_MAX): ONE CTA, one launch.  Thread t takes entries t, t + 1024, ... (a row of
// 1024 per step); the verdicts of the decode and the name check collect in shared memory; the list, the counters,
// the verdicts and last the sequence word go straight into the host-visible result block: hdr_host = {n_alive,
// n_changed, seq, name_err} then {miss, panic, range} as u64.
template <class Rule>
__global__ void __launch_bounds__(HEALTH_SMALL_THREADS) k_health_raw_small(RawHealthArgs a,
                                                                           uint32_t* __restrict__ changed_host,
                                                                           uint32_t* __restrict__ hdr_host,
                                                                           uint32_t seq) {
  pdl_enter();
  constexpr uint32_t NW = HEALTH_SMALL_NW;
  __shared__ uint32_t s_set[RawNameSet<Rule::SET_CAP>::SLOTS];
  __shared__ RawCtrl s_ctrl;
  __shared__ uint32_t s_err;
  __shared__ uint32_t s_bal[HEALTH_SMALL_ROWS][NW];  // "changed" ballot of (row, warp)
  __shared__ uint32_t s_now[HEALTH_SMALL_ROWS][NW];  // "healthy now" ballot of (row, warp)
  __shared__ uint32_t s_scan[NW], s_alv[NW];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = a.in.n;
  if (tid == 0) {
    s_ctrl.miss = s_ctrl.panic = s_ctrl.range = ~0ull;
    s_err = 0;
  }
  RawNameSet<Rule::SET_CAP> set = {s_set, a.in.bytes, a.set_off};
  set.build(a.n_set);  // (its barriers also publish s_ctrl and s_err)
  const uint32_t rows = (n + HEALTH_SMALL_THREADS - 1) / HEALTH_SMALL_THREADS;
  uint32_t n_alive = 0;
#pragma unroll 1
  for (uint32_t r = 0; r < rows; r++) {  // uniform
    const uint32_t i = r * HEALTH_SMALL_THREADS + tid;
    const bool in = i < n;
    uint32_t s = 0, was = 0;
    if (in) s = raw_health_step<Rule>(a, set, i, &s_ctrl, &s_err, &was);
    const bool now = in && (s & 1u) != 0;
    const bool chg = in && (now ? 1u : 0u) != (was & 1u);
    const uint32_t bc = __ballot_sync(KVG_FULL, chg), bn = __ballot_sync(KVG_FULL, now);
    if (lane == 0) {
      s_bal[r][warp] = bc;
      s_now[r][warp] = bn;
    }
    n_alive += now ? 1u : 0u;
  }
  __syncthreads();  // every row's ballots are in place before any thread reads another warp's
  uint32_t alive, total;
  health_small_list(rows, n_alive, s_bal, s_now, s_scan, s_alv, changed_host, alive, total);
  if (tid == 0) {
    hdr_host[0] = alive;
    hdr_host[1] = total;
    hdr_host[3] = s_err;
    unsigned long long* v = reinterpret_cast<unsigned long long*>(hdr_host + 4);
    v[0] = s_ctrl.miss;
    v[1] = s_ctrl.panic;
    v[2] = s_ctrl.range;
    __threadfence_system();
    *((volatile uint32_t*)&hdr_host[2]) = seq;  // the host polls this word
  }
}

// The look-back form: k_compact<RawHealthOp<Rule>, KVG_BLOCK, C_ROWS>.  Item = new byte | prior byte << W; a change of
// bit 0 is listed.  The verdicts go to ctrl (RawCtrl), the name check to sc->key_err, the counters to sc.
template <class Rule>
struct RawHealthOp {
  using Item = uint32_t;
  static constexpr uint32_t W = Rule::STATE_BITS;
  RawHealthArgs a;
  RawNameSet<Rule::SET_CAP> set;  // slot: compact_enter
  uint32_t n;
  RawCtrl* ctrl;
  ScanCtrl* sc;
  uint32_t* changed;
  uint32_t local_alive;
  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    if (!ok) return 0;
    uint32_t was;
    const uint32_t s = raw_health_step<Rule>(a, set, i, ctrl, &sc->key_err, &was);
    return s | was << W;
  }
  __device__ __forceinline__ bool pred(const Item& x, uint32_t) {
    const uint32_t now = x & ((1u << W) - 1), was = x >> W;
    local_alive += now & 1u;
    return ((now ^ was) & 1u) != 0;
  }
  __device__ __forceinline__ uint32_t prepare(const Item&) const { return 0; }
  __device__ __forceinline__ void emit(uint32_t pos, const Item& x, uint32_t i, uint32_t) {
    changed[pos] = (i << 1) | (x & 1u);
  }
  __device__ __forceinline__ void tile_epilogue() {
    const uint32_t s = warp_sum(local_alive);
    if (lane_id() == 0 && s) atomicAdd(&sc->n_alive, s);
    local_alive = 0;
  }
  __device__ __forceinline__ void finish(uint32_t total) { sc->n_changed = total; }
};
template <class Rule>
__device__ __forceinline__ void compact_enter(RawHealthOp<Rule>& op) {
  __shared__ uint32_t s_set[RawNameSet<Rule::SET_CAP>::SLOTS];
  op.set.slot = s_set;
  op.set.build(op.a.n_set);
}
// without the bound ptxas holds the vGPU instantiation to 40 registers and spills
template <class Rule>
constexpr int COMPACT_MIN_BLOCKS<RawHealthOp<Rule>> = 1;
template <class Rule>
inline RawHealthOp<Rule> raw_health_op(const RawHealthArgs& a, RawCtrl* ctrl, ScanCtrl* sc, uint32_t* changed) {
  RawHealthOp<Rule> op;
  op.a = a;
  op.set = {nullptr, a.in.bytes, a.set_off};
  op.n = a.in.n;
  op.ctrl = ctrl;
  op.sc = sc;
  op.changed = changed;
  op.local_alive = 0;
  return op;
}

// ---- the launch plan of both raw scans (host side; kvg_api_snap.inc and the CPU emulator build it alike) ---------
// What differs between the two walks: a record of rec_words uint4; column c is interned when interned(broken, c), a
// handle above max_hnd[c] being the range error of field range_field[c]; broken & bad_addr puts the names in index
// mode.  The snapshot's mode flag mode[m] is 1 iff bit m of broken is clear, and column c's string table is
// n_names[c], names_off[c], names_bytes[c].  empty_result and scan (the scan and fetch of the packed records) are the
// library's, defined in kvg_api_snap.inc.
template <class S, class T>
using Member = T S::*;
struct PciWalk {
  using Raw = kvg_pci_raw;
  using Snap = kvg_pci_snap;
  using Result = kvg_pci_result;
  static constexpr uint32_t fields = KVG_RAW_FIELDS, rec_words = 1;
  static constexpr auto decode = k_raw_decode;
  static constexpr auto pack = k_raw_pack;
  static constexpr const char *decode_label = "raw_decode", *intern_label = "raw_intern", *pack_label = "raw_pack";
  static bool interned(uint32_t broken, uint32_t c) {
    return broken & (c == RAW_COL_GROUP ? RAW_BAD_GROUP : RAW_BAD_DEVICE);
  }
  static constexpr uint32_t bad_addr = RAW_BAD_ADDR;
  static constexpr uint32_t max_hnd[2] = {0xffffffffu, 0xffffu}, range_field[2] = {KVG_RAW_DEVICE, KVG_RAW_DEVICE};
  static constexpr Member<Snap, uint8_t> mode[3] = {&Snap::packed_addr, &Snap::groups_numeric,
                                                     &Snap::devices_numeric};
  static constexpr Member<Snap, uint32_t> n_names[2] = {&Snap::n_group_names, &Snap::n_device_names};
  static constexpr Member<Snap, const uint32_t*> names_off[2] = {&Snap::group_off, &Snap::device_off};
  static constexpr Member<Snap, const uint8_t*> names_bytes[2] = {&Snap::group_bytes, &Snap::device_bytes};
  // kvg_last_error: "<fn>: a read ... at <where>", "<panic_at><where>", "<range_at><where>" (numa_field: its own)
  static constexpr const char* fn = "kvg_scan_pci_raw";
  static constexpr const char* panic_at = "the reference panics (slice bounds out of range, data[2:]) at ";
  static constexpr const char* range_at = "more than 65536 distinct device strings at ";
  static constexpr uint32_t numa_field = KVG_RAW_NUMA;
  static constexpr const char* field_name[KVG_RAW_FIELDS] = {"name",        "vendor",    "driver",
                                                             "iommu_group", "numa_node", "device"};
  static int empty_result(kvg_ctx* ctx, void** blk, Result** res);
  static int scan(kvg_ctx* ctx, const Snap* s, Result** res);
};
struct MdevWalk {
  using Raw = kvg_mdev_raw;
  using Snap = kvg_mdev_snap;
  using Result = kvg_mdev_result;
  static constexpr uint32_t fields = KVG_MRAW_FIELDS, rec_words = 2;
  static constexpr auto decode = k_mraw_decode;
  static constexpr auto pack = k_mraw_pack;
  static constexpr const char *decode_label = "mraw_decode", *intern_label = "mraw_intern", *pack_label = "mraw_pack";
  // the types always; the parents when one is not a canonical BDF
  static bool interned(uint32_t broken, uint32_t c) { return c == MRAW_COL_TYPE || (broken & MRAW_BAD_PARENT); }
  static constexpr uint32_t bad_addr = MRAW_BAD_UUID;
  // 65,535 types at most (load_type_dict)
  static constexpr uint32_t max_hnd[2] = {65534u, 0xffffffffu}, range_field[2] = {KVG_MRAW_TYPE, KVG_MRAW_LINK};
  static constexpr Member<Snap, uint8_t> mode[2] = {&Snap::uuid_ok, &Snap::parents_packed};
  static constexpr Member<Snap, uint32_t> n_names[2] = {&Snap::n_types, &Snap::n_parent_names};
  static constexpr Member<Snap, const uint32_t*> names_off[2] = {&Snap::type_off, &Snap::parent_off};
  static constexpr Member<Snap, const uint8_t*> names_bytes[2] = {&Snap::type_bytes, &Snap::parent_bytes};
  static constexpr const char* fn = "kvg_scan_mdev_raw";
  static constexpr const char* panic_at = "the reference panics (index out of range, a link target without '/') at ";
  static constexpr const char* range_at = "more than 65535 distinct mdev_type/name contents at ";
  static constexpr uint32_t numa_field = KVG_MRAW_NUMA;
  static constexpr const char* field_name[KVG_MRAW_FIELDS] = {"name", "mdev_type/name", "link", "numa_node"};
  static int empty_result(kvg_ctx* ctx, void** blk, Result** res);
  static int scan(kvg_ctx* ctx, const Snap* s, Result** res);
};

// the snapshot's mode flags from the walk's broken bits, and back
template <class W>
inline void raw_snap_modes(typename W::Snap* s, uint32_t broken) {
  uint32_t m = 0;
  for (auto flag : W::mode) s->*flag = !((broken >> m++) & 1u);
}
template <class W>
inline uint32_t raw_snap_broken(const typename W::Snap& s) {
  uint32_t broken = 0, m = 0;
  for (auto flag : W::mode) broken |= (s.*flag ? 0u : 1u) << m++;
  return broken;
}

// The probe table of each column holds raw_slots(n) words, at least twice as many as entries
inline size_t raw_slots(size_t n) {
  size_t slots = 64;
  while (slots < 2 * n) slots <<= 1;
  return slots;
}
// The index-mode work of both columns, column after column: probe tables, then slots, handles and handle spans per
// entry
struct RawWork {
  uint64_t* table;
  uint32_t *slot_of, *hnd;
  uint2* tab;
};
// column c of it, with the probe mask k_raw_probe takes
struct RawColumn {
  uint64_t* table;
  uint32_t mask;
  uint32_t *slot_of, *hnd;
  uint2* tab;
};
inline RawColumn raw_column(const RawWork& w, size_t n, uint32_t c) {
  const size_t slots = raw_slots(n);
  return {w.table + c * slots, (uint32_t)(slots - 1), w.slot_of + c * n, w.hnd + c * n, w.tab + c * n};
}
template <class W>
inline RawInternOp raw_intern_op(const RawColumn& col, const uint2* span, uint32_t n, uint32_t c, RawCtrl* ctrl) {
  RawInternOp op;
  op.table = col.table;
  op.slot_of = col.slot_of;
  op.span = span;
  op.n = n;
  op.col = c;
  op.max_hnd = W::max_hnd[c];
  op.range_field = W::range_field[c];
  op.hnd = col.hnd;
  op.tab = col.tab;
  op.ctrl = ctrl;
  return op;
}
// the pack runs iff the names are in index mode or a column is interned
template <class W>
inline bool raw_pack_needed(uint32_t broken) {
  return (broken & W::bad_addr) || W::interned(broken, 0) || W::interned(broken, 1);
}
template <class W>
inline RawPackArgs raw_pack_args(const RawWork& w, uint32_t n, uint32_t broken) {
  RawPackArgs a = {};
  a.n = n;
  a.index_addr = (broken & W::bad_addr) ? 1u : 0u;
  for (uint32_t c = 0; c < 2; c++)
    if (W::interned(broken, c)) {
      const RawColumn col = raw_column(w, n, c);
      a.table[c] = col.table;
      a.slot_of[c] = col.slot_of;
      a.hnd[c] = col.hnd;
    }
  return a;
}

}  // namespace kvg
