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
