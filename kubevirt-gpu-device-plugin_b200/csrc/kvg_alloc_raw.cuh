// kvg_alloc_raw.cuh — the passthrough plugin's Allocate decisions from the raw reads the reference makes for them
// (kvg_pci_allocate_raw): the readers of the group re-check and of EGM discovery, and the EGM key rule, on the GPU.
//
//   k_araw_members  one thread per group member: the link basename against the group string, then the vendor file
//                   (generic_device_plugin.go:387-399), into the record k_pci_allocate_check judges: group 0 on a match
//                   (1 otherwise) against a wanted group of 0, vendor 0x10de when the vendor read back as "10de"
//                   (0xffff otherwise).  How the member ended goes to one code byte per member (ARAW_*) in mapped host
//                   memory, written only when it is not ARAW_PASS.
//   k_araw_keys     one CTA: the EGM class entries (discoverEGMDevicesFunc :120-157), kept or not; the fields of the
//                   kept ones (strings.Fields); every field's key (strings.ToLower(strings.TrimSpace)) interned into a
//                   handle, dense in order of first appearance, through an FNV-1a table of the lowered runes; then
//                   every DevicesID's key looked up in it.  Writes the EGM device lists k_pci_allocate_check takes: a
//                   kept entry lists its fields' handles, any other entry the one handle ARAW_NEVER, which no ID
//                   carries; an ID matching no field gets ARAW_NOT_EGM (>= the n_egm_gpus it is launched with).
//   k_pci_allocate_check (kvg_scan.cuh), unchanged, then decides first_bad and the EGM match of every request.
#pragma once
#include "../../include/kvgpu.h"
#include "kvg_common.cuh"
#include "kvg_alloc.cuh"
#include "kvg_case.cuh"
#include "kvg_snap.cuh"

namespace kvg {

constexpr uint32_t ARAW_THREADS = 256;
constexpr uint32_t ARAW_KEY_THREADS = PREF_THREADS;  // pref_excl_sum scans the block
constexpr uint32_t ARAW_NEVER = KVG_ALLOC_RAW_MAX_EGM_KEYS;  // the handle of an entry that is not kept
constexpr uint32_t ARAW_NOT_EGM = KVG_ALLOC_MAX_EGM_GPUS;    // an ID that matches no field
// how a member's re-check ended; a missing read stops the request like a failure, so the host finds it at first_bad
enum : uint32_t { ARAW_PASS = 0, ARAW_FAIL = 1, ARAW_PANIC = 2, ARAW_MISS_LINK = 3, ARAW_MISS_VENDOR = 4 };

__device__ __forceinline__ uint32_t araw_member(const uint8_t* b, const uint32_t* o, uint32_t st) {
  if (!(st >> KVG_AMEM_LINK & 1u)) return ARAW_MISS_LINK;
  if (st >> (8 + KVG_AMEM_LINK) & 1u) return ARAW_FAIL;
  const uint2 g = raw_base_span(b, o[KVG_AMEM_LINK], o[KVG_AMEM_LINK + 1]);
  if (!raw_same(b, g, make_uint2(o[KVG_AMEM_GROUP], o[KVG_AMEM_GROUP + 1]))) return ARAW_FAIL;  // :388
  if (!(st >> KVG_AMEM_VENDOR & 1u)) return ARAW_MISS_VENDOR;
  if (st >> (8 + KVG_AMEM_VENDOR) & 1u) return ARAW_FAIL;
  if (o[KVG_AMEM_VENDOR + 1] - o[KVG_AMEM_VENDOR] < 2) return ARAW_PANIC;  // data[2:] (:300)
  const uint2 v = raw_id_span(b, o[KVG_AMEM_VENDOR], o[KVG_AMEM_VENDOR + 1]);
  const bool nv = v.y - v.x == 4 && b[v.x] == '1' && b[v.x + 1] == '0' && b[v.x + 2] == 'd' && b[v.x + 3] == 'e';
  return nv ? ARAW_PASS : ARAW_FAIL;  // :393
}

__global__ void __launch_bounds__(ARAW_THREADS) k_araw_members(const uint32_t* __restrict__ off,
                                                               const uint16_t* __restrict__ state,
                                                               const uint8_t* __restrict__ bytes, uint32_t n,
                                                               uint4* __restrict__ recs, uint32_t* __restrict__ want,
                                                               uint8_t* code_host) {
  pdl_enter();
  const uint32_t i = blockIdx.x * ARAW_THREADS + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = araw_member(bytes, off + (size_t)i * KVG_AMEM_FIELDS, __ldg(&state[i]));
  const bool link_ok = c == ARAW_PASS || c == ARAW_PANIC || c == ARAW_MISS_VENDOR;
  recs[i] = make_uint4(i, c == ARAW_PASS ? 0x10deu : 0xffffu, link_ok ? 0u : 1u, 0u);
  want[i] = 0;
  if (c != ARAW_PASS) ((volatile uint8_t*)code_host)[i] = (uint8_t)c;
}

// ---- keys --------------------------------------------------------------------------------------------------------
// the lowered rune at b[*k] (utf8.DecodeRune: an invalid byte is U+FFFD, width 1), *k advanced past it
__device__ __forceinline__ uint32_t araw_key_rune(const uint8_t* b, uint32_t* k, uint32_t e) {
  uint32_t w;
  const uint32_t r = raw_decode_rune(b + *k, e - *k, &w);
  *k += w;
  return case_lower(r);
}
__device__ __forceinline__ uint64_t araw_key_hash(const uint8_t* b, uint2 s) {
  uint64_t h = 1469598103934665603ull;
  for (uint32_t k = s.x; k < s.y;) h = (h ^ araw_key_rune(b, &k, s.y)) * 1099511628211ull;
  return h;
}
// the same key: the same lowered runes (spans in two buffers)
__device__ __forceinline__ bool araw_key_same(const uint8_t* bx, uint2 x, const uint8_t* by, uint2 y) {
  uint32_t i = x.x, j = y.x;
  while (i < x.y && j < y.y)
    if (araw_key_rune(bx, &i, x.y) != araw_key_rune(by, &j, y.y)) return false;
  return i == x.y && j == y.y;
}
// strings.TrimSpace over UTF-8
__device__ __forceinline__ uint2 araw_trim(const uint8_t* b, uint32_t a, uint32_t e) {
  uint32_t w;
  while (a < e && raw_space(raw_decode_rune(b + a, e - a, &w))) a += w;
  while (e > a && raw_space(raw_decode_last_rune(b + a, e - a, &w))) e -= w;
  return make_uint2(a, e);
}
// strings.Fields over [a, e): calls f(start, end) per field, in order; returns the count
template <class F>
__device__ __forceinline__ uint32_t araw_fields(const uint8_t* b, uint32_t a, uint32_t e, F f) {
  uint32_t n = 0, start = 0, w;
  bool in = false;
  for (uint32_t k = a; k < e; k += w) {
    const bool sp = raw_space(raw_decode_rune(b + k, e - k, &w));
    if (!sp && !in) start = k;
    if (sp && in) f(n++, start, k);
    in = !sp;
  }
  if (in) f(n++, start, e);
  return n;
}

struct ArawKeysArgs {
  const uint32_t* egm_off;  // [n_egm * KVG_AEGM_FIELDS + 1]
  const uint16_t* egm_state;
  const uint8_t* egm_bytes;
  uint32_t n_egm;
  const uint32_t* id_off;   // [n_ids + 1]
  const uint8_t* id_bytes;
  uint32_t n_ids;
  uint32_t* list_off;       // [n_egm + 1]: k_pci_allocate_check's egm_off
  uint32_t* list;           // [list_off[n_egm]]: its egm_gpu (the probe slot of each field while the table fills)
  uint2* tok;               // [..]: each list position's field span; {1, 0} for ARAW_NEVER
  uint32_t* tok_entry;      // [..]: the entry of each list position
  uint32_t* rank;           // [..]: the handle of each first appearance
  uint64_t* table;          // [mask + 1] words [1][lowest list position with the key]; 0 = free
  uint32_t mask;
  uint32_t* ids_out;        // [n_ids]: k_pci_allocate_check's ids
  uint8_t* kept_host;       // [n_egm]
  unsigned long long* verdict_host;  // {miss, range}: (entry << 8) | field, lowest first; ~0 = none
  uint32_t* seq_host;       // NULL: the caller waits for a later kernel
  uint32_t seq;
};

// k_araw_keys' work for n_egm entries spanning nb_egm bytes (host side): a field takes a byte and a space at least, a
// list not kept one handle, so nb_egm + n_egm bounds the list positions (n_list); the key table has `slots` words.
struct ArawKeysSize {
  size_t n_list, slots;
};
inline ArawKeysSize araw_keys_size(uint32_t n_egm, size_t nb_egm) {
  const size_t n_list = n_egm ? nb_egm + n_egm : 0;
  return {n_list, raw_slots(n_list)};
}
// k_araw_keys' arguments: the EGM and ID tables where the kernel reads them, work arrays of araw_keys_size, the host
// outputs, and the sequence word, which the key kernel writes only when no request follows it to the check kernel
inline ArawKeysArgs araw_keys_args(const ArawKeysSize& ks, const uint32_t* egm_off, const uint16_t* egm_state,
                                   const uint8_t* egm_bytes, uint32_t n_egm, const uint32_t* id_off,
                                   const uint8_t* id_bytes, uint32_t n_ids, uint32_t* list_off, uint32_t* list,
                                   uint2* tok, uint32_t* tok_entry, uint32_t* rank, uint64_t* table, uint32_t* ids_out,
                                   uint8_t* kept_host, unsigned long long* verdict_host, uint32_t n_reqs,
                                   uint32_t* seq_word, uint32_t seq) {
  return {egm_off, egm_state, egm_bytes, n_egm, id_off, id_bytes, n_ids, list_off, list, tok, tok_entry, rank, table,
          (uint32_t)(ks.slots - 1), ids_out, kept_host, verdict_host, n_reqs ? nullptr : seq_word, seq};
}

// discoverEGMDevicesFunc's rule for entry e: the number of fields of a kept entry, 0 for any other.  `miss` (NULL: do
// not note) receives the reads it reaches that were not made.
__device__ __forceinline__ uint32_t araw_egm_entry(const ArawKeysArgs& a, uint32_t e, unsigned long long* miss) {
  const uint8_t* b = a.egm_bytes;
  const uint32_t* o = a.egm_off + (size_t)e * KVG_AEGM_FIELDS;
  const uint32_t st = __ldg(&a.egm_state[e]);
  const uint32_t na = o[KVG_AEGM_NAME];
  if (o[KVG_AEGM_NAME + 1] - na < 3 || b[na] != 'e' || b[na + 1] != 'g' || b[na + 2] != 'm') return 0;  // :134
  if (!(st >> KVG_AEGM_GPUS & 1u)) {
    if (miss) atomicMin(miss, ((unsigned long long)e << 8) | KVG_AEGM_GPUS);
    return 0;
  }
  if (st >> (8 + KVG_AEGM_GPUS) & 1u) return 0;  // :137-141
  const uint32_t n = araw_fields(b, o[KVG_AEGM_GPUS], o[KVG_AEGM_GPUS + 1], [](uint32_t, uint32_t, uint32_t) {});
  if (n == 0) return 0;  // :142-145
  if (!(st >> KVG_AEGM_STAT & 1u)) {
    if (miss) atomicMin(miss, ((unsigned long long)e << 8) | KVG_AEGM_STAT);
    return 0;
  }
  return (st >> (8 + KVG_AEGM_STAT) & 1u) ? 0 : n;  // :146-150
}

__global__ void __launch_bounds__(ARAW_KEY_THREADS) k_araw_keys(ArawKeysArgs a) {
  pdl_enter();
  __shared__ uint32_t s[ARAW_KEY_THREADS / 32 + 1];
  __shared__ unsigned long long s_miss, s_range;
  const uint32_t t = threadIdx.x;
  if (t == 0) s_miss = s_range = ~0ull;
  for (uint32_t k = t; k <= a.mask; k += ARAW_KEY_THREADS) a.table[k] = 0;
  __syncthreads();
  // 1. keep or not; list lengths (a kept entry's fields, else one ARAW_NEVER) -> list_off
  uint32_t carry = 0;
  for (uint32_t c = 0; c < a.n_egm; c += ARAW_KEY_THREADS) {
    const uint32_t e = c + t;
    uint32_t len = 0;
    if (e < a.n_egm) {
      const uint32_t nf = araw_egm_entry(a, e, &s_miss);
      ((volatile uint8_t*)a.kept_host)[e] = nf ? 1 : 0;
      len = nf ? nf : 1;
    }
    uint32_t tot;
    const uint32_t x = carry + pref_excl_sum(len, s, tot);
    if (e < a.n_egm) a.list_off[e] = x;
    carry += tot;
  }
  if (t == 0) a.list_off[a.n_egm] = carry;
  __syncthreads();
  const uint32_t n_list = carry;
  // 2. the field spans at their list positions
  for (uint32_t e = t; e < a.n_egm; e += ARAW_KEY_THREADS) {
    const uint32_t at = a.list_off[e];
    const uint32_t* o = a.egm_off + (size_t)e * KVG_AEGM_FIELDS;
    if (araw_egm_entry(a, e, nullptr)) {
      araw_fields(a.egm_bytes, o[KVG_AEGM_GPUS], o[KVG_AEGM_GPUS + 1], [&](uint32_t j, uint32_t x, uint32_t y) {
        a.tok[at + j] = make_uint2(x, y);
        a.tok_entry[at + j] = e;
      });
    } else {
      a.tok[at] = make_uint2(1, 0);
      a.tok_entry[at] = e;
    }
  }
  __syncthreads();
  // 3. every field into the table: the slot of its key, whose word ends as the lowest position with that key
  for (uint32_t k = t; k < n_list; k += ARAW_KEY_THREADS) {
    const uint2 sp = a.tok[k];
    if (sp.y < sp.x) continue;
    const unsigned long long mine = (1ull << 32) | k;
    unsigned long long* cas = reinterpret_cast<unsigned long long*>(a.table);
    for (uint32_t slot = (uint32_t)araw_key_hash(a.egm_bytes, sp) & a.mask;; slot = (slot + 1) & a.mask) {
      unsigned long long w = ld_relaxed_u64(a.table + slot);
      if (w == 0) {
        w = atomicCAS(cas + slot, 0ull, mine);
        if (w == 0) {
          a.list[k] = slot;
          break;
        }
      }
      if (araw_key_same(a.egm_bytes, sp, a.egm_bytes, a.tok[(uint32_t)w])) {
        atomicMin(cas + slot, mine);
        a.list[k] = slot;
        break;
      }
    }
  }
  __syncthreads();
  // 4. handles: first appearances in list order -> 0, 1, ...; one beyond the cap is the range error of its entry
  carry = 0;
  for (uint32_t c = 0; c < n_list; c += ARAW_KEY_THREADS) {
    const uint32_t k = c + t;
    bool first = false;
    if (k < n_list) {
      const uint2 sp = a.tok[k];
      first = sp.y >= sp.x && (uint32_t)ld_relaxed_u64(a.table + a.list[k]) == k;
    }
    uint32_t tot;
    const uint32_t h = carry + pref_excl_sum(first ? 1u : 0u, s, tot);
    if (first) {
      a.rank[k] = h;
      if (h >= KVG_ALLOC_RAW_MAX_EGM_KEYS)
        atomicMin(&s_range, ((unsigned long long)a.tok_entry[k] << 8) | KVG_AEGM_GPUS);
    }
    carry += tot;
  }
  __syncthreads();
  // 5. the lists, and every ID's handle
  for (uint32_t k = t; k < n_list; k += ARAW_KEY_THREADS) {
    const uint2 sp = a.tok[k];
    const uint32_t h = sp.y < sp.x ? ARAW_NEVER : a.rank[(uint32_t)ld_relaxed_u64(a.table + a.list[k])];
    a.list[k] = min(h, ARAW_NEVER);
  }
  for (uint32_t j = t; j < a.n_ids; j += ARAW_KEY_THREADS) {
    const uint2 sp = araw_trim(a.id_bytes, a.id_off[j], a.id_off[j + 1]);
    uint32_t h = ARAW_NOT_EGM;
    for (uint32_t slot = (uint32_t)araw_key_hash(a.id_bytes, sp) & a.mask;; slot = (slot + 1) & a.mask) {
      const unsigned long long w = ld_relaxed_u64(a.table + slot);
      if (w == 0) break;
      if (araw_key_same(a.id_bytes, sp, a.egm_bytes, a.tok[(uint32_t)w])) {
        const uint32_t r = a.rank[(uint32_t)w];
        h = r < ARAW_NEVER ? r : ARAW_NOT_EGM;
        break;
      }
    }
    a.ids_out[j] = h;
  }
  __syncthreads();
  if (t == 0) {
    ((volatile unsigned long long*)a.verdict_host)[0] = s_miss;
    ((volatile unsigned long long*)a.verdict_host)[1] = s_range;
  }
  __threadfence_system();  // the kept bytes and verdicts are on their way before the sequence word
  __syncthreads();
  if (t == 0 && a.seq_host) {
    __threadfence_system();
    *((volatile uint32_t*)a.seq_host) = a.seq;
  }
}

}  // namespace kvg
