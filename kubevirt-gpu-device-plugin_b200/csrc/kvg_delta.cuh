// kvg_delta.cuh — K7: the keyed diff of two scans (kvg_scan_pci_delta, kvg_scan_mdev_delta,
// kvg_dev_scan_pci_shard_fetch_delta, kvg_dev_scan_mdev_shard_fetch_delta).
//
//   k_delta_merge<Tr>  merge path over the previous scan's survivors and the new ones (ascending key), one change
//                      entry per key whose survivor differs, compacted in key order by the look-back tile body of
//                      kvg_common.cuh; every entry tags the keys of the two group-by maps whose member sequence it
//                      changes.  Also checks that the new list ascends strictly.  Tr is the record trait:
//                      PciDeltaRec (16-byte survivors keyed by address) or MdevDeltaRec (32-byte survivors keyed by
//                      the 128-bit big-endian UUID).
//   k_delta_merge_shard<Tr>  the same merge over a rank's three lists, one per blockIdx.y: its local survivors
//                      (change entries), the members of the two kinds of keys it owns (key tags only)
//   k_delta_lists      the four key lists (dirty / gone of both maps) from those tags: one look-back compaction per
//                      list (blockIdx.y) through the same tile body
//   k_mdev_delta_types the previous result's type keys in the new key space: same sanitised label, or none
//   k_raw_rekey<MDEV>, k_raw_xlate<MDEV>  kvg_scan_pci_raw_delta / kvg_scan_mdev_raw_delta outside the all-numeric
//                      pair: both snapshots' survivors onto the entry-name space they share (PciRawDeltaRec /
//                      MdevRawDeltaRec), and each previous key to the new key with the same string
#pragma once
#include "../../include/kvgpu.h"
#include "kvg_common.cuh"
#include "kvg_order.cuh"
#include "kvg_scan.cuh"

namespace kvg {

constexpr int DELTA_THREADS = 128, DELTA_ROWS = 8;
constexpr uint32_t DELTA_TILE = DELTA_THREADS * DELTA_ROWS;  // merged positions per CTA
constexpr uint32_t DELTA_NONE = 0xffffffffu;
// ScanCtrl::reserved2 words the delta kernels write: change count, "new list not ascending", the four list lengths
enum : uint32_t { DELTA_W_CHANGES = 8, DELTA_W_ERROR = 9, DELTA_W_LISTS = 10 };

// index of `key` in the ascending distinct keys, or DELTA_NONE
__device__ __forceinline__ uint32_t delta_find(const uint32_t* keys, uint32_t n, uint32_t key) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(&keys[mid]) < key)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo < n && __ldg(&keys[lo]) == key ? lo : DELTA_NONE;
}

// The distinct keys of one group-by map in both results, with one tag word per key: a key is marked by storing
// the call's tag, so the words never need clearing.
struct DeltaKeys {
  const uint32_t* keys_now;  // the new result's keys (ascending)
  uint32_t n_now;
  uint32_t* flag_now;        // tag: dirty
  const uint32_t* keys_prev; // the previous result's keys
  uint32_t n_prev;
  uint32_t* flag_prev;       // tag: gone
  // mark<true>: previous key -> the new key that is the same key, or DELTA_NONE (type ids: same label)
  const uint32_t* xlate;

  // A change entry whose member left key `prev_key` and joined key `now_key` (either side may be absent):
  // the key it joined is dirty; the key it left is dirty if it still exists, else gone.  XLATE: prev_key is
  // translated into the new key space first; without it a key means the same thing in both results.
  template <bool XLATE = false>
  __device__ __forceinline__ void mark(bool has_now, uint32_t now_key, bool has_prev, uint32_t prev_key,
                                       uint32_t tag) const {
    if (has_now) {
      const uint32_t k = delta_find(keys_now, n_now, now_key);
      if (k != DELTA_NONE) flag_now[k] = tag;
    }
    const uint32_t same = XLATE && has_prev ? __ldg(&xlate[prev_key]) : prev_key;
    if (has_prev && !(has_now && same == now_key)) {
      uint32_t k = XLATE && same == DELTA_NONE ? DELTA_NONE : delta_find(keys_now, n_now, same);
      if (k != DELTA_NONE)
        flag_now[k] = tag;
      else if ((k = delta_find(keys_prev, n_prev, prev_key)) != DELTA_NONE)
        flag_prev[k] = tag;
    }
  }
  // mark<true> when both keys are already indices into keys_now / keys_prev (the re-keyed raw delta): no searches
  __device__ __forceinline__ void mark_index(bool has_now, uint32_t now_k, bool has_prev, uint32_t prev_k,
                                             uint32_t tag) const {
    if (has_now) flag_now[now_k] = tag;
    if (!has_prev) return;
    const uint32_t same = __ldg(&xlate[prev_k]);
    if (has_now && same == now_k) return;
    if (same != DELTA_NONE)
      flag_now[same] = tag;
    else
      flag_prev[prev_k] = tag;
  }
};

// ---- record traits of k_delta_merge ------------------------------------------------------------------------
//   Rec                       one survivor (what the CTA stages in shared memory)
//   Key key(rec), key_at(list, i), le(a, b), eq(a, b)   the merge key and its order
//   ld(p) / ldg(p)            streaming / read-only loads of one survivor
//   diff(p, q, k0)            KVG_CH_* bits of two survivors with the same key
//   emit(out, pos, ...)       the change entry (OUT_UNITS x 16 bytes) and the keys of both maps it dirties

// kvg_pci_surv: {addr, group, device | numa << 16, name}; key = addr; maps: deviceMap, iommuMap
struct PciDeltaRec {
  using Rec = uint4;
  using Key = uint32_t;
  static constexpr uint32_t OUT_UNITS = 2;
  __device__ __forceinline__ static Key key(const Rec& r) { return r.x; }
  __device__ __forceinline__ static Key key_at(const Rec* list, uint32_t i) {
    return __ldg(reinterpret_cast<const uint32_t*>(list + i));
  }
  __device__ __forceinline__ static bool le(Key a, Key b) { return a <= b; }
  __device__ __forceinline__ static bool eq(Key a, Key b) { return a == b; }
  __device__ __forceinline__ static Rec ld(const Rec* p) { return ld_stream(p); }
  __device__ __forceinline__ static Rec ldg(const Rec* p) { return __ldg(p); }
  __device__ __forceinline__ static uint32_t diff(const Rec& p, const Rec& q, const DeltaKeys&) {
    return (p.y != q.y ? (uint32_t)KVG_CH_GROUP : 0u) | ((p.z & 0xffffu) != (q.z & 0xffffu) ? (uint32_t)KVG_CH_DEVICE : 0u) |
           ((p.z >> 16) != (q.z >> 16) ? (uint32_t)KVG_CH_NUMA : 0u);
  }
  // kvgpu.h kvg_pci_change; a key is dirty iff the (addr, numa) sequence of its members changed
  __device__ __forceinline__ static void emit(uint4* out, uint32_t pos, uint32_t what, bool hp, bool hn, uint32_t a,
                                              uint32_t b, const Rec& p, const Rec& q, const DeltaKeys& dev,
                                              const DeltaKeys& grp, uint32_t tag) {
    st_stream(out + 2 * (size_t)pos, make_uint4(hp ? p.x : q.x, what, p.y, q.y));
    st_stream(out + 2 * (size_t)pos + 1,
              make_uint4((p.z & 0xffffu) | (q.z << 16), (p.z >> 16) | (q.z & 0xffff0000u), b, a));
    mark(what, hp, hn, p, q, dev, grp, tag);
  }
  // the keys alone (the sharded merge's owned lists tag keys and write no entry)
  __device__ __forceinline__ static void mark(uint32_t what, bool hp, bool hn, const Rec& p, const Rec& q,
                                              const DeltaKeys& dev, const DeltaKeys& grp, uint32_t tag) {
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_DEVICE | KVG_CH_NUMA))
      dev.mark(hn, q.z & 0xffffu, hp, p.z & 0xffffu, tag);
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_GROUP | KVG_CH_NUMA)) grp.mark(hn, q.y, hp, p.y, tag);
  }
};

// kvg_mdev_surv: lo = the UUID bytes, hi = {parent, type_key | numa << 16, src, pad}; key = the UUID as a 128-bit
// big-endian number (Walk order), i.e. each little-endian word byte-swapped; maps: vGpuMap (type ids, translated
// by label), gpuVgpuMap (parent handles)
struct MdevDeltaRec {
  using Rec = MdevItem;
  struct Key {
    uint64_t hi, lo;
  };
  static constexpr uint32_t OUT_UNITS = 3;
  __device__ __forceinline__ static Key key_of(const uint4& u) {
    return {((uint64_t)__byte_perm(u.x, 0, 0x0123) << 32) | __byte_perm(u.y, 0, 0x0123),
            ((uint64_t)__byte_perm(u.z, 0, 0x0123) << 32) | __byte_perm(u.w, 0, 0x0123)};
  }
  __device__ __forceinline__ static Key key(const Rec& r) { return key_of(r.lo); }
  __device__ __forceinline__ static Key key_at(const Rec* list, uint32_t i) { return key_of(__ldg(&list[i].lo)); }
  __device__ __forceinline__ static bool le(Key a, Key b) { return a.hi < b.hi || (a.hi == b.hi && a.lo <= b.lo); }
  __device__ __forceinline__ static bool eq(Key a, Key b) { return a.hi == b.hi && a.lo == b.lo; }
  __device__ __forceinline__ static Rec ld(const Rec* p) {
    const uint4* u = reinterpret_cast<const uint4*>(p);
    return {ld_stream(u), ld_stream(u + 1)};
  }
  __device__ __forceinline__ static Rec ldg(const Rec* p) {
    const uint4* u = reinterpret_cast<const uint4*>(p);
    return {__ldg(u), __ldg(u + 1)};
  }
  // the label decides the type: type.xlate maps a previous canonical id to the new one with the same label
  __device__ __forceinline__ static uint32_t diff(const Rec& p, const Rec& q, const DeltaKeys& type) {
    return (__ldg(&type.xlate[p.hi.y & 0xffffu]) != (q.hi.y & 0xffffu) ? (uint32_t)KVG_CH_TYPE : 0u) |
           (p.hi.x != q.hi.x ? (uint32_t)KVG_CH_PARENT : 0u) |
           ((p.hi.y >> 16) != (q.hi.y >> 16) ? (uint32_t)KVG_CH_NUMA : 0u);
  }
  // kvgpu.h kvg_mdev_change; a vGpuMap key is dirty iff its (uuid, numa) sequence changed, a gpuVgpuMap key iff
  // its uuid sequence did
  __device__ __forceinline__ static void emit(uint4* out, uint32_t pos, uint32_t what, bool hp, bool hn, uint32_t a,
                                              uint32_t b, const Rec& p, const Rec& q, const DeltaKeys& type,
                                              const DeltaKeys& par, uint32_t tag) {
    st_stream(out + 3 * (size_t)pos, hp ? p.lo : q.lo);
    st_stream(out + 3 * (size_t)pos + 1, make_uint4(what, p.hi.x, q.hi.x, (p.hi.y & 0xffffu) | (q.hi.y << 16)));
    st_stream(out + 3 * (size_t)pos + 2, make_uint4((p.hi.y >> 16) | (q.hi.y & 0xffff0000u), b, a, 0u));
    mark(what, hp, hn, p, q, type, par, tag);
  }
  // the keys alone (the sharded merge's owned lists tag keys and write no entry)
  __device__ __forceinline__ static void mark(uint32_t what, bool hp, bool hn, const Rec& p, const Rec& q,
                                              const DeltaKeys& type, const DeltaKeys& par, uint32_t tag) {
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_TYPE | KVG_CH_NUMA))
      type.mark<true>(hn, q.hi.y & 0xffffu, hp, p.hi.y & 0xffffu, tag);
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_PARENT)) par.mark(hn, q.hi.x, hp, p.hi.x, tag);
  }
};

// The re-keyed PCI survivor of kvg_scan_pci_raw_delta (k_raw_rekey): {name rank, index of its group in the side's
// grp_keys, index of its device id in the side's dev_keys | numa << 16, the side's own address handle}; key = the
// name rank, which two snapshots share.  A previous key index goes to the new key index with the same string through
// DeltaKeys::xlate: k0.xlate is the whole table (previous device indices from 0, previous group indices from
// RAW_XLATE_GROUP), so that diff, which sees k0 only, reads both; k1.xlate points at the group part.
constexpr uint32_t RAW_XLATE_GROUP = 65536;
struct PciRawDeltaRec : PciDeltaRec {
  __device__ __forceinline__ static uint32_t diff(const Rec& p, const Rec& q, const DeltaKeys& dev) {
    const uint32_t* xl = dev.xlate;
    return (__ldg(&xl[RAW_XLATE_GROUP + p.y]) != q.y ? (uint32_t)KVG_CH_GROUP : 0u) |
           (__ldg(&xl[p.z & 0xffffu]) != (q.z & 0xffffu) ? (uint32_t)KVG_CH_DEVICE : 0u) |
           ((p.z >> 16) != (q.z >> 16) ? (uint32_t)KVG_CH_NUMA : 0u);
  }
  // kvg_pci_change with each side's own handles: the new address when the name survives now, else the previous one
  __device__ __forceinline__ static void emit(uint4* out, uint32_t pos, uint32_t what, bool hp, bool hn, uint32_t a,
                                              uint32_t b, const Rec& p, const Rec& q, const DeltaKeys& dev,
                                              const DeltaKeys& grp, uint32_t tag) {
    const uint32_t pg = hp ? __ldg(&grp.keys_prev[p.y]) : 0u, ng = hn ? __ldg(&grp.keys_now[q.y]) : 0u;
    const uint32_t pd = hp ? __ldg(&dev.keys_prev[p.z & 0xffffu]) : 0u, nd = hn ? __ldg(&dev.keys_now[q.z & 0xffffu]) : 0u;
    st_stream(out + 2 * (size_t)pos, make_uint4(hn ? q.w : p.w, what, pg, ng));
    st_stream(out + 2 * (size_t)pos + 1, make_uint4(pd | (nd << 16), (p.z >> 16) | (q.z & 0xffff0000u), b, a));
    mark(what, hp, hn, p, q, dev, grp, tag);
  }
  __device__ __forceinline__ static void mark(uint32_t what, bool hp, bool hn, const Rec& p, const Rec& q,
                                              const DeltaKeys& dev, const DeltaKeys& grp, uint32_t tag) {
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_DEVICE | KVG_CH_NUMA))
      dev.mark_index(hn, q.z & 0xffffu, hp, p.z & 0xffffu, tag);
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_GROUP | KVG_CH_NUMA)) grp.mark_index(hn, q.y, hp, p.y, tag);
  }
};

// The re-keyed mdev survivor of kvg_scan_mdev_raw_delta: lo = the UUID bytes, hi = {index of its parent in the side's
// par_keys, canonical type id | numa << 16, name rank, 0}; key = the name rank.  k0.xlate is the table of the merge:
// previous canonical type ids -> new ones by label (k_mdev_delta_types) from 0, previous parent indices -> new ones
// by string from RAW_XLATE_GROUP; k1.xlate points at the parent part.
struct MdevRawDeltaRec : MdevDeltaRec {
  using Key = uint32_t;
  __device__ __forceinline__ static Key key(const Rec& r) { return r.hi.z; }
  __device__ __forceinline__ static Key key_at(const Rec* list, uint32_t i) { return __ldg(&list[i].hi.z); }
  __device__ __forceinline__ static bool le(Key a, Key b) { return a <= b; }
  __device__ __forceinline__ static bool eq(Key a, Key b) { return a == b; }
  __device__ __forceinline__ static uint32_t diff(const Rec& p, const Rec& q, const DeltaKeys& type) {
    const uint32_t* xl = type.xlate;
    return (__ldg(&xl[p.hi.y & 0xffffu]) != (q.hi.y & 0xffffu) ? (uint32_t)KVG_CH_TYPE : 0u) |
           (__ldg(&xl[RAW_XLATE_GROUP + p.hi.x]) != q.hi.x ? (uint32_t)KVG_CH_PARENT : 0u) |
           ((p.hi.y >> 16) != (q.hi.y >> 16) ? (uint32_t)KVG_CH_NUMA : 0u);
  }
  // kvg_mdev_change with each side's own parent handles: the new UUID bytes when the name survives now
  __device__ __forceinline__ static void emit(uint4* out, uint32_t pos, uint32_t what, bool hp, bool hn, uint32_t a,
                                              uint32_t b, const Rec& p, const Rec& q, const DeltaKeys& type,
                                              const DeltaKeys& par, uint32_t tag) {
    const uint32_t pp = hp ? __ldg(&par.keys_prev[p.hi.x]) : 0u, np = hn ? __ldg(&par.keys_now[q.hi.x]) : 0u;
    st_stream(out + 3 * (size_t)pos, hn ? q.lo : p.lo);
    st_stream(out + 3 * (size_t)pos + 1, make_uint4(what, pp, np, (p.hi.y & 0xffffu) | (q.hi.y << 16)));
    st_stream(out + 3 * (size_t)pos + 2, make_uint4((p.hi.y >> 16) | (q.hi.y & 0xffff0000u), b, a, 0u));
    mark(what, hp, hn, p, q, type, par, tag);
  }
  __device__ __forceinline__ static void mark(uint32_t what, bool hp, bool hn, const Rec& p, const Rec& q,
                                              const DeltaKeys& type, const DeltaKeys& par, uint32_t tag) {
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_TYPE | KVG_CH_NUMA))
      type.mark<true>(hn, q.hi.y & 0xffffu, hp, p.hi.y & 0xffffu, tag);
    if (what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_PARENT)) par.mark_index(hn, q.hi.x, hp, p.hi.x, tag);
  }
};

// previous-list elements among the first d merged positions; equal keys take the previous element first
template <class Tr>
__device__ __forceinline__ uint32_t delta_split(const typename Tr::Rec* a, uint32_t na, const typename Tr::Rec* b,
                                                uint32_t nb, uint32_t d) {
  uint32_t lo = d > nb ? d - nb : 0, hi = min(d, na);
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (Tr::le(Tr::key_at(a, mid), Tr::key_at(b, d - 1 - mid)))
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// The merged sequence as a classify operator: record i of the tile front-end is merged position i.  The CTA has
// staged its previous-list slice [i0, i0 + na) and new-list slice [j0, j0 + nb) in s_rec and the merge in s_code
// (bit 31: new list, low bits: index in that list).  An equal pair is adjacent in the merge, previous first:
//   previous element a at position i: matched iff the new element b = i - a (the next one at its merge position)
//                                     has its key -> it reports the pair, if the pair differs
//   new element b at position i:      matched iff the previous element i - b - 1 has its key -> silent
// Either neighbour may lie outside the CTA's slice and is then read from global memory.
template <class Tr>
struct DeltaMergeOp {
  using Rec = typename Tr::Rec;
  struct Item {
    uint32_t code, what;
  };
  const Rec* prev;
  uint32_t n_prev;
  const Rec* now;
  uint32_t n_now;
  uint32_t n;    // merged positions: n_prev + n_now
  uint4* out;    // the change entries, Tr::OUT_UNITS x 16 bytes each
  ScanCtrl* ctrl;
  DeltaKeys k0, k1;  // the two group-by maps (PCI: deviceMap, iommuMap; mdev: vGpuMap, gpuVgpuMap)
  uint32_t tag;
  const Rec* s_rec;
  const uint32_t* s_code;
  uint32_t d0, i0, na, j0, nb;

  __device__ __forceinline__ Rec rec_prev(uint32_t a) const { return a - i0 < na ? s_rec[a - i0] : Tr::ldg(prev + a); }
  __device__ __forceinline__ Rec rec_now(uint32_t b) const { return b - j0 < nb ? s_rec[na + b - j0] : Tr::ldg(now + b); }

  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    Item it = {0u, 0u};
    if (!ok || i - d0 >= na + nb) return it;
    const uint32_t code = s_code[i - d0], x = code & 0x7fffffffu;
    it.code = code;
    if (code >> 31) {
      const uint32_t a = i - x;  // previous-list elements before it
      if (a == 0 || !Tr::eq(Tr::key(rec_prev(a - 1)), Tr::key(rec_now(x)))) it.what = KVG_CH_ADDED;
    } else {
      const uint32_t b = i - x;  // new-list elements before it
      const Rec p = rec_prev(x);
      if (b >= n_now) {
        it.what = KVG_CH_REMOVED;
      } else {
        const Rec q = rec_now(b);
        it.what = !Tr::eq(Tr::key(q), Tr::key(p)) ? (uint32_t)KVG_CH_REMOVED : Tr::diff(p, q, k0);
      }
    }
    return it;
  }
  __device__ __forceinline__ bool pred(const Item& it, uint32_t) const { return it.what != 0; }
  __device__ __forceinline__ uint32_t prepare(const Item&) const { return 0; }
  // the change at merged position i: ENTRY, its entry at `pos` and the keys it dirties; otherwise the keys alone
  template <bool ENTRY>
  __device__ __forceinline__ void apply(uint32_t pos, const Item& it, uint32_t i) const {
    const uint32_t x = it.code & 0x7fffffffu;
    const uint32_t a = (it.code >> 31) ? DELTA_NONE : x;
    const uint32_t b = (it.code >> 31) ? x : ((it.what & KVG_CH_REMOVED) ? DELTA_NONE : i - x);
    const bool hp = a != DELTA_NONE, hn = b != DELTA_NONE;
    const Rec p = hp ? rec_prev(a) : Rec{};
    const Rec q = hn ? rec_now(b) : Rec{};
    if constexpr (ENTRY)
      Tr::emit(out, pos, it.what, hp, hn, a, b, p, q, k0, k1, tag);
    else
      Tr::mark(it.what, hp, hn, p, q, k0, k1, tag);
  }
  __device__ __forceinline__ void emit(uint32_t pos, const Item& it, uint32_t i, uint32_t) const {
    apply<true>(pos, it, i);
  }
  __device__ __forceinline__ void tile_epilogue() {}
  __device__ __forceinline__ void finish(uint32_t total) { ctrl->reserved2[DELTA_W_CHANGES] = total; }
};

// Stage merge tile `tile` of o in the CTA: the two diagonal searches, both list slices in s_rec (checking that the
// new one ascends strictly) and the merge codes in s_code.  Sets o's slice fields and shared-memory pointers.
template <class Tr>
__device__ __forceinline__ void delta_stage(DeltaMergeOp<Tr>& o, uint32_t tile, typename Tr::Rec* s_rec,
                                            uint32_t* s_code, uint32_t* s_split) {
  using Rec = typename Tr::Rec;
  const uint32_t d0 = tile * DELTA_TILE, d1 = min(o.n, d0 + DELTA_TILE);
  if (threadIdx.x == 0 || threadIdx.x == 32) {
    const uint32_t hi = threadIdx.x != 0;
    s_split[hi] = delta_split<Tr>(o.prev, o.n_prev, o.now, o.n_now, hi ? d1 : d0);
  }
  __syncthreads();
  const uint32_t i0 = s_split[0], i1 = s_split[1];
  o.d0 = d0;
  o.i0 = i0;
  o.j0 = d0 - i0;
  if (i1 < i0 || i1 - i0 > d1 - d0) {  // out-of-order diagonals: only an unordered new list makes them
    if (threadIdx.x == 0) o.ctrl->reserved2[DELTA_W_ERROR] = 1u;
    o.na = o.nb = 0;
  } else {
    o.na = i1 - i0;
    o.nb = (d1 - d0) - o.na;
  }
  for (uint32_t k = threadIdx.x; k < o.na + o.nb; k += DELTA_THREADS) {
    if (k < o.na) {
      s_rec[k] = Tr::ld(o.prev + o.i0 + k);
    } else {
      const uint32_t b = o.j0 + (k - o.na);
      const Rec r = Tr::ld(o.now + b);
      s_rec[k] = r;
      if (b > 0 && Tr::le(Tr::key(r), Tr::key_at(o.now, b - 1))) o.ctrl->reserved2[DELTA_W_ERROR] = 1u;  // strict ascent
    }
  }
  __syncthreads();
  {  // each thread merges DELTA_ROWS consecutive positions from its own diagonal
    const uint32_t na = o.na, nb = o.nb, cnt = na + nb;
    const uint32_t p0 = min(cnt, threadIdx.x * DELTA_ROWS), p1 = min(cnt, p0 + DELTA_ROWS);
    uint32_t lo = p0 > nb ? p0 - nb : 0, hi = min(p0, na);
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (Tr::le(Tr::key(s_rec[mid]), Tr::key(s_rec[na + p0 - 1 - mid])))
        lo = mid + 1;
      else
        hi = mid;
    }
    uint32_t ia = lo, ib = p0 - lo;
    for (uint32_t p = p0; p < p1; p++) {
      const bool take_prev = ib >= nb || (ia < na && Tr::le(Tr::key(s_rec[ia]), Tr::key(s_rec[na + ib])));
      s_code[p] = take_prev ? o.i0 + ia++ : (0x80000000u | (o.j0 + ib++));
    }
  }
  __syncthreads();
  o.s_rec = s_rec;
  o.s_code = s_code;
}

// One CTA per DELTA_TILE merged positions.  O(n_prev + n_now): two diagonal searches per CTA, a shared-memory merge,
// one pass of the look-back compaction.  The tag doubles as the look-back epoch.  Static shared memory: DELTA_TILE
// staged survivors (16 KiB PCI, 32 KiB mdev) and the merge codes (4 KiB).
template <class Tr>
__global__ void __launch_bounds__(DELTA_THREADS) k_delta_merge(DeltaMergeOp<Tr> op, uint64_t* tile_state) {
  using Rec = typename Tr::Rec;
  pdl_enter();
  __shared__ Rec s_rec[DELTA_TILE];
  __shared__ uint32_t s_code[DELTA_TILE];
  __shared__ uint32_t s_split[2];
  __shared__ uint32_t s_wtot[DELTA_THREADS / 32], s_woff[DELTA_THREADS / 32];
  __shared__ uint32_t s_base;
  DeltaMergeOp<Tr> o = op;
  const uint32_t n_tiles = (o.n + DELTA_TILE - 1) / DELTA_TILE, tile = blockIdx.x;
  if (n_tiles == 0) {
    if (tile == 0 && threadIdx.x == 0) o.finish(0);
    return;
  }
  if (tile >= n_tiles) return;
  delta_stage<Tr>(o, tile, s_rec, s_code, s_split);
  lookback_tile<DeltaMergeOp<Tr>, DELTA_THREADS, DELTA_ROWS>(o, tile, n_tiles, tile_state, o.tag, s_wtot, s_woff, s_base);
}

// The launch arguments below are built on the host, by kvg_api_delta.inc and by the CPU emulator alike.

// k_delta_merge's operator over prev[0, n_prev) and now[0, n_now) (Tr::Rec in 16-byte units): entries to out, counts
// to ctrl.  keys / n_keys: the distinct keys of the first map now and before, then those of the second map; flag:
// their tag words in the same order; xlate: the first map's cross-map (mdev type ids) or NULL; tag: never repeated.
template <class Tr>
inline DeltaMergeOp<Tr> delta_merge_op(const uint4* prev, uint32_t n_prev, const uint4* now, uint32_t n_now, uint4* out,
                                       ScanCtrl* ctrl, const uint32_t* const* keys, const uint32_t* n_keys,
                                       uint32_t* const* flag, const uint32_t* xlate, uint32_t tag) {
  DeltaMergeOp<Tr> op = {};
  op.prev = reinterpret_cast<const typename Tr::Rec*>(prev);
  op.n_prev = n_prev;
  op.now = reinterpret_cast<const typename Tr::Rec*>(now);
  op.n_now = n_now;
  op.n = n_prev + n_now;
  op.out = out;
  op.ctrl = ctrl;
  op.k0 = {keys[0], n_keys[0], flag[0], keys[1], n_keys[1], flag[1], xlate};
  op.k1 = {keys[2], n_keys[2], flag[2], keys[3], n_keys[3], flag[3], nullptr};
  op.tag = tag;
  return op;
}
// k_delta_merge's grid over n merged positions: at least one CTA, which writes the zero count
inline uint32_t delta_merge_tiles(uint32_t n) { return n ? (n + DELTA_TILE - 1) / DELTA_TILE : 1; }

// The sharded forms (kvg_dev_scan_pci_shard_fetch_delta, kvg_dev_scan_mdev_shard_fetch_delta): one merge per
// blockIdx.y over one pair of this rank's lists, all three checked for strict ascent.
//   y = 0  the local survivors: change entries through the look-back tile body; its DeltaKeys hold no keys, so it
//          tags none (mdev: k0 still carries the label cross-map that KVG_CH_TYPE reads)
//   y = 1  the members of the owned device ids / type ids: deviceMap / vGpuMap tags only (k1 empty), no entries
//   y = 2  the members of the owned groups / parents: iommuMap / gpuVgpuMap tags only (k0 keyless), no entries
// Each row has its own tile count and its surplus CTAs exit before any look-back.  Only row 0 takes part in one
// (words tile_state[0 ..)), and a tile waits only on earlier tiles of that row, as in k_delta_lists.
template <class Tr>
struct DeltaShardArgs {
  DeltaMergeOp<Tr> o[3];
};
template <class Tr>
__global__ void __launch_bounds__(DELTA_THREADS) k_delta_merge_shard(DeltaShardArgs<Tr> args, uint64_t* tile_state) {
  pdl_enter();
  __shared__ typename Tr::Rec s_rec[DELTA_TILE];
  __shared__ uint32_t s_code[DELTA_TILE];
  __shared__ uint32_t s_split[2];
  __shared__ uint32_t s_wtot[DELTA_THREADS / 32], s_woff[DELTA_THREADS / 32];
  __shared__ uint32_t s_base;
  // picked by value: indexing the parameter array by blockIdx.y made ptxas spill (64 registers, 8-byte stack frame)
  DeltaMergeOp<Tr> o = blockIdx.y == 0 ? args.o[0] : blockIdx.y == 1 ? args.o[1] : args.o[2];
  const uint32_t n_tiles = (o.n + DELTA_TILE - 1) / DELTA_TILE, tile = blockIdx.x;
  if (n_tiles == 0) {
    if (blockIdx.y == 0 && tile == 0 && threadIdx.x == 0) o.finish(0);
    return;
  }
  if (tile >= n_tiles) return;
  delta_stage<Tr>(o, tile, s_rec, s_code, s_split);
  if (blockIdx.y == 0) {
    lookback_tile<DeltaMergeOp<Tr>, DELTA_THREADS, DELTA_ROWS>(o, tile, n_tiles, tile_state, o.tag, s_wtot, s_woff,
                                                               s_base);
    return;
  }
  for (uint32_t k = threadIdx.x; k < o.na + o.nb; k += DELTA_THREADS) {
    const typename DeltaMergeOp<Tr>::Item it = o.load(o.d0 + k, true);
    if (it.what) o.template apply<false>(0, it, o.d0 + k);
  }
}
// The three rows from op, the merge of the local survivors: row 0 is op without keys, its k0 keeping only the
// cross-map; rows 1 and 2 merge prev[y - 1] and now[y - 1], the previous and the new members of the owned keys of the
// first / second map, keep that map's keys and write no entries.  Returns the grid's columns: the longest row's tiles.
template <class Tr>
inline uint32_t delta_shard_args(DeltaShardArgs<Tr>& a, const DeltaMergeOp<Tr>& op, const uint4* const (&prev)[2],
                                 const uint32_t (&n_prev)[2], const uint4* const (&now)[2],
                                 const uint32_t (&n_now)[2]) {
  const DeltaKeys none = {}, xlate_only = {nullptr, 0, nullptr, nullptr, 0, nullptr, op.k0.xlate};
  uint32_t cols = 1;
  for (int y = 0; y < 3; y++) {
    DeltaMergeOp<Tr>& o = a.o[y];
    o = op;
    if (y > 0) {
      o.prev = reinterpret_cast<const typename Tr::Rec*>(prev[y - 1]);
      o.n_prev = n_prev[y - 1];
      o.now = reinterpret_cast<const typename Tr::Rec*>(now[y - 1]);
      o.n_now = n_now[y - 1];
      o.n = o.n_prev + o.n_now;
      o.out = nullptr;
    }
    if (y != 1) o.k0 = xlate_only;
    if (y != 2) o.k1 = none;
    const uint32_t t = delta_merge_tiles(o.n);
    if (t > cols) cols = t;
  }
  return cols;
}

// One of the four key lists: keys whose tag word holds this call's tag, ascending.  Dirty lists give the key's
// index in the new result, gone lists the key itself (u16 device ids, u32 groups).
struct DeltaListOp {
  using Item = uint32_t;
  const uint32_t* flag;
  uint32_t n;
  uint32_t tag;
  const uint32_t* keys;  // NULL: the index goes out
  uint32_t* out32;
  uint16_t* out16;       // non-NULL: the list is u16
  uint32_t* count;

  __device__ __forceinline__ Item load(uint32_t i, bool ok) const { return ok ? flag[i] : 0u; }
  __device__ __forceinline__ bool pred(const Item& f, uint32_t) const { return f == tag; }
  __device__ __forceinline__ uint32_t prepare(const Item&) const { return 0; }
  __device__ __forceinline__ void emit(uint32_t pos, const Item&, uint32_t i, uint32_t) const {
    const uint32_t v = keys ? __ldg(&keys[i]) : i;
    if (out16)
      out16[pos] = (uint16_t)v;
    else
      out32[pos] = v;
  }
  __device__ __forceinline__ void tile_epilogue() {}
  __device__ __forceinline__ void finish(uint32_t total) { *count = total; }
};
struct DeltaListArgs {
  DeltaListOp o[4];  // dirty, gone of the first map (deviceMap / vGpuMap), then of the second
};
// grid (tiles of the longest list, 4); list y uses the look-back words tile_state[y * state_stride ..).  One CTA per
// tile, no tile loop: the loop of lookback_tiles measured 2 % slower here (10.35 against 10.1 us at 1 M records,
// H100 SXM 80 GB with a 700 W power limit).
__global__ void __launch_bounds__(KVG_BLOCK) k_delta_lists(DeltaListArgs args, uint64_t* tile_state, uint32_t state_stride,
                                                           uint32_t epoch) {
  pdl_enter();
  __shared__ uint32_t s_wtot[KVG_WARPS], s_woff[KVG_WARPS];
  __shared__ uint32_t s_base;
  DeltaListOp op = args.o[blockIdx.y];
  const uint32_t n_tiles = (op.n + C_TILE - 1) / C_TILE, tile = blockIdx.x;
  if (n_tiles == 0) {
    if (tile == 0 && threadIdx.x == 0) op.finish(0);
    return;
  }
  if (tile >= n_tiles) return;
  lookback_tile<DeltaListOp, KVG_BLOCK, C_ROWS>(op, tile, n_tiles, tile_state + (size_t)blockIdx.y * state_stride, epoch,
                                                s_wtot, s_woff, s_base);
}
// The four lists of op's two maps, counted into ctrl->reserved2[DELTA_W_LISTS ..]; out: where they go, the first gone
// list as u16 when gone0_u16 (PCI device ids).  Returns the grid's columns: the longest list's tiles.
template <class Tr>
inline uint32_t delta_list_args(DeltaListArgs& la, const DeltaMergeOp<Tr>& op, void* const (&out)[4], bool gone0_u16) {
  uint32_t* cnt = &op.ctrl->reserved2[DELTA_W_LISTS];
  uint32_t cols = 1;
  for (int m = 0; m < 2; m++) {
    const DeltaKeys& k = m ? op.k1 : op.k0;
    const bool u16 = m == 0 && gone0_u16;
    la.o[2 * m] = {k.flag_now, k.n_now, op.tag, nullptr, (uint32_t*)out[2 * m], nullptr, cnt + 2 * m};
    la.o[2 * m + 1] = {k.flag_prev, k.n_prev, op.tag, k.keys_prev, u16 ? nullptr : (uint32_t*)out[2 * m + 1],
                       u16 ? (uint16_t*)out[2 * m + 1] : nullptr, cnt + 2 * m + 1};
    for (const uint32_t n : {k.n_now, k.n_prev}) {
      const uint32_t t = (n + C_TILE - 1) / C_TILE;
      if (t > cols) cols = t;
    }
  }
  return cols;
}

// The previous result's type keys in the new key space.  The canonical ids of two scans are not comparable (each
// numbers its own dictionary), labels are: xlate[c] for every previous type key c is the new type key with a
// byte-identical label, or DELTA_NONE.  kvg_scan_mdev_delta passes the survivors' type keys, so a label that is in
// the new dictionary without a survivor is no key and maps to DELTA_NONE.  The sharded form passes every canonical id
// of both dictionaries: a rank's local survivors may carry types another rank owns, so every id needs its image, and
// DeltaKeys::mark<true> then finds the image among the rank's owned keys or not at all (gone).  One CTA: the new keys
// go into an open-addressed table in global memory (slot = tag << 32 | new key index; a slot holding another call's
// tag is empty, so the table is never cleared), then every previous key probes it.  The FNV-1a hashes of k_mdev_labels place and filter; equality is decided on length and bytes.
// O(KT_prev + KT_now) expected probes.
constexpr uint32_t XMAP_THREADS = 1024;
constexpr uint32_t XMAP_SLOTS = 1u << 17;  // >= 2 x 65,535 type keys
// the table's probe mask for n_keys new keys: at least 64 slots and twice the keys, a power of two
inline uint32_t delta_xmap_mask(uint32_t n_keys) {
  uint32_t slots = 64;
  while (slots < 2 * n_keys) slots <<= 1;
  return slots - 1;
}
struct MdevTypeLabels {  // one dictionary: labels indexed by canonical id, and the ids that are keys
  const uint32_t* keys;  // the canonical ids to translate (from) / to look up (into), ascending
  uint32_t n_keys;
  const uint8_t* bytes;  // label of id c at bytes + off[c], len[c] bytes
  const uint32_t* off;
  const uint32_t* len;
  const uint64_t* hash;
};
__device__ __forceinline__ bool delta_label_eq(const MdevTypeLabels& a, uint32_t ca, const MdevTypeLabels& b, uint32_t cb) {
  if (__ldg(&a.hash[ca]) != __ldg(&b.hash[cb])) return false;
  const uint32_t len = __ldg(&a.len[ca]);
  if (__ldg(&b.len[cb]) != len) return false;
  const uint8_t *x = a.bytes + __ldg(&a.off[ca]), *y = b.bytes + __ldg(&b.off[cb]);
  for (uint32_t t = 0; t < len; t++)
    if (__ldg(&x[t]) != __ldg(&y[t])) return false;
  return true;
}
__global__ void __launch_bounds__(XMAP_THREADS) k_mdev_delta_types(MdevTypeLabels now, MdevTypeLabels prev,
                                                                    uint64_t* table, uint32_t mask, uint32_t tag,
                                                                    uint32_t* xlate) {
  pdl_enter();
  const uint64_t mine = (uint64_t)tag << 32;
  unsigned long long* cas = reinterpret_cast<unsigned long long*>(table);
  for (uint32_t k = threadIdx.x; k < now.n_keys; k += XMAP_THREADS) {
    bool placed = false;
    for (uint32_t s = (uint32_t)__ldg(&now.hash[__ldg(&now.keys[k])]) & mask; !placed; s = (s + 1) & mask) {
      uint64_t w = ld_relaxed_u64(table + s);
      while (!placed && (uint32_t)(w >> 32) != tag) {  // another call's slot is free
        const uint64_t seen = atomicCAS(cas + s, (unsigned long long)w, (unsigned long long)(mine | k));
        placed = seen == w;
        w = seen;
      }
    }
  }
  __syncthreads();
  for (uint32_t j = threadIdx.x; j < prev.n_keys; j += XMAP_THREADS) {
    const uint32_t c = __ldg(&prev.keys[j]);
    uint32_t to = DELTA_NONE;
    for (uint32_t s = (uint32_t)__ldg(&prev.hash[c]) & mask;; s = (s + 1) & mask) {
      const uint64_t w = ld_relaxed_u64(table + s);
      if ((uint32_t)(w >> 32) != tag) break;  // free: no new key has this label
      const uint32_t cn = __ldg(&now.keys[(uint32_t)w]);
      if (delta_label_eq(prev, c, now, cn)) {
        to = cn;
        break;
      }
    }
    xlate[c] = to;
  }
}

// ---- the re-key of kvg_scan_pci_raw_delta / kvg_scan_mdev_raw_delta: two snapshots in any mode pair onto the name
// space they share ---------------------------------------------------------------------------------------------------
//   k_raw_rekey  one thread per survivor of either side: the name's merge-path rank (its index plus the other side's
//                names below it, by binary search), the indices of its keys among its side's keys, the strict ascent
//                of the new names; and one thread per new key of a string-keyed map: into that map's table
//   k_raw_xlate  one thread per previous key of a string-keyed map: the new key index with the same string, or
//                DELTA_NONE
// PCI: both maps are string-keyed (device ids, groups).  mdev: the survivor keeps its canonical type id (vGpuMap keys
// are translated by label, k_mdev_delta_types) and only the parents (gpuVgpuMap) go through the tables.
// A string is either bytes the walk read or, in a numeric column, the canonical formatting of the number, produced
// one character at a time so that nothing is materialised.
enum : uint32_t { RSTR_BYTES, RSTR_DEC, RSTR_HEX4, RSTR_BDF, RSTR_UUID };
struct RawStr {
  const uint8_t* p;
  uint32_t len, v, kind;
};
__device__ __forceinline__ uint8_t rstr_hex(uint32_t d) { return (uint8_t)(d < 10 ? '0' + d : 'a' + d - 10); }
__device__ __forceinline__ uint8_t rstr_at(const RawStr& s, uint32_t i) {
  if (s.kind == RSTR_BYTES) return __ldg(&s.p[i]);
  if (s.kind == RSTR_HEX4) return rstr_hex((s.v >> (4 * (3 - i))) & 15u);
  if (s.kind == RSTR_DEC) {
    uint32_t v = s.v;
    for (uint32_t k = i + 1; k < s.len; k++) v /= 10;
    return (uint8_t)('0' + v % 10);
  }
  if (s.kind == RSTR_UUID) {  // 8-4-4-4-12 lower-case hex of the 16 bytes at p
    if (i == 8 || i == 13 || i == 18 || i == 23) return '-';
    const uint32_t h = i - (i > 8) - (i > 13) - (i > 18) - (i > 23);
    const uint32_t b = __ldg(&s.p[h >> 1]);
    return rstr_hex((h & 1) ? b & 15u : b >> 4);
  }
  // "dddd:bb:dd.f" of domain << 16 | bus << 8 | dev << 3 | fn (kvg_snap.cuh raw_bdf)
  if (i == 4 || i == 7) return ':';
  if (i == 10) return '.';
  const uint32_t f = i < 4 ? s.v >> 16 : i < 7 ? (s.v >> 8) & 0xffu : i < 10 ? (s.v >> 3) & 31u : s.v & 7u;
  const uint32_t w = i < 4 ? 3 - i : i < 7 ? 6 - i : i < 10 ? 9 - i : 0;
  return rstr_hex((f >> (4 * w)) & 15u);
}
__device__ __forceinline__ RawStr rstr_dec(uint32_t v) {
  uint32_t len = 1;
  for (uint32_t x = v; x >= 10; x /= 10) len++;
  return {nullptr, len, v, RSTR_DEC};
}
// byte-wise order: <0, 0, >0
__device__ __forceinline__ int rstr_cmp(const RawStr& a, const RawStr& b) {
  const uint32_t m = min(a.len, b.len);
  for (uint32_t i = 0; i < m; i++) {
    const uint32_t x = rstr_at(a, i), y = rstr_at(b, i);
    if (x != y) return x < y ? -1 : 1;
  }
  return a.len < b.len ? -1 : a.len > b.len ? 1 : 0;
}
__device__ __forceinline__ uint64_t rstr_fnv(const RawStr& s) {
  uint64_t h = 1469598103934665603ull;
  for (uint32_t i = 0; i < s.len; i++) h = (h ^ rstr_at(s, i)) * 1099511628211ull;
  return h;
}

// One snapshot's survivors and the strings behind them.  Map m: PCI 0 = deviceMap, 1 = iommuMap; mdev 0 = vGpuMap
// (no keys here), 1 = gpuVgpuMap.
enum : uint32_t { RAW_NUM_ADDR = 1u, RAW_NUM_DEVICE = 2u, RAW_NUM_GROUP = 4u };  // mdev: UUID names, -, parents
struct RawDeltaSide {
  const uint4* surv;        // kvg_pci_surv (PCI) or kvg_mdev_surv (mdev, two uint4), Walk order
  uint32_t n;
  const uint32_t* off;      // the walk's offsets and bytes: the names and key strings in index mode (NULL when numeric)
  const uint8_t* bytes;
  const uint2* tab[2];      // handle -> span in bytes of the map's key strings in index mode
  const uint32_t* keys[2];  // the distinct keys of the side's result
  uint32_t n_keys[2];
  uint32_t numeric;         // RAW_NUM_*: the columns in numeric mode

  __device__ __forceinline__ RawStr span_str(uint2 s) const { return {bytes + s.x, s.y - s.x, 0u, RSTR_BYTES}; }
  __device__ __forceinline__ RawStr walk_name(uint32_t w, uint32_t fields) const {
    const uint32_t* o = off + (size_t)w * fields;
    return span_str(make_uint2(__ldg(&o[0]), __ldg(&o[1])));
  }
  template <bool MDEV>
  __device__ __forceinline__ RawStr name(uint32_t i) const {
    if constexpr (MDEV) {  // the UUID bytes of a canonical snapshot, else the name at the Walk index `src`
      if (numeric & RAW_NUM_ADDR) return {reinterpret_cast<const uint8_t*>(surv + 2 * (size_t)i), 36u, 0u, RSTR_UUID};
      return walk_name(__ldg(&surv[2 * (size_t)i + 1].z), KVG_MRAW_FIELDS);
    } else {
      const uint32_t addr = __ldg(&surv[i].x);
      if (numeric & RAW_NUM_ADDR) return {nullptr, 12u, addr, RSTR_BDF};
      return walk_name(addr, KVG_RAW_FIELDS);
    }
  }
  template <bool MDEV>
  __device__ __forceinline__ RawStr key(uint32_t m, uint32_t h) const {
    if (m == 0) return (numeric & RAW_NUM_DEVICE) ? RawStr{nullptr, 4u, h, RSTR_HEX4} : span_str(__ldg(&tab[0][h]));
    if (numeric & RAW_NUM_GROUP) return MDEV ? RawStr{nullptr, 12u, h, RSTR_BDF} : rstr_dec(h);
    return span_str(__ldg(&tab[1][h]));
  }
};

constexpr uint32_t REKEY_THREADS = 256;
struct RawRekeyArgs {
  RawDeltaSide side[2];  // previous, new
  uint4* out[2];         // PciRawDeltaRec / MdevRawDeltaRec survivors of each side
  uint64_t* table[2];    // per map: the new keys, slot = tag << 32 | key index (another call's tag: free)
  uint32_t mask[2];
  uint32_t tag;
  uint32_t* xlate;       // the merge's table: map 0 from 0 (PCI), map 1 from RAW_XLATE_GROUP
  ScanCtrl* ctrl;        // reserved2[DELTA_W_ERROR]: the new names do not ascend strictly
};

template <bool MDEV>
__global__ void __launch_bounds__(REKEY_THREADS) k_raw_rekey(RawRekeyArgs a) {
  pdl_enter();
  const uint32_t t = blockIdx.x * REKEY_THREADS + threadIdx.x;
  const uint32_t n0 = a.side[0].n;
  if (t < n0 + a.side[1].n) {
    const uint32_t s = t < n0 ? 0 : 1, i = s ? t - n0 : t;
    const RawDeltaSide& me = a.side[s];
    const RawDeltaSide& other = a.side[s ^ 1];
    const RawStr nm = me.name<MDEV>(i);
    uint32_t lo = 0, hi = other.n;  // the other side's names below this one
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (rstr_cmp(other.name<MDEV>(mid), nm) < 0)
        lo = mid + 1;
      else
        hi = mid;
    }
    if (s == 1 && i > 0 && rstr_cmp(me.name<MDEV>(i - 1), nm) >= 0) a.ctrl->reserved2[DELTA_W_ERROR] = 1u;
    if constexpr (MDEV) {  // {uuid bytes}, {parent index, type_key | numa << 16, rank, 0}
      const uint4 u = __ldg(&me.surv[2 * (size_t)i]), r = __ldg(&me.surv[2 * (size_t)i + 1]);
      a.out[s][2 * (size_t)i] = u;
      a.out[s][2 * (size_t)i + 1] = make_uint4(delta_find(me.keys[1], me.n_keys[1], r.x), r.y, i + lo, 0u);
    } else {
      const uint4 r = __ldg(&me.surv[i]);
      const uint32_t gi = delta_find(me.keys[1], me.n_keys[1], r.y);
      const uint32_t di = delta_find(me.keys[0], me.n_keys[0], r.z & 0xffffu);
      a.out[s][i] = make_uint4(i + lo, gi, di | (r.z & 0xffff0000u), r.x);
    }
  }
  const RawDeltaSide& now = a.side[1];
  const uint64_t mine = (uint64_t)a.tag << 32;
  for (uint32_t m = MDEV ? 1 : 0; m < 2; m++) {
    if (t >= now.n_keys[m]) continue;
    unsigned long long* cas = reinterpret_cast<unsigned long long*>(a.table[m]);
    bool placed = false;
    for (uint32_t s = (uint32_t)rstr_fnv(now.key<MDEV>(m, __ldg(&now.keys[m][t]))) & a.mask[m]; !placed;
         s = (s + 1) & a.mask[m]) {
      uint64_t w = ld_relaxed_u64(a.table[m] + s);
      while (!placed && (uint32_t)(w >> 32) != a.tag) {
        const uint64_t seen = atomicCAS(cas + s, (unsigned long long)w, (unsigned long long)(mine | t));
        placed = seen == w;
        w = seen;
      }
    }
  }
}

template <bool MDEV>
__global__ void __launch_bounds__(REKEY_THREADS) k_raw_xlate(RawRekeyArgs a) {
  pdl_enter();
  const uint32_t t = blockIdx.x * REKEY_THREADS + threadIdx.x;
  const RawDeltaSide &prev = a.side[0], &now = a.side[1];
  uint32_t m = 1, k = t;  // mdev: parents only
  if constexpr (!MDEV) {
    m = t < prev.n_keys[0] ? 0 : 1;
    k = m ? t - prev.n_keys[0] : t;
  }
  if (k >= prev.n_keys[m]) return;
  const RawStr want = prev.key<MDEV>(m, __ldg(&prev.keys[m][k]));
  uint32_t to = DELTA_NONE;
  for (uint32_t s = (uint32_t)rstr_fnv(want) & a.mask[m];; s = (s + 1) & a.mask[m]) {
    const uint64_t w = ld_relaxed_u64(a.table[m] + s);
    if ((uint32_t)(w >> 32) != a.tag) break;  // free: no new key has this string
    const uint32_t j = (uint32_t)w;
    if (rstr_cmp(now.key<MDEV>(m, __ldg(&now.keys[m][j])), want) == 0) {
      to = j;
      break;
    }
  }
  a.xlate[(m ? RAW_XLATE_GROUP : 0u) + k] = to;
}

// The launch arguments, built on the host by kvg_api_delta.inc and by the CPU emulator alike.
// Both snapshots fully numeric: the plain merge on the decoded survivors, no re-key
inline bool raw_rekey_needed(uint32_t prev_numeric, uint32_t now_numeric, uint32_t all) {
  return prev_numeric != all || now_numeric != all;
}
// the two sides' survivors re-keyed into `rekeyed` (the previous side first; mdev: two uint4 per survivor), the key
// tables of the string-keyed maps at `table` (raw_rekey_table_words of it), the translation into `xlate` (at least
// RAW_XLATE_GROUP + the previous side's map-1 keys); returns the grids of k_raw_rekey and k_raw_xlate
template <bool MDEV>
inline RawRekeyArgs raw_rekey_args(const RawDeltaSide& prev, const RawDeltaSide& now, uint4* rekeyed, uint64_t* table,
                                   uint32_t* xlate, uint32_t tag, ScanCtrl* ctrl, uint32_t* grid_rekey,
                                   uint32_t* grid_xlate) {
  RawRekeyArgs a = {};
  a.side[0] = prev;
  a.side[1] = now;
  a.mask[0] = MDEV ? 0u : delta_xmap_mask(now.n_keys[0]);
  a.mask[1] = delta_xmap_mask(now.n_keys[1]);
  a.out[0] = rekeyed;
  a.out[1] = rekeyed + (MDEV ? 2 : 1) * (size_t)prev.n;
  a.table[0] = table;
  a.table[1] = table + (MDEV ? 0 : a.mask[0] + 1);
  a.tag = tag;
  a.xlate = xlate;
  a.ctrl = ctrl;
  uint32_t n = prev.n + now.n, nk = now.n_keys[1] + 0;
  if (!MDEV && now.n_keys[0] > nk) nk = now.n_keys[0];
  if (nk > n) n = nk;
  *grid_rekey = n ? (n + REKEY_THREADS - 1) / REKEY_THREADS : 1;
  n = (MDEV ? 0 : prev.n_keys[0]) + prev.n_keys[1];
  *grid_xlate = n ? (n + REKEY_THREADS - 1) / REKEY_THREADS : 1;
  return a;
}
// the table words raw_rekey_args uses for a new side with n_keys keys per map
inline size_t raw_rekey_table_words(bool mdev, const uint32_t (&n_keys)[2]) {
  return (mdev ? 0 : (size_t)delta_xmap_mask(n_keys[0]) + 1) + delta_xmap_mask(n_keys[1]) + 1;
}

}  // namespace kvg
