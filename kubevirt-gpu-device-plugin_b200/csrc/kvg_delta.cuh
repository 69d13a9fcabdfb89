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

}  // namespace kvg
