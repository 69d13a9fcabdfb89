// kvg_delta.cuh — K7: the keyed diff of two PCI scans (kvg_scan_pci_delta).
//
//   k_delta_merge   merge path over the previous scan's survivors and the new ones (16-byte records, ascending
//                   address in word 0): one change entry per address whose survivor differs, compacted in address
//                   order by the look-back tile body of kvg_scan.cuh; every entry tags the deviceMap / iommuMap keys
//                   whose member sequence it changes.  Also checks that the new list ascends strictly.
//   k_delta_lists   the four key lists (dirty / gone of both maps) from those tags: one look-back compaction per
//                   list (blockIdx.y) through the same tile body
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

__device__ __forceinline__ uint32_t delta_addr(const uint4* list, uint32_t i) {
  return __ldg(reinterpret_cast<const uint32_t*>(list + i));
}
// previous-list elements among the first d merged positions; equal addresses take the previous element first
__device__ __forceinline__ uint32_t delta_split(const uint4* a, uint32_t na, const uint4* b, uint32_t nb, uint32_t d) {
  uint32_t lo = d > nb ? d - nb : 0, hi = min(d, na);
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (delta_addr(a, mid) <= delta_addr(b, d - 1 - mid))
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}
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

  // A change entry whose member left key `prev_key` and joined key `now_key` (either side may be absent):
  // the key it joined is dirty; the key it left is dirty if it still exists, else gone.
  __device__ __forceinline__ void mark(bool has_now, uint32_t now_key, bool has_prev, uint32_t prev_key,
                                       uint32_t tag) const {
    if (has_now) {
      const uint32_t k = delta_find(keys_now, n_now, now_key);
      if (k != DELTA_NONE) flag_now[k] = tag;
    }
    if (has_prev && !(has_now && prev_key == now_key)) {
      uint32_t k = delta_find(keys_now, n_now, prev_key);
      if (k != DELTA_NONE)
        flag_now[k] = tag;
      else if ((k = delta_find(keys_prev, n_prev, prev_key)) != DELTA_NONE)
        flag_prev[k] = tag;
    }
  }
};

// what differs between two survivors of the same address (kvg_pci_surv: {addr, group, device | numa << 16, name})
__device__ __forceinline__ uint32_t delta_diff(const uint4& p, const uint4& q) {
  return (p.y != q.y ? (uint32_t)KVG_CH_GROUP : 0u) | ((p.z & 0xffffu) != (q.z & 0xffffu) ? (uint32_t)KVG_CH_DEVICE : 0u) |
         ((p.z >> 16) != (q.z >> 16) ? (uint32_t)KVG_CH_NUMA : 0u);
}

// The merged sequence as a classify operator: record i of the tile front-end is merged position i.  The CTA has
// staged its previous-list slice [i0, i0 + na) and new-list slice [j0, j0 + nb) in s_rec and the merge in s_code
// (bit 31: new list, low bits: index in that list).  An equal pair is adjacent in the merge, previous first:
//   previous element a at position i: matched iff the new element b = i - a (the next one at its merge position)
//                                     has its address -> it reports the pair, if the pair differs
//   new element b at position i:      matched iff the previous element i - b - 1 has its address -> silent
// Either neighbour may lie outside the CTA's slice and is then read from global memory.
struct DeltaMergeOp {
  struct Item {
    uint32_t code, what;
  };
  const uint4* prev;
  uint32_t n_prev;
  const uint4* now;
  uint32_t n_now;
  uint32_t n;    // merged positions: n_prev + n_now
  uint4* out;    // kvg_pci_change, 2 x 16 bytes per entry
  ScanCtrl* ctrl;
  DeltaKeys dev, grp;
  uint32_t tag;
  const uint4* s_rec;
  const uint32_t* s_code;
  uint32_t d0, i0, na, j0, nb;

  __device__ __forceinline__ uint4 rec_prev(uint32_t a) const { return a - i0 < na ? s_rec[a - i0] : __ldg(prev + a); }
  __device__ __forceinline__ uint4 rec_now(uint32_t b) const { return b - j0 < nb ? s_rec[na + b - j0] : __ldg(now + b); }

  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    Item it = {0u, 0u};
    if (!ok || i - d0 >= na + nb) return it;
    const uint32_t code = s_code[i - d0], x = code & 0x7fffffffu;
    it.code = code;
    if (code >> 31) {
      const uint32_t a = i - x;  // previous-list elements before it
      if (a == 0 || rec_prev(a - 1).x != rec_now(x).x) it.what = KVG_CH_ADDED;
    } else {
      const uint32_t b = i - x;  // new-list elements before it
      const uint4 p = rec_prev(x);
      if (b >= n_now) {
        it.what = KVG_CH_REMOVED;
      } else {
        const uint4 q = rec_now(b);
        it.what = q.x != p.x ? (uint32_t)KVG_CH_REMOVED : delta_diff(p, q);
      }
    }
    return it;
  }
  __device__ __forceinline__ bool pred(const Item& it, uint32_t) const { return it.what != 0; }
  __device__ __forceinline__ uint32_t prepare(const Item&) const { return 0; }
  // the change entry (kvgpu.h kvg_pci_change) and the keys it dirties
  __device__ __forceinline__ void emit(uint32_t pos, const Item& it, uint32_t i, uint32_t) const {
    const uint32_t x = it.code & 0x7fffffffu;
    const uint32_t a = (it.code >> 31) ? DELTA_NONE : x;
    const uint32_t b = (it.code >> 31) ? x : ((it.what & KVG_CH_REMOVED) ? DELTA_NONE : i - x);
    const bool hp = a != DELTA_NONE, hn = b != DELTA_NONE;
    const uint4 p = hp ? rec_prev(a) : make_uint4(0, 0, 0, 0);
    const uint4 q = hn ? rec_now(b) : make_uint4(0, 0, 0, 0);
    st_stream(out + 2 * (size_t)pos, make_uint4(hp ? p.x : q.x, it.what, p.y, q.y));
    st_stream(out + 2 * (size_t)pos + 1,
              make_uint4((p.z & 0xffffu) | (q.z << 16), (p.z >> 16) | (q.z & 0xffff0000u), b, a));
    // a key is dirty iff the (addr, numa) sequence of its members changed
    if (it.what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_DEVICE | KVG_CH_NUMA))
      dev.mark(hn, q.z & 0xffffu, hp, p.z & 0xffffu, tag);
    if (it.what & (KVG_CH_ADDED | KVG_CH_REMOVED | KVG_CH_GROUP | KVG_CH_NUMA)) grp.mark(hn, q.y, hp, p.y, tag);
  }
  __device__ __forceinline__ void tile_epilogue() {}
  __device__ __forceinline__ void finish(uint32_t total) { ctrl->reserved2[DELTA_W_CHANGES] = total; }
};

// One CTA per DELTA_TILE merged positions.  O(n_prev + n_now): two diagonal searches per CTA, a shared-memory merge,
// one pass of the look-back compaction.  The tag doubles as the look-back epoch.
__global__ void __launch_bounds__(DELTA_THREADS) k_delta_merge(DeltaMergeOp op, uint64_t* tile_state) {
  pdl_enter();
  __shared__ uint4 s_rec[DELTA_TILE];
  __shared__ uint32_t s_code[DELTA_TILE];
  __shared__ uint32_t s_split[2];
  __shared__ uint32_t s_wtot[DELTA_THREADS / 32], s_woff[DELTA_THREADS / 32];
  __shared__ uint32_t s_base;
  DeltaMergeOp o = op;
  const uint32_t n_tiles = (o.n + DELTA_TILE - 1) / DELTA_TILE, tile = blockIdx.x;
  if (n_tiles == 0) {
    if (tile == 0 && threadIdx.x == 0) o.finish(0);
    return;
  }
  if (tile >= n_tiles) return;
  const uint32_t d0 = tile * DELTA_TILE, d1 = min(o.n, d0 + DELTA_TILE);
  if (threadIdx.x == 0 || threadIdx.x == 32) {
    const uint32_t hi = threadIdx.x != 0;
    s_split[hi] = delta_split(o.prev, o.n_prev, o.now, o.n_now, hi ? d1 : d0);
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
      s_rec[k] = ld_stream(o.prev + o.i0 + k);
    } else {
      const uint32_t b = o.j0 + (k - o.na);
      const uint4 r = ld_stream(o.now + b);
      s_rec[k] = r;
      if (b > 0 && delta_addr(o.now, b - 1) >= r.x) o.ctrl->reserved2[DELTA_W_ERROR] = 1u;  // strict ascent
    }
  }
  __syncthreads();
  {  // each thread merges DELTA_ROWS consecutive positions from its own diagonal
    const uint32_t na = o.na, nb = o.nb, cnt = na + nb;
    const uint32_t p0 = min(cnt, threadIdx.x * DELTA_ROWS), p1 = min(cnt, p0 + DELTA_ROWS);
    uint32_t lo = p0 > nb ? p0 - nb : 0, hi = min(p0, na);
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (s_rec[mid].x <= s_rec[na + p0 - 1 - mid].x)
        lo = mid + 1;
      else
        hi = mid;
    }
    uint32_t ia = lo, ib = p0 - lo;
    for (uint32_t p = p0; p < p1; p++) {
      const bool take_prev = ib >= nb || (ia < na && s_rec[ia].x <= s_rec[na + ib].x);
      s_code[p] = take_prev ? o.i0 + ia++ : (0x80000000u | (o.j0 + ib++));
    }
  }
  __syncthreads();
  o.s_rec = s_rec;
  o.s_code = s_code;
  lookback_tile<DeltaMergeOp, DELTA_THREADS, DELTA_ROWS>(o, tile, n_tiles, tile_state, o.tag, s_wtot, s_woff, s_base);
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
  DeltaListOp o[4];  // deviceMap dirty, deviceMap gone, iommuMap dirty, iommuMap gone
};
// grid (tiles of the longest list, 4); list y uses the look-back words tile_state[y * state_stride ..)
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

}  // namespace kvg
