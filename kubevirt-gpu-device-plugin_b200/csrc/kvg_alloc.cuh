// kvg_alloc.cuh — GetPreferredAllocation of the passthrough plugin (generic_device_plugin.go:470-608) on the device:
// k_preferred_alloc packs every container request of one call onto NUMA nodes in one launch.
//
// A request's entries are its n_must must-include IDs, then its n_avail available IDs, in kubelet order.  Each entry is
// an interned handle (equal iff the ID strings are equal) and a dense node index, or PREF_NONE for the reference's -1
// (no topology, an advertised node of -1, or not a device of the plugin).  With P the number of distinct must-include
// IDs, the rule per request is:
//   1. the must-include IDs, first occurrences in order; sel[node] counts them per node
//   2. P > size fails (n_out = -1), whatever else the request holds
//   3. P < size: the target is the first candidate node with sel + free >= size, where free counts the available
//      entries that are not must-include IDs, duplicates included.  Candidates are ordered by the smallest must
//      position on the node, else by the smallest available position, so one min-reduction of that key over the
//      qualifying nodes finds the target.  A target of PREF_NONE stops the search with no fill; any other target
//      gives its available first occurrences that are not must-include IDs, in order, up to size
//   4. still short: the available first occurrences not taken yet, in order, up to size
// The picks are entry positions within the request: the must picks, then the fill, then the fallback, each ascending.
//
// Scratch (pref_scratch_words): per request, first[E] (the smallest position of each handle, by atomicMin) and, per
// node slot, sel, free and key (E + 1 slots, PREF_NONE last).  Each CTA initialises the slices of its own requests,
// so no clearing launch precedes the kernel.
#pragma once
#include "kvg_common.cuh"

namespace kvg {

static constexpr int PREF_THREADS = 1024;
static constexpr uint32_t PREF_NONE = 0xffffffffu;  // = KVG_PREF_NODE_NONE
static constexpr uint32_t PREF_MAX_GRID = 65535;    // more requests than this: each CTA takes several in turn

// Words of scratch for n_ids entries in n_reqs requests: first[n_ids], then sel, free and key of n_ids + n_reqs slots.
__host__ __device__ inline size_t pref_scratch_words(size_t n_ids, size_t n_reqs) {
  return n_ids + 3 * (n_ids + n_reqs);
}

// Exclusive sum over the PREF_THREADS threads of the block; `total` receives the block sum.  s: 33 shared words.
// The third __syncthreads lets the next call reuse s.
__device__ __forceinline__ uint32_t pref_excl_sum(uint32_t v, uint32_t* s, uint32_t& total) {
  constexpr uint32_t NW = PREF_THREADS / 32;
  static_assert(NW == 32, "one warp scans the warp totals");
  const uint32_t incl = warp_incl_sum(v);
  if (lane_id() == 31) s[warp_id()] = incl;
  __syncthreads();
  if (warp_id() == 0) {
    const uint32_t w = s[lane_id()];
    const uint32_t wi = warp_incl_sum(w);
    s[lane_id()] = wi - w;
    if (lane_id() == 31) s[NW] = wi;
  }
  __syncthreads();
  const uint32_t r = s[warp_id()] + incl - v;
  total = s[NW];
  __syncthreads();
  return r;
}

// The first k positions i in [lo, hi) with pred(i), ascending, to out[0..]; returns how many were taken (<= k).
// Chunks of PREF_THREADS with a running carry; the loop ends with the first chunk that reaches k.  carry is the same in
// every thread, so every thread makes the same number of trips.
template <class Pred>
__device__ __forceinline__ uint32_t pref_take(uint32_t lo, uint32_t hi, uint32_t k, Pred pred, uint32_t* out,
                                              uint32_t* s) {
  uint32_t carry = 0;
  for (uint32_t c = lo; c < hi && carry < k; c += PREF_THREADS) {
    const uint32_t i = c + threadIdx.x;
    const bool p = i < hi && pred(i);
    uint32_t tot;
    const uint32_t r = carry + pref_excl_sum(p ? 1u : 0u, s, tot);
    if (p && r < k) out[r] = i;
    carry += tot;
  }
  return min(carry, k);
}

// reqs[r] = {n_must, n_avail, size (int32), pad}; req_off[r] = the request's first entry; ids[j] = {handle, node}.
// Per request r: res_host[2r] = n_out (int32, -1 when P > size), res_host[2r + 1] = P, and the picks at
// out_host[req_off[r] ..].  The last CTA to finish (done counts them; the host zeroes it) writes the sequence word.
__global__ void __launch_bounds__(PREF_THREADS) k_preferred_alloc(const uint4* __restrict__ reqs,
                                                                  const uint32_t* __restrict__ req_off,
                                                                  const uint2* __restrict__ ids, uint32_t n_reqs,
                                                                  uint32_t n_ids, uint32_t* scratch, uint32_t* done,
                                                                  uint32_t* res_host, uint32_t* out_host,
                                                                  uint32_t* seq_host, uint32_t seq) {
  pdl_enter();
  __shared__ uint32_t s[PREF_THREADS / 32 + 1];
  __shared__ uint32_t s_must, s_key;
  const size_t n_slots = (size_t)n_ids + n_reqs;
  for (uint32_t r = blockIdx.x; r < n_reqs; r += gridDim.x) {
    const uint4 q = reqs[r];
    const uint32_t n_must = q.x, E = q.x + q.y, off = req_off[r];
    const int32_t size = (int32_t)q.z;
    const uint2* id = ids + off;
    uint32_t* first = scratch + off;
    uint32_t* sel = scratch + n_ids + off + r;
    uint32_t* fre = sel + n_slots;
    uint32_t* key = fre + n_slots;
    for (uint32_t i = threadIdx.x; i < E; i += PREF_THREADS) first[i] = PREF_NONE;
    for (uint32_t i = threadIdx.x; i <= E; i += PREF_THREADS) {
      sel[i] = 0;
      fre[i] = 0;
      key[i] = PREF_NONE;
    }
    if (threadIdx.x == 0) {
      s_must = 0;
      s_key = PREF_NONE;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < E; i += PREF_THREADS) atomicMin(&first[id[i].x], i);
    __syncthreads();
    const auto slot_of = [&](uint32_t i) {
      const uint32_t nd = id[i].y;
      return nd == PREF_NONE ? E : nd;
    };
    // per node: sel = distinct must-include IDs, free = available entries of other IDs, key = the smallest position
    uint32_t mine = 0;
    for (uint32_t i = threadIdx.x; i < E; i += PREF_THREADS) {
      const uint32_t f = first[id[i].x], slot = slot_of(i);
      atomicMin(&key[slot], i);
      if (i < n_must) {
        if (f == i) {
          atomicAdd(&sel[slot], 1u);
          mine++;
        }
      } else if (f >= n_must) {
        atomicAdd(&fre[slot], 1u);
      }
    }
    mine = warp_sum(mine);
    if (lane_id() == 0 && mine) atomicAdd(&s_must, mine);
    __syncthreads();
    const uint32_t P = s_must;
    int32_t n_out = -1;
    if ((int64_t)P <= size) {
      uint32_t* out = out_host + off;
      // an entry at or past n_must that is its handle's first occurrence is an available ID that is not must-include
      const auto fresh = [&](uint32_t i) { return first[id[i].x] == i; };
      uint32_t n = pref_take(0, n_must, P, fresh, out, s);
      if ((int64_t)n < size) {
        const uint32_t want = (uint32_t)size;
        uint32_t kmin = PREF_NONE;
        for (uint32_t i = threadIdx.x; i <= E; i += PREF_THREADS)
          if (sel[i] + fre[i] >= want) kmin = min(kmin, key[i]);
        kmin = warp_min(kmin);
        if (lane_id() == 0 && kmin != PREF_NONE) atomicMin(&s_key, kmin);
        __syncthreads();
        const uint32_t target = s_key == PREF_NONE ? E : slot_of(s_key);  // E: no target, or the -1 node
        if (target != E)
          n += pref_take(n_must, E, want - n, [&](uint32_t i) { return slot_of(i) == target && fresh(i); }, out + n, s);
        if (n < want)  // the fill, if any, took every entry of the target
          n += pref_take(n_must, E, want - n,
                         [&](uint32_t i) { return fresh(i) && (target == E || slot_of(i) != target); }, out + n, s);
      }
      n_out = (int32_t)n;
    }
    if (threadIdx.x == 0) {
      ((volatile uint32_t*)res_host)[2 * (size_t)r] = (uint32_t)n_out;
      ((volatile uint32_t*)res_host)[2 * (size_t)r + 1] = P;
    }
    __syncthreads();  // s_must / s_key are read before the next request resets them
  }
  __threadfence_system();  // this thread's picks and results are on their way before the CTA counts itself done
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(done, 1u) == gridDim.x - 1) {
    __threadfence_system();
    *((volatile uint32_t*)seq_host) = seq;
  }
}

}  // namespace kvg
