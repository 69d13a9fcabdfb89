// kvg_scan.cuh — record classification and stable compaction.
//
//   k_classify_ragged<Op>  K3/K5 at bandwidth-bound sizes: every CTA classifies one tile and writes its
//                          survivors at a TILE-LOCAL base (no cross-tile dependency); k_tile_offsets scans
//                          the tile counts, k_pack_survivors makes the list dense
//   k_compact<Op,T,R>      one launch, decoupled look-back on the tile counts: K3 at latency-bound sizes, K6
//        PciClassifyOp       createIommuDeviceMap's filter (device_plugin.go:201-244) + name join
//        MdevClassifyOp      createVgpuIDMap's filter (:268-289)
//        HealthOp<Rule>      K6: state diff against the previous tick, one health rule per record kind:
//                            PciHealthRule (alive), MdevHealthRule (present / XID-marked vGPUs),
//                            GroupHealthRule (alive and the IOMMU group's VFIO node exists)
//   k_health_small<Rule>   K6 at poll-loop sizes: one CTA, TMA-staged, transitions into mapped host memory
//                          (Keyed<Rule>, either form: the prior state joined by UUID / address instead of by index)
//   k_mdev_labels / _canon K5: label rule (:341-342) + merge of equal labels
//   k_mdev_label_match     the same label rule against one name: the vGPU plugin's Allocate-time re-check
//   k_pci_allocate_check   the passthrough plugin's Allocate decisions: group link and vendor per group member, and
//                          the EGM all-GPUs match, for every container request of one call
//   k_gen_*                counter-based synthetic snapshots (twins of oracle/kvg_oracle.c kvo_gen_*)
#pragma once
#include "../../include/kvgpu.h"
#include "kvg_common.cuh"
#include "kvg_parse.cuh"
#include "kvg_order.cuh"

namespace kvg {

// device-resident control block of one scan (zeroed by one memset per step)
struct ScanCtrl {
  uint32_t n_own[2];      // sharded scans: records in the owned list of ordering 0 / 1
  uint32_t own_max[2];    // sharded scans: their largest keys (radix plan)
  uint32_t n_gathered;    // sharded scans, NCCL mode: length of the all-gathered survivor list
  uint32_t key_err;       // keyed health, look-back form: the keys do not ascend strictly
  uint32_t reserved[2];
  uint32_t n_surv;        // survivors of the classify kernel
  uint32_t max_group;     // max iommu group / parent among survivors (radix pass count)
  uint32_t max_devkey;    // max device / type key among survivors
  uint32_t n_dev_keys;    // distinct keys found by the heads kernels
  uint32_t n_groups;
  uint32_t n_alive;       // health
  uint32_t n_changed;
  uint32_t pad0;
  uint32_t reserved2[16];
};

// ------------------------------------------------------------------------------------------------
// The one-launch look-back compaction (lookback_tiles), in two shapes:
//   K3 at latency-bound sizes, k_compact<PciClassifyOp, 128, 8>: small CTAs (1024 records kept in registers), one
//   per tile, thousands of them, dispatched in blockIdx order by the hardware.  Many resident CTAs per SM hide the
//   count -> look-back -> write-out latency chain of each other; predecessors were dispatched earlier, so the
//   classic decoupled look-back usually finds an inclusive prefix close by.  (Measured alternative: every tile
//   publishes its count and sums ALL earlier counts itself, a thread per earlier tile — no chain, but several
//   dependent L2 round trips per thread for the last tiles; it was slower at 1 M records.  The chained scan stays.)
//   K6, k_compact<HealthOp<Rule>, KVG_BLOCK, C_ROWS>: a persistent, co-resident grid of 2048-record tiles (compact_grid).
//   A look-back predecessor is owned by a resident CTA that reaches it no later than this CTA reaches its own tile
//   (no ticket needed).  One CTA per tile measured about 5 % slower at 4 Mi records (39.5 against 37.7 us, H100 SXM
//   with a 400 W power limit).
// ------------------------------------------------------------------------------------------------
// An operator that keeps a per-CTA table in shared memory fills it in an overload of compact_enter (HealthOp<Rule>
// with a set).
template <class Op>
__device__ __forceinline__ void compact_enter(Op&) {}
// The min-blocks launch bound of k_compact<Op>; 0 emits none.  With 16 KiB of static shared memory
// (HealthOp<GroupHealthRule>) ptxas otherwise caps the kernel at 32 registers and spills; a bound of 1 block lifts the
// cap.  Every other operator keeps the plain bound, so its code is unchanged.
template <class Op>
constexpr int COMPACT_MIN_BLOCKS = 0;
template <class Op, int THREADS, int ROWS>
__global__ void __launch_bounds__(THREADS, COMPACT_MIN_BLOCKS<Op>) k_compact(Op op, uint64_t* tile_state, uint32_t epoch) {
  pdl_enter();
  compact_enter(op);
  lookback_tiles<Op, THREADS, ROWS>(op, tile_state, epoch);
}

// ---- K3: PCI classify ---------------------------------------------------------------------------
// record = {addr, vendor | device<<16, iommu_group, driver | flags<<8 | numa<<16}
// device_plugin.go:203-238: any of the vendor/driver/iommu/device read errors drops the entry,
// vendor must be "10de" (:209), driver must be in supportedVfioDrivers (:217, :75-78)
__device__ __forceinline__ bool pci_record_alive(const uint4& r) {
  // low 12 bits of r.w = driver | (drop flags << 8): alive iff they equal 1 or 2 exactly
  static_assert(KVG_DRV_VFIO_PCI == 1 && KVG_DRV_NVGRACE == 2, "driver codes");
  static_assert((KVG_PF_VENDOR_ERR | KVG_PF_DRIVER_ERR | KVG_PF_IOMMU_ERR | KVG_PF_DEVICE_ERR) == 0xf, "flags");
  return (r.y & 0xffffu) == 0x10deu && ((r.w & 0x0fffu) - 1u) < 2u;
}
// The passthrough plugin's Allocate-time re-check of one group member (generic_device_plugin.go:388-397): its
// iommu_group link reads back as the group the maps hold for it (`want`, the same interned handle), and its vendor
// reads back as "10de".  Nothing else of the record counts: not the driver, the device id, the NUMA node or any other
// read error, so the rule stays the reference's whatever pci_record_alive comes to require.
__device__ __forceinline__ bool pci_group_check_pass(const uint4& r, uint32_t want) {
  const uint32_t flags = (r.w >> 8) & 0xffu;
  return !(flags & KVG_PF_IOMMU_ERR) && r.z == want && !(flags & KVG_PF_VENDOR_ERR) && (r.y & 0xffffu) == 0x10deu;
}
// What the PCI and mdev classify operators share: a survivor goes out as Self::UNITS 16-byte streaming stores of
// Self::make, and the largest Self::keys of the survivors a thread wrote bound the radix passes of the two
// orderings: keys().x -> ScanCtrl::max_devkey (ordering 0), keys().y -> max_group (ordering 1).
template <class Self>
struct SurvivorOp {
  uint4* out;
  ScanCtrl* ctrl;
  uint32_t local_max_x = 0, local_max_y = 0;  // per-thread running maxima of keys() (registers)

  template <class Item>
  __device__ __forceinline__ void emit(uint32_t pos, const Item& r, uint32_t i, uint32_t aux) {
    constexpr int U = Self::UNITS;
    const Self& self = static_cast<const Self&>(*this);
    uint4 s[U];
    self.make(r, i, aux, s);
#pragma unroll
    for (int u = 0; u < U; u++) st_stream(out + (size_t)pos * U + u, s[u]);
    const uint2 k = self.keys(r, aux);
    local_max_x = max(local_max_x, k.x);
    local_max_y = max(local_max_y, k.y);
  }
  __device__ __forceinline__ void tile_epilogue() {
    uint32_t g = warp_max(local_max_y), d = warp_max(local_max_x);
    if (lane_id() == 0) {
      if (g) atomicMax(&ctrl->max_group, g);
      if (d) atomicMax(&ctrl->max_devkey, d);
    }
    local_max_x = 0;
    local_max_y = 0;
  }
  __device__ __forceinline__ void finish(uint32_t total) { ctrl->n_surv = total; }
  // the thread's maxima as k_tile_offsets reads a tile_max slot: {group, dev}
  __device__ __forceinline__ uint2 take_maxima() {
    uint2 m = make_uint2(local_max_y, local_max_x);
    local_max_x = local_max_y = 0;
    return m;
  }
};

struct PciClassifyOp : SurvivorOp<PciClassifyOp> {
  using Item = uint4;
  static constexpr int UNITS = 1;  // 16-byte units per survivor
  const uint4* recs;
  uint32_t n;
  const uint32_t* nv_index;  // device id -> name pool slot (K1's k_pciids_names)

  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    return ok ? ld_stream(recs + i) : make_uint4(0, 0, 0, 0xff00u);
  }
  __device__ __forceinline__ bool pred(const Item& r, uint32_t) const { return pci_record_alive(r); }
  // the name join: one load per survivor from the flattened table of vendor 10de
  // (nv_index == NULL: the parse is still running on its own stream; the final ordering kernel joins the names)
  __device__ __forceinline__ uint32_t prepare(const Item& r) const { return nv_index ? __ldg(&nv_index[r.y >> 16]) : P_NONE; }
  // the survivor record (kvgpu.h kvg_pci_surv)
  __device__ __forceinline__ void make(const Item& r, uint32_t, uint32_t name_slot, uint4* s) const {
    uint32_t device = r.y >> 16;
    uint32_t flags = (r.w >> 8) & 0xffu;
    int32_t numa = (int32_t)r.w >> 16;  // sign-extended int16
    if ((flags & KVG_PF_NUMA_ERR) || numa < 0) numa = 0;  // :227-230, :316-318
    s[0].x = r.x;
    s[0].y = r.z;
    s[0].z = device | ((uint32_t)numa << 16);
    s[0].w = name_slot;
  }
  // keys of the two group-by maps: {device id (deviceMap), iommu group (iommuMap)}
  __device__ __forceinline__ uint2 keys(const Item& r, uint32_t) const { return make_uint2(r.y >> 16, r.z); }
};
// the deferred name join of a dense PCI survivor list no ordering walks (the rank's own shard of a sharded scan):
// runs on the side stream behind the parse, beside the exchange and the orderings
__global__ void __launch_bounds__(KVG_BLOCK) k_join_names(uint4* __restrict__ recs, const uint32_t* __restrict__ n_ptr,
                                                          const uint32_t* __restrict__ nv_index) {
  pdl_enter();
  const uint32_t n = *n_ptr;
  for (uint32_t i = blockIdx.x * KVG_BLOCK + threadIdx.x; i < n; i += gridDim.x * KVG_BLOCK) {
    uint32_t* w = reinterpret_cast<uint32_t*>(recs + i);
    w[3] = __ldg(&nv_index[w[2] & 0xffffu]);
  }
}

// ---- K5: mdev classify --------------------------------------------------------------------------
struct MdevItem {
  uint4 lo, hi;
};
// createVgpuIDMap's keep rule (:270-279): the type and the parent were read, and the type is in the dictionary.
// hi = {parent, type_idx | flags<<16 | pad<<24, parent_numa | pad.., pad}
__device__ __forceinline__ bool mdev_record_alive(const uint4& hi, uint32_t n_types) {
  const uint32_t flags = (hi.y >> 16) & 0xffu;
  return (flags & (KVG_MF_TYPE_ERR | KVG_MF_PARENT_ERR)) == 0 && (hi.y & 0xffffu) < n_types;
}
struct MdevClassifyOp : SurvivorOp<MdevClassifyOp> {
  using Item = MdevItem;
  static constexpr int UNITS = 2;  // 16-byte units per survivor
  const uint4* recs;  // 2 x uint4 per record
  uint32_t n;
  const uint16_t* type_canon;  // [n_types] canonical id per raw dictionary entry
  uint32_t n_types;

  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    Item it;
    if (ok) {
      it.lo = ld_stream(recs + 2 * (size_t)i);
      it.hi = ld_stream(recs + 2 * (size_t)i + 1);
    } else {
      it.lo = make_uint4(0, 0, 0, 0);
      it.hi = make_uint4(0, 0xffu << 16, 0, 0);
    }
    return it;
  }
  __device__ __forceinline__ bool pred(const Item& r, uint32_t) const { return mdev_record_alive(r.hi, n_types); }
  __device__ __forceinline__ uint32_t prepare(const Item& r) const { return type_canon[r.hi.y & 0xffffu]; }
  // the survivor record (kvgpu.h kvg_mdev_surv)
  __device__ __forceinline__ void make(const Item& r, uint32_t i, uint32_t canon, uint4* s) const {
    uint32_t flags = (r.hi.y >> 16) & 0xffu;
    int32_t numa = (int32_t)(int16_t)(r.hi.z & 0xffffu);
    if ((flags & KVG_MF_NUMA_ERR) || numa < 0) numa = 0;  // :281-284, :316-318
    s[0] = r.lo;
    s[1].x = r.hi.x;
    s[1].y = canon | ((uint32_t)numa << 16);
    s[1].z = i;
    s[1].w = 0;
  }
  // keys of the two group-by maps: {canonical type (vGpuMap), parent GPU (gpuVgpuMap)}
  __device__ __forceinline__ uint2 keys(const Item& r, uint32_t canon) const { return make_uint2(canon, r.hi.x); }
};

// ---- K6: health re-scan -------------------------------------------------------------------------
// Every health source is one rule: what its record is and how the state byte of a record moves from tick to tick.
// Bit 0 of a state byte is the health the transition list reports; the rest is the rule's own.
//   UNITS, UNIT        16-byte units per record, and the one unit next() reads
//   STATE_BITS         bits of the state byte the rule uses
//   STAGE_ROWS         rows of 1024 records per 192 KiB TMA round of k_health_small
//   SET_CAP            0, or the cap of a sorted, deduplicated set (set, n_set) every CTA copies into shared memory
//   next(r, s, set)    the state byte after this tick from unit UNIT of the record, the previous byte and the shared
//                      copy of the set
// k_health_small<Rule> runs it at poll-loop sizes, k_compact<HealthOp<Rule>, KVG_BLOCK, C_ROWS> above them.

// membership in the sorted set xs[0..n), n <= CAP (a power of two): lo = the last position whose value is <= v, found
// by log2(CAP) fixed steps (no data-dependent trip count; 10 for the XID set, 12 for the group set), then one compare;
// nothing is loaded when n == 0
template <uint32_t CAP>
__device__ __forceinline__ bool sorted_has(const uint32_t* xs, uint32_t n, uint32_t v) {
  static_assert(CAP >= 2 && (CAP & (CAP - 1)) == 0, "a power of two");
  if (n == 0) return false;
  uint32_t lo = 0;
#pragma unroll
  for (uint32_t step = CAP / 2; step; step >>= 1)
    if (lo + step < n && xs[lo + step] <= v) lo += step;
  return xs[lo] == v;
}
// every thread of the CTA copies its share of a sorted set into shared memory (the caller synchronises before the
// first use)
__device__ __forceinline__ void load_sorted_set(uint32_t* dst, const uint32_t* src, uint32_t n) {
  for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
}

// PCI (kvg_health_rescan): state = alive (0 / 1)
struct PciHealthRule {
  static constexpr uint32_t UNITS = 1, UNIT = 0, STAGE_ROWS = 12, SET_CAP = 0, STATE_BITS = 1;
  __device__ __forceinline__ uint32_t next(const uint4& r, uint32_t, const uint32_t*) const {
    return pci_record_alive(r) ? 1u : 0u;
  }
};

// vGPUs (kvg_health_rescan_mdev): healthy = present and not marked by a critical XID on the parent GPU.
// Per record two bits, p (present: mdev_record_alive) and m (marked), m => p.  A tick with the sorted, deduplicated
// parent handles X:  p' = alive,  m' = p' && (parent in X || (p && m)),  healthy = p && !m.  The state byte keeps them
// as bit 0 = healthy (p && !m), bit 1 = marked (p && m).  The rule reads the second unit of the 32-byte record.
// `in_x()` is the membership test of the record's parent, asked only of a present, unmarked record: the handle in X
// here, the parent string among the XID bus ids in the raw rule (kvg_snap.cuh).
constexpr uint32_t HEALTH_MDEV_HEALTHY = 1u, HEALTH_MDEV_MARKED = 2u;
template <class InX>
__device__ __forceinline__ uint32_t health_mdev_next(const uint4& hi, uint32_t s, uint32_t n_types, InX&& in_x) {
  if (!mdev_record_alive(hi, n_types)) return 0;
  const bool marked = (s & HEALTH_MDEV_MARKED) || in_x();
  return marked ? HEALTH_MDEV_MARKED : HEALTH_MDEV_HEALTHY;
}
struct MdevHealthRule {
  static constexpr uint32_t UNITS = 2, UNIT = 1, STAGE_ROWS = 6, SET_CAP = KVG_HEALTH_MAX_XID, STATE_BITS = 2;
  const uint32_t* set;  // X
  uint32_t n_set, n_types;
  __device__ __forceinline__ uint32_t next(const uint4& r, uint32_t s, const uint32_t* xs) const {
    return health_mdev_next(r, s, n_types, [&] { return sorted_has<KVG_HEALTH_MAX_XID>(xs, n_set, r.x); });
  }
};

// passthrough GPUs by IOMMU group (kvg_health_rescan_groups): healthy = alive and the group's VFIO node exists.  One
// bit per record, as for PCI.  A tick with the sorted, deduplicated handles G of the groups whose node exists now (the
// encoding of kvg_pci_rec.iommu_group, r.z of the record):  h' = pci_record_alive(r) && r.z in G.  `in_g()` is the
// membership test of the record's group, asked only of an alive record (the raw rule: the group string among the
// node names).
template <class InG>
__device__ __forceinline__ uint32_t health_group_next(const uint4& r, InG&& in_g) {
  return pci_record_alive(r) && in_g() ? 1u : 0u;
}
struct GroupHealthRule {
  static constexpr uint32_t UNITS = 1, UNIT = 0, STAGE_ROWS = 12, SET_CAP = KVG_HEALTH_MAX_GROUPS, STATE_BITS = 1;
  const uint32_t* set;  // G
  uint32_t n_set;
  __device__ __forceinline__ uint32_t next(const uint4& r, uint32_t, const uint32_t* gs) const {
    return health_group_next(r, [&] { return sorted_has<KVG_HEALTH_MAX_GROUPS>(gs, n_set, r.z); });
  }
};

// ---- where the prior state byte comes from -----------------------------------------------------
// A rule as it stands is index-keyed: the prior byte of record i is state[i], updated in place.  Keyed<Rule> is the
// same rule with the prior byte joined by the record's key (kvg_health_rescan_mdev_keyed / _groups_keyed): the
// previous call's list is (prev_key, prev_state)[0..n_prev), ascending by key; this call writes its own keys to
// `key` and its state bytes to the kernel's `state` (the other slot), every record, so keys absent now are forgotten.
// The kernels test KEYED_RULE<Rule>; an index rule compiles exactly the code it compiled before.
//   HealthKey<Rule>: the key type, the unit of the record holding it, and its order
template <class Rule>
struct HealthKey;
// the UUID (unit 0 of the 32-byte record) as a 128-bit big-endian number: the order of kvg_scan_mdev_delta
template <>
struct HealthKey<MdevHealthRule> {
  using Key = uint4;
  static constexpr uint32_t UNIT = 0;
  __device__ __forceinline__ static Key of(const uint4& u) { return u; }
  __device__ __forceinline__ static bool eq(const Key& a, const Key& b) {
    return ((a.x ^ b.x) | (a.y ^ b.y) | (a.z ^ b.z) | (a.w ^ b.w)) == 0;
  }
  __device__ __forceinline__ static bool lt(const Key& a, const Key& b) {
    const uint32_t a0 = __byte_perm(a.x, 0, 0x0123), b0 = __byte_perm(b.x, 0, 0x0123);
    if (a0 != b0) return a0 < b0;
    const uint32_t a1 = __byte_perm(a.y, 0, 0x0123), b1 = __byte_perm(b.y, 0, 0x0123);
    if (a1 != b1) return a1 < b1;
    const uint32_t a2 = __byte_perm(a.z, 0, 0x0123), b2 = __byte_perm(b.z, 0, 0x0123);
    if (a2 != b2) return a2 < b2;
    return __byte_perm(a.w, 0, 0x0123) < __byte_perm(b.w, 0, 0x0123);
  }
};
// the address handle (r.x of the 16-byte PCI record)
template <>
struct HealthKey<GroupHealthRule> {
  using Key = uint32_t;
  static constexpr uint32_t UNIT = 0;
  __device__ __forceinline__ static Key of(const uint4& u) { return u.x; }
  __device__ __forceinline__ static bool eq(Key a, Key b) { return a == b; }
  __device__ __forceinline__ static bool lt(Key a, Key b) { return a < b; }
};

template <class Rule>
struct Keyed : Rule {
  using K = HealthKey<Rule>;
  using Key = typename K::Key;
  const Key* prev_key;
  const uint8_t* prev_state;
  uint32_t n_prev;
  Key* key;       // this call's keys, [n]
  uint32_t* err;  // look-back form: set when a key does not exceed its predecessor's (ScanCtrl::key_err)
  // the prior byte of `k`, the key of record i: the same position first (the list did not change), else a binary
  // search of the previous keys (L2-resident at poll-loop sizes); 0 for a key the previous list lacks
  __device__ __forceinline__ uint32_t search(const Key& k) const {
    uint32_t lo = 0, hi = n_prev;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (K::lt(__ldg(&prev_key[mid]), k))
        lo = mid + 1;
      else
        hi = mid;
    }
    return lo < n_prev && K::eq(__ldg(&prev_key[lo]), k) ? __ldg(&prev_state[lo]) : 0u;
  }
  __device__ __forceinline__ uint32_t find(const Key& k, uint32_t i) const {
    return i < n_prev && K::eq(__ldg(&prev_key[i]), k) ? (uint32_t)__ldg(&prev_state[i]) : search(k);
  }
};
template <class Rule>
constexpr bool KEYED_RULE = false;
template <class Rule>
constexpr bool KEYED_RULE<Keyed<Rule>> = true;
// dynamic shared memory the small form adds for a keyed rule: the ascent error flag
template <class Rule>
constexpr uint32_t KEYED_SMEM = 0;
template <class Rule>
constexpr uint32_t KEYED_SMEM<Keyed<Rule>> = 16;

// the look-back form (above HEALTH_SMALL_MAX records, or with kernel timing on): k_compact<HealthOp<Rule>, 256, 8>.
// Item.x = new state | old state byte << W.  The state byte is written whenever it changes, a transition or not (a
// marked vGPU that vanishes loses its mark without a health change); a change of bit 0 is listed.  A one-bit state
// changes only with a transition, so emit writes it, where pred writes a wider one.  That, and reading state[i] as an
// argument of next() (a rule that ignores it loads it after its own work), keeps the group instantiation at 48
// registers: with the write in pred for every width, or the byte read first, ptxas takes 53 to 56.
// A keyed rule joins the prior byte in load (which also reads the key's unit when the rule reads another), checks
// that the key exceeds the previous record's, and writes the record's key and new byte to this call's slot there:
// every record, so pred and emit write no state.
template <class Rule>
struct HealthOp {
  using Item = uint4;
  static constexpr uint32_t W = Rule::STATE_BITS;
  static constexpr bool KEYED = KEYED_RULE<Rule>;
  const uint4* recs;  // Rule::UNITS x uint4 per record
  uint32_t n;
  Rule rule;
  const uint32_t* set;  // the rule's set in shared memory (compact_enter); unused without one
  uint8_t* state;       // one byte per record, updated in place (keyed: this call's slot)
  uint32_t* changed;
  ScanCtrl* ctrl;
  uint32_t local_alive;
  __device__ __forceinline__ uint32_t prepare(const Item&) const { return 0; }
  __device__ __forceinline__ Item load(uint32_t i, bool ok) const {
    if (!ok) return make_uint4(0, 0, 0, 0);
    uint4 r = ld_stream(recs + (size_t)i * Rule::UNITS + Rule::UNIT);
    if constexpr (KEYED) {
      using K = typename Rule::K;
      constexpr uint32_t KU = K::UNIT;
      const typename K::Key key = K::of(KU == Rule::UNIT ? r : ld_stream(recs + (size_t)i * Rule::UNITS + KU));
      if (i && !K::lt(K::of(__ldg(recs + (size_t)(i - 1) * Rule::UNITS + KU)), key)) *rule.err = 1u;
      const uint32_t was = rule.find(key, i), s = rule.next(r, was, set);
      rule.key[i] = key;
      state[i] = (uint8_t)s;
      r.x = s | (was << W);
    } else {
      r.x = rule.next(r, state[i], set) | ((uint32_t)state[i] << W);
    }
    return r;
  }
  __device__ __forceinline__ bool pred(const Item& r, uint32_t i) {
    const uint32_t now = r.x & ((1u << W) - 1), was = r.x >> W;
    local_alive += now & 1u;
    if constexpr (W == 1) return now != was;
    if constexpr (!KEYED)
      if (now != was) state[i] = (uint8_t)now;
    return ((now ^ was) & 1u) != 0;
  }
  __device__ __forceinline__ void emit(uint32_t pos, const Item& r, uint32_t i, uint32_t) {
    changed[pos] = (i << 1) | (r.x & 1u);
    if constexpr (W == 1 && !KEYED) state[i] = (uint8_t)(r.x & 1u);
  }
  __device__ __forceinline__ void tile_epilogue() {
    uint32_t a = warp_sum(local_alive);
    if (lane_id() == 0 && a) atomicAdd(&ctrl->n_alive, a);
    local_alive = 0;
  }
  __device__ __forceinline__ void finish(uint32_t total) { ctrl->n_changed = total; }
};
template <class Rule>
__device__ __forceinline__ void compact_enter(HealthOp<Rule>& op) {
  if constexpr (Rule::SET_CAP > 0) {
    __shared__ uint32_t s_set[Rule::SET_CAP];
    load_sorted_set(s_set, op.rule.set, op.rule.n_set);
    op.set = s_set;
    __syncthreads();
  }
}
template <>
constexpr int COMPACT_MIN_BLOCKS<HealthOp<GroupHealthRule>> = 1;
template <>
constexpr int COMPACT_MIN_BLOCKS<HealthOp<Keyed<GroupHealthRule>>> = 1;

// K6 at poll-loop sizes (BASELINE.json config 5: 10,000 devices at 1 kHz): ONE CTA, one launch, one host
// synchronisation.  The records are read where the host left them (mapped pinned memory: zero-copy over PCIe,
// every load of a thread in flight at once), the transitions are written — in record order — straight into
// the host-visible result block, and the two counters follow.  No staging copy, no look-back, no second
// device-to-host copy.  Dynamic shared memory: the stage, then the rule's set.
// the key type of a keyed rule (an index rule has none: a placeholder the compiler drops)
template <class Rule>
struct KeyOfT {
  using T = uint32_t;
};
template <class Rule>
struct KeyOfT<Keyed<Rule>> {
  using T = typename Keyed<Rule>::Key;
};
template <class Rule>
using KeyOf = typename KeyOfT<Rule>::T;
constexpr uint32_t HEALTH_SMALL_THREADS = 1024;
constexpr uint32_t HEALTH_SMALL_ROWS = 32;                                        // rows of 1024 records
constexpr uint32_t HEALTH_SMALL_MAX = HEALTH_SMALL_THREADS * HEALTH_SMALL_ROWS;  // 32,768 records
constexpr uint32_t HEALTH_STAGE_BYTES = 192u << 10;                               // one TMA round
template <class Rule>
constexpr uint32_t HEALTH_SMALL_SMEM = HEALTH_STAGE_BYTES + Rule::SET_CAP * 4 + KEYED_SMEM<Rule>;
// The end of both one-CTA health kernels (k_health_small, k_health_raw_small of kvg_snap.cuh), once every row has
// left its ballots in s_bal ("changed") and s_now ("healthy now") behind a block barrier, and each thread its count of
// healthy records in n_alive: 32 rows x 32 warps = one counter per thread, in record order, so ONE block scan places
// every transition; the list goes to changed_host, and every thread gets the totals.  Returns after the block barrier
// that follows the list's system fence, so thread 0 may publish the header and the flag.
constexpr uint32_t HEALTH_SMALL_NW = HEALTH_SMALL_THREADS / 32;
__device__ __forceinline__ void health_small_list(uint32_t rows, uint32_t n_alive,
                                                  uint32_t (*s_bal)[HEALTH_SMALL_NW],
                                                  uint32_t (*s_now)[HEALTH_SMALL_NW], uint32_t* s_scan,
                                                  uint32_t* s_alv, uint32_t* __restrict__ changed_host,
                                                  uint32_t& alive, uint32_t& total) {
  constexpr uint32_t NW = HEALTH_SMALL_NW;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t crow = tid >> 5, cw = tid & 31;
  const uint32_t mybal = crow < rows ? s_bal[crow][cw] : 0;
  const uint32_t mycnt = __popc(mybal);
  const uint32_t incl = warp_incl_sum(mycnt);
  const uint32_t wal = warp_sum(n_alive);
  if (lane == 31) s_scan[warp] = incl;
  if (lane == 0) s_alv[warp] = wal;
  __syncthreads();
  uint32_t base = 0;
  total = 0;
  alive = 0;
#pragma unroll
  for (uint32_t w = 0; w < NW; w++) {
    const uint32_t c = s_scan[w];
    if (w < warp) base += c;
    total += c;
    alive += s_alv[w];
  }
  // thread (crow, cw) writes the transitions of warp cw in row crow: lane order == record order
  uint32_t pos = base + incl - mycnt;
  const uint32_t nowb = crow < rows ? s_now[crow][cw] : 0;
  for (uint32_t m = mybal; m; m &= m - 1) {
    const uint32_t l = (uint32_t)__ffs((int)m) - 1;
    const uint32_t i = crow * HEALTH_SMALL_THREADS + cw * 32 + l;
    changed_host[pos++] = (i << 1) | ((nowb >> l) & 1u);
  }
  __threadfence_system();  // the list entries of every thread are on their way before the flag
  __syncthreads();
}
template <class Rule>
__global__ void __launch_bounds__(HEALTH_SMALL_THREADS) k_health_small(Rule rule, const uint4* __restrict__ recs,
                                                                       uint32_t n, uint8_t* __restrict__ state,
                                                                       uint32_t* __restrict__ changed_host,
                                                                       uint32_t* __restrict__ hdr_host, uint32_t seq) {
  pdl_enter();
  constexpr uint32_t NW = HEALTH_SMALL_THREADS / 32, U = Rule::UNITS, SR = Rule::STAGE_ROWS;
  static_assert(SR * HEALTH_SMALL_THREADS * 16 * U == HEALTH_STAGE_BYTES, "one round");
#ifndef KVG_HOST_EMU
  extern __shared__ __align__(128) uint8_t hs_smem[];
#else
  static __attribute__((aligned(128))) uint8_t hs_smem[HEALTH_SMALL_SMEM<Rule>];
#endif
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ uint32_t s_bal[HEALTH_SMALL_ROWS][NW];  // "changed" ballot of (row, warp) -> its position in the list
  __shared__ uint32_t s_now[HEALTH_SMALL_ROWS][NW];  // "healthy now" ballot of (row, warp)
  __shared__ uint32_t s_scan[NW], s_alv[NW];
  const uint4* stage = reinterpret_cast<const uint4*>(hs_smem);
  uint32_t* set = reinterpret_cast<uint32_t*>(hs_smem + HEALTH_STAGE_BYTES);
  // keyed: the ascent error flag behind the set; thread 0's copy of the last key of the previous round
  [[maybe_unused]] uint32_t* keyed_err = reinterpret_cast<uint32_t*>(hs_smem + HEALTH_STAGE_BYTES + Rule::SET_CAP * 4);
  [[maybe_unused]] KeyOf<Rule> keyed_last{};
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rows = (n + HEALTH_SMALL_THREADS - 1) / HEALTH_SMALL_THREADS;
  if (tid == 0) {
    mbar_init(&s_bar, 1);
    mbar_fence_init();
    if constexpr (KEYED_RULE<Rule>) *keyed_err = 0;
  }
  if constexpr (Rule::SET_CAP > 0) load_sorted_set(set, rule.set, rule.n_set);
  __syncthreads();
  uint32_t n_alive = 0, phase = 0;
  for (uint32_t r0 = 0; r0 < rows; r0 += SR) {
    // the whole round (<= 192 KiB of the snapshot) is requested at once by the TMA unit: over PCIe what counts
    // is bytes in flight, and a bulk copy keeps them in flight without a register per load
    const uint32_t first = r0 * HEALTH_SMALL_THREADS;
    const uint32_t cnt = min(n - first, SR * HEALTH_SMALL_THREADS);
    if (tid == 0) {
      if constexpr (KEYED_RULE<Rule>)  // the stage still holds the previous (full) round
        if (r0) keyed_last = Rule::K::of(stage[(SR * HEALTH_SMALL_THREADS - 1) * U + Rule::K::UNIT]);
      mbar_arrive_expect_tx(&s_bar, cnt * 16 * U);
      for (uint32_t off = 0; off < cnt * 16 * U; off += 16384)
        tma_load_1d(hs_smem + off, reinterpret_cast<const uint8_t*>(recs + first * U) + off,
                    min(16384u, cnt * 16 * U - off), &s_bar);
    }
    uint32_t was[SR];
    [[maybe_unused]] KeyOf<Rule> pk[SR];
#pragma unroll
    for (uint32_t k = 0; k < SR; k++) {  // the previous state (device memory) meanwhile
      const uint32_t i = first + k * HEALTH_SMALL_THREADS + tid;
      if constexpr (KEYED_RULE<Rule>) {  // keyed: the previous list's entry at the same position
        const bool same = i < n && i < rule.n_prev;
        pk[k] = same ? __ldg(&rule.prev_key[i]) : KeyOf<Rule>{};
        was[k] = same ? __ldg(&rule.prev_state[i]) : 0;
      } else {
        was[k] = i < n ? state[i] : 0;
      }
    }
    mbar_wait(&s_bar, phase);
    phase ^= 1;
#pragma unroll
    for (uint32_t k = 0; k < SR; k++) {
      if (r0 + k < rows) {  // uniform
        const uint32_t i = first + k * HEALTH_SMALL_THREADS + tid;
        const bool in = i < n;
        if constexpr (KEYED_RULE<Rule>) {
          // the join (a miss at the same position searches the previous keys), the ascent check against the
          // record before (the stage, or the last key of the previous round), and this call's key
          using K = typename Rule::K;
          const uint32_t j = k * HEALTH_SMALL_THREADS + tid;
          const KeyOf<Rule> key = K::of(stage[j * U + K::UNIT]);
          if (in) {
            if (!(i < rule.n_prev && K::eq(pk[k], key))) was[k] = rule.search(key);
            if (j ? !K::lt(K::of(stage[(j - 1) * U + K::UNIT]), key) : (r0 && !K::lt(keyed_last, key))) *keyed_err = 1u;
            rule.key[i] = key;
          }
        }
        // (lanes past n compute s from stale stage bytes and use none of it)
        const uint32_t s = rule.next(stage[(k * HEALTH_SMALL_THREADS + tid) * U + Rule::UNIT], was[k], set);
        const bool now = in && (s & 1u) != 0;
        const bool chg = in && (now ? 1u : 0u) != (was[k] & 1u);
        if constexpr (KEYED_RULE<Rule>) {
          if (in) state[i] = (uint8_t)s;  // this call's slot: every record
        } else {
          if (in && s != was[k]) state[i] = (uint8_t)s;
        }
        const uint32_t bc = __ballot_sync(KVG_FULL, chg), bn = __ballot_sync(KVG_FULL, now);
        if (lane == 0) {
          s_bal[r0 + k][warp] = bc;
          s_now[r0 + k][warp] = bn;
        }
        n_alive += now ? 1u : 0u;
      }
    }
    __syncthreads();  // every read of the stage is done before the next round's copy lands in it
  }
  uint32_t alive, total;
  health_small_list(rows, n_alive, s_bal, s_now, s_scan, s_alv, changed_host, alive, total);
  if (tid == 0) {
    hdr_host[0] = alive;
    hdr_host[1] = total;
    if constexpr (KEYED_RULE<Rule>) hdr_host[3] = *keyed_err;
    __threadfence_system();
    *((volatile uint32_t*)&hdr_host[2]) = seq;  // the host polls this word: no driver call on the way back
  }
}

// ------------------------------------------------------------------------------------------------
// mdev type dictionary: label = Trim(raw, "\n") then \s+ -> "_"  (device_plugin.go:341-342);
// canonical id = smallest raw index with an identical label (they are ONE vGpuMap key).
// ------------------------------------------------------------------------------------------------
// The label rule, the one definition the scan's dictionary and the Allocate-time check share, in the reference's two
// steps: mdev_label_trim narrows raw[a, b) to Trim(raw, "\n"); mdev_label_emit feeds the label of that span -- every
// RE2 \s+ run as one '_' -- to emit(c) byte by byte, and stops early (returns false) when emit returns false.
// mdev_label_rule is the two in order.  k_mdev_labels calls them one by one and sets up its outputs in between: set up
// before the trim, they make nvcc lay out its loops differently.
__device__ __forceinline__ void mdev_label_trim(const uint8_t* __restrict__ raw, uint32_t& a, uint32_t& b) {
  while (a < b && raw[a] == '\n') a++;
  while (b > a && raw[b - 1] == '\n') b--;
}
template <class Emit>
__device__ __forceinline__ bool mdev_label_emit(const uint8_t* __restrict__ raw, uint32_t a, uint32_t b, Emit&& emit) {
  for (uint32_t i = a; i < b;) {
    uint8_t c;
    if (d_re2_space(raw[i])) {
      c = '_';
      while (i < b && d_re2_space(raw[i])) i++;
    } else {
      c = raw[i++];
    }
    if (!emit(c)) return false;
  }
  return true;
}
template <class Emit>
__device__ __forceinline__ bool mdev_label_rule(const uint8_t* __restrict__ raw, uint32_t a, uint32_t b, Emit&& emit) {
  mdev_label_trim(raw, a, b);
  return mdev_label_emit(raw, a, b, emit);
}

__global__ void k_mdev_labels(const uint8_t* __restrict__ raw, const uint32_t* __restrict__ raw_off,
                              uint32_t n_types, uint8_t* __restrict__ label,
                              uint32_t* __restrict__ label_len, uint64_t* __restrict__ label_hash) {
  pdl_enter();
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_types) return;
  uint32_t a = raw_off[k], b = raw_off[k + 1];
  mdev_label_trim(raw, a, b);
  uint8_t* out = label + raw_off[k];  // sanitised text is never longer than the raw text
  uint32_t o = 0;
  uint64_t h = 1469598103934665603ull;  // FNV-1a of the label: cheap first-level equality test
  mdev_label_emit(raw, a, b, [&](uint8_t c) {
    out[o++] = c;
    h = (h ^ c) * 1099511628211ull;
    return true;
  });
  label_len[k] = o;
  label_hash[k] = h;
}

// Allocate-time re-check (generic_vgpu_device_plugin.go:216-221): match[k] = 1 iff the label of file k is the name
// (name_len bytes; `name` holds min(name_len, raw_off[n]) of them, all a label can reach).  One CTA, one thread per
// file, striding; the bytes go straight to mapped host memory, then the sequence word the host polls.
static constexpr int LABEL_MATCH_THREADS = 1024;
__global__ void __launch_bounds__(LABEL_MATCH_THREADS) k_mdev_label_match(const uint8_t* __restrict__ raw,
                                                                           const uint32_t* __restrict__ raw_off,
                                                                           uint32_t n, const uint8_t* __restrict__ name,
                                                                           uint64_t name_len, uint8_t* match_host,
                                                                           uint32_t* seq_host, uint32_t seq) {
  pdl_enter();
  for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) {
    uint32_t o = 0;
    const bool same = mdev_label_rule(raw, raw_off[k], raw_off[k + 1],
                                      [&](uint8_t c) { return o < name_len && name[o++] == c; });
    match_host[k] = same && o == name_len;
  }
  __threadfence_system();  // every thread's bytes are on their way before the sequence word
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    *((volatile uint32_t*)seq_host) = seq;
  }
}

// The passthrough plugin's Allocate decisions for every container request of one AllocateRequest
// (generic_device_plugin.go:352-444): the re-check of each requested group's members (:387-399) and the EGM match
// (egmPathsForAllocatedGPUs :159-184).  One CTA per request, striding over the requests when there are more than the
// grid; req[r] = {first member, members, first ID, IDs}.
//   re-check: first_bad_host[r] = the smallest position within the request whose record fails pci_group_check_pass
//     against its wanted group, or its member count.  Each thread stops at its first failure (its positions ascend);
//     the warps reduce with one REDUX each and the block through one shared word.
//   EGM (n_egm > 0): the request's ID handles below n_egm_gpus set their bits of a shared bitmap; then device e is
//     taken (take_host[r * n_egm + e] = 1) iff every handle it lists, egm_gpu[egm_off[e] .. egm_off[e + 1]), has its
//     bit set.  An empty list is taken, as the reference's loop takes it.
// Results go straight to mapped host memory; the last CTA to finish (done counts them; the host zeroes it) writes the
// sequence word the host polls.
static constexpr int GROUP_CHECK_THREADS = 1024;
static constexpr uint32_t ALLOC_CHECK_MAX_GRID = 65535;  // more requests than this: each CTA takes several in turn
__global__ void __launch_bounds__(GROUP_CHECK_THREADS) k_pci_allocate_check(
    const uint4* __restrict__ req, const uint4* __restrict__ recs, const uint32_t* __restrict__ want,
    const uint32_t* __restrict__ ids, const uint32_t* __restrict__ egm_off, const uint32_t* __restrict__ egm_gpu,
    uint32_t n_reqs, uint32_t n_egm, uint32_t n_egm_gpus, uint32_t* done, uint32_t* first_bad_host,
    uint8_t* take_host, uint32_t* seq_host, uint32_t seq) {
  pdl_enter();
  __shared__ uint32_t block_min;
  __shared__ uint32_t present[KVG_ALLOC_MAX_EGM_GPUS / 32];
  const uint32_t n_words = (n_egm_gpus + 31) / 32;
  for (uint32_t r = blockIdx.x; r < n_reqs; r += gridDim.x) {
    const uint4 q = req[r];
    const uint32_t n = q.y;
    if (threadIdx.x == 0) block_min = n;
    if (n_egm)
      for (uint32_t w = threadIdx.x; w < n_words; w += blockDim.x) present[w] = 0;
    uint32_t m = n;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
      if (!pci_group_check_pass(recs[q.x + i], want[q.x + i])) {
        m = i;
        break;
      }
    m = warp_min(m);
    __syncthreads();  // block_min and the bitmap are initialised
    if (lane_id() == 0) atomicMin(&block_min, m);
    if (n_egm)
      for (uint32_t j = threadIdx.x; j < q.w; j += blockDim.x) {
        const uint32_t h = ids[q.z + j];
        if (h < n_egm_gpus) atomicOr(&present[h / 32], 1u << (h % 32));
      }
    __syncthreads();
    if (threadIdx.x == 0) ((volatile uint32_t*)first_bad_host)[r] = block_min;
    for (uint32_t e = threadIdx.x; e < n_egm; e += blockDim.x) {
      uint32_t k = egm_off[e];
      const uint32_t end = egm_off[e + 1];
      while (k < end && (present[egm_gpu[k] / 32] >> (egm_gpu[k] % 32) & 1u)) k++;
      ((volatile uint8_t*)take_host)[(size_t)r * n_egm + e] = k == end;
    }
    __syncthreads();  // block_min and the bitmap are read before the next request resets them
  }
  __threadfence_system();  // this thread's results are on their way before the CTA counts itself done
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(done, 1u) == gridDim.x - 1) {
    __threadfence_system();
    *((volatile uint32_t*)seq_host) = seq;
  }
}
// k_pci_allocate_check's req table (host side): the requests' members and IDs lie one request after another
inline void allocate_check_reqs(const kvg_alloc_req* reqs, uint32_t n_reqs, uint4* req) {
  for (uint32_t r = 0, rec_at = 0, id_at = 0; r < n_reqs; r++) {
    req[r] = make_uint4(rec_at, reqs[r].n_members, id_at, reqs[r].n_ids);
    rec_at += reqs[r].n_members;
    id_at += reqs[r].n_ids;
  }
}
// canonical id = smallest raw index with an identical label: hash + length first (independent,
// pipelined loads), bytes only on a hash match
__global__ void k_mdev_canon(const uint8_t* __restrict__ label, const uint32_t* __restrict__ raw_off,
                             const uint32_t* __restrict__ label_len,
                             const uint64_t* __restrict__ label_hash, uint32_t n_types,
                             uint16_t* __restrict__ canon) {
  pdl_enter();
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_types) return;
  const uint32_t len = label_len[k];
  const uint64_t h = label_hash[k];
  const uint8_t* mine = label + raw_off[k];
  uint32_t c = k;
  for (uint32_t j = 0; j < k; j++) {
    if (label_hash[j] != h || label_len[j] != len) continue;
    const uint8_t* other = label + raw_off[j];
    bool eq = true;
    for (uint32_t t = 0; t < len && eq; t++) eq = other[t] == mine[t];
    if (eq) {
      c = j;
      break;
    }
  }
  canon[k] = (uint16_t)c;
}

// ------------------------------------------------------------------------------------------------
// synthetic snapshots (splitmix64, counter based) — identical to kvo_gen_pci / kvo_gen_mdev
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__global__ void k_gen_pci(uint4* __restrict__ out, uint64_t first, uint32_t n,
                          const uint16_t* __restrict__ nv_ids, uint32_t n_nv_ids,
                          uint32_t group_bits) {
  pdl_enter();
  const uint64_t SEED = 0x10DE000020250711ull;
  const uint16_t other[8] = {0x8086, 0x1002, 0x15b3, 0x1022, 0x144d, 0x14e4, 0x1af4, 0x10df};
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    uint64_t i = first + k;
    uint64_t r0 = mix64(SEED + 2 * i), r1 = mix64(SEED + 2 * i + 1);
    bool nvidia = (r0 & 0xFF) < 128;
    uint32_t vendor = nvidia ? 0x10deu : other[(r0 >> 8) & 7];
    uint32_t device;
    if (nvidia && ((r0 >> 16) & 0xFF) < 230 && n_nv_ids)
      device = nv_ids[(uint32_t)((r0 >> 24) & 0xFFFFFF) % n_nv_ids];
    else
      device = (uint32_t)((r0 >> 24) & 0xFFFF);
    uint32_t d = (uint32_t)((r0 >> 48) & 0xFF);
    uint32_t flags = 0, driver;
    if (d < 154)
      driver = KVG_DRV_VFIO_PCI;
    else if (d < 179)
      driver = KVG_DRV_NVGRACE;
    else if (d < 218)
      driver = 3;
    else if (d < 231)
      driver = 4;
    else {
      driver = KVG_DRV_NONE;
      flags |= KVG_PF_DRIVER_ERR;
    }
    uint32_t g = (uint32_t)(i >> 1);
    if (group_bits) {
      uint32_t mask = group_bits >= 32 ? 0xFFFFFFFFu : ((1u << group_bits) - 1);
      uint32_t hi = g & ~mask, lo = g & mask;
      lo = (lo * 0x9E3779B1u) & mask;
      lo ^= lo >> (group_bits / 2 + 1);
      g = hi | (lo & mask);
    }
    int32_t numa = (int32_t)(r1 & 7) - 1;
    if (((r1 >> 8) & 0xFF) == 0) flags |= KVG_PF_VENDOR_ERR;
    if (((r1 >> 16) & 0xFF) == 0) flags |= KVG_PF_IOMMU_ERR;
    if (((r1 >> 24) & 0xFF) == 0) flags |= KVG_PF_DEVICE_ERR;
    if (((r1 >> 32) & 0xFF) == 0) flags |= KVG_PF_NUMA_ERR;
    uint4 r;
    r.x = (uint32_t)i;
    r.y = vendor | (device << 16);
    r.z = g;
    r.w = driver | (flags << 8) | (((uint32_t)numa & 0xffffu) << 16);
    out[k] = r;
  }
}
__global__ void k_gen_mdev(uint4* __restrict__ out, uint64_t first, uint32_t n) {
  pdl_enter();
  const uint64_t SEED = 0x4D44455600010000ull;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    uint64_t j = first + k;
    uint64_t r0 = mix64(SEED + 2 * j), r1 = mix64(SEED + 2 * j + 1);
    // uuid = BE32(j) | BE64(r0) | BE32(r1 low 32)   (little-endian words hold big-endian bytes)
    uint4 lo;
    lo.x = __byte_perm((uint32_t)j, 0, 0x0123);
    lo.y = __byte_perm((uint32_t)(r0 >> 32), 0, 0x0123);
    lo.z = __byte_perm((uint32_t)r0, 0, 0x0123);
    lo.w = __byte_perm((uint32_t)r1, 0, 0x0123);
    uint32_t flags = 0;
    if (((r1 >> 40) & 0xFF) == 0) flags |= KVG_MF_TYPE_ERR;
    if (((r1 >> 48) & 0xFF) == 0) flags |= KVG_MF_PARENT_ERR;
    if (((r1 >> 56) & 0xFF) == 0) flags |= KVG_MF_NUMA_ERR;
    int32_t numa = (int32_t)((j >> 5) & 3) - 1;
    uint4 hi;
    hi.x = (uint32_t)(j >> 5);
    hi.y = (uint32_t)(r0 >> 56) | (flags << 16);
    hi.z = (uint32_t)numa & 0xffffu;
    hi.w = 0;
    out[2 * (size_t)k] = lo;
    out[2 * (size_t)k + 1] = hi;
  }
}

// L2 flush helper: stream zeros through a buffer larger than L2
__global__ void k_fill(uint4* __restrict__ p, size_t n16, uint32_t v) {
  pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16;
       i += (size_t)gridDim.x * blockDim.x)
    p[i] = make_uint4(v, v, v, v);
}
__global__ void k_fill32(uint32_t* __restrict__ p, size_t n, uint32_t v) {
  pdl_enter();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x)
    p[i] = v;
}

// ------------------------------------------------------------------------------------------------
// K3/K5 default form: classification without any cross-tile dependency.
//   k_classify_ragged  every CTA owns one tile (THREADS x ROWS records, 128-bit streaming loads, all
//                      in flight at once), evaluates the predicate, joins the name and writes its
//                      survivors — already in output format — at the TILE-LOCAL base tile*TILE of a
//                      scratch array, plus one count per tile.  Reads each record once, writes each
//                      survivor once, no waiting on other CTAs: this is the HBM-roofline kernel.
//   k_tile_offsets     exclusive scan of the tile counts (one CTA; n_tiles is ~N/1024)
//   k_pack_survivors   dense, order-preserving copy scratch -> survivors using the known offsets
// The single-pass look-back compaction (k_compact, used below 2 M records) moves fewer bytes,
// but at sizes that are bandwidth-bound each of its CTAs spends most of its lifetime waiting for its
// base offset, which makes it slower end to end than this split form there.
// ------------------------------------------------------------------------------------------------
template <class Op, int THREADS, int ROWS>
__global__ void __launch_bounds__(THREADS) k_classify_ragged(Op op, uint32_t* __restrict__ tile_count,
                                                             uint2* __restrict__ tile_max) {
  pdl_enter();
  using Tile = ClassifyTile<Op, THREADS, ROWS>;
  constexpr uint32_t NW = Tile::NW;
  __shared__ uint32_t s_wtot[NW];
  __shared__ uint2 s_wmax[NW];
  const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
  const uint32_t tile = blockIdx.x;
  Tile ct;
  ct.classify(op, tile);
  if (lane == 0) s_wtot[warp] = ct.wtot;
  __syncthreads();
  uint32_t off = tile * Tile::TILE;  // tile-local base: survivors of a tile stay contiguous and ordered
#pragma unroll
  for (uint32_t w = 0; w < NW; w++) {
    uint32_t c = s_wtot[w];
    if (w < warp) off += c;
    if (w == NW - 1 && threadIdx.x == 0) {
      uint32_t tot = 0;
#pragma unroll
      for (uint32_t v = 0; v < NW; v++) tot += s_wtot[v];
      tile_count[tile] = tot;
    }
  }
  ct.emit(off, [&](uint32_t pos, const typename Op::Item& r, uint32_t i, uint32_t a) { op.emit(pos, r, i, a); });
  // largest keys of the tile (they bound the radix pass counts): per-tile slot, no global atomics
  uint2 m = op.take_maxima();
  m.x = warp_max(m.x);
  m.y = warp_max(m.y);
  if (lane == 0) s_wmax[warp] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint2 t = s_wmax[0];
#pragma unroll
    for (uint32_t w = 1; w < NW; w++) {
      t.x = max(t.x, s_wmax[w].x);
      t.y = max(t.y, s_wmax[w].y);
    }
    tile_max[tile] = t;
  }
}

// exclusive scan of tile_count[0..n_tiles) -> tile_off[0..n_tiles], total -> ctrl->n_surv, and the
// reduction of the per-tile maxima -> ctrl->max_group / max_devkey.  Chained scan: 2048 counts per
// CTA, coalesced, base by decoupled look-back (a few dozen CTAs at most, launched in order).
struct TileOffsetsArgs {
  const uint32_t* tile_count;
  const uint2* tile_max;        // optional per-tile maxima to reduce into ctrl
  const uint32_t* n_items_ptr;  // device-side item count (C_TILE items per tile) or NULL
  uint32_t n_tiles_host;
  uint32_t* tile_off;
  uint32_t* total_out;
  uint64_t* state;
};
struct TileOffsetsArgs2 {
  TileOffsetsArgs o[2];
};
__global__ void __launch_bounds__(KVG_BLOCK) k_tile_offsets(TileOffsetsArgs2 aa, ScanCtrl* ctrl,
                                                            uint32_t epoch) {
  pdl_enter();
  const TileOffsetsArgs A = blockIdx.y ? aa.o[1] : aa.o[0];
  const uint32_t* __restrict__ tile_count = A.tile_count;
  const uint2* __restrict__ tile_max = A.tile_max;
  const uint32_t* n_items_ptr = A.n_items_ptr;
  const uint32_t n_tiles_host = A.n_tiles_host;
  uint32_t* __restrict__ tile_off = A.tile_off;
  uint32_t* total_out = A.total_out;
  uint64_t* state = A.state;
  // n_tiles is either known on the host or derived from a device-side item count (C_TILE items/tile)
  const uint32_t n_tiles = n_items_ptr ? (*n_items_ptr + C_TILE - 1) / C_TILE : n_tiles_host;
  if (blockIdx.x * C_TILE >= n_tiles) {
    if (n_tiles == 0 && blockIdx.x == 0 && threadIdx.x == 0) {
      *total_out = 0;
      tile_off[0] = 0;
    }
    return;
  }
  const uint32_t last_chunk = (n_tiles - 1) / C_TILE;
  __shared__ uint32_t scratch[KVG_WARPS + 1];
  __shared__ uint32_t s_base;
  const uint32_t chunk = blockIdx.x;
  const uint32_t i0 = chunk * C_TILE + threadIdx.x * C_ROWS;
  uint32_t v[C_ROWS], sum = 0, mg = 0, md = 0;
#pragma unroll
  for (uint32_t k = 0; k < C_ROWS; k++) {
    uint32_t i = i0 + k;
    v[k] = i < n_tiles ? tile_count[i] : 0;
    sum += v[k];
    if (tile_max && i < n_tiles) {
      uint2 m = tile_max[i];
      mg = max(mg, m.x);
      md = max(md, m.y);
    }
  }
  uint32_t total;
  uint32_t excl = block_excl_sum(sum, scratch, &total);
  if (warp_id() == 0) {
    uint32_t base = lookback_sum(state, chunk, total, epoch);
    if (lane_id() == 0) {
      s_base = base;
      if (chunk == last_chunk) {
        *total_out = base + total;
        tile_off[n_tiles] = base + total;
      }
    }
  }
  mg = warp_max(mg);
  md = warp_max(md);
  if (lane_id() == 0) {
    if (mg) atomicMax(&ctrl->max_group, mg);
    if (md) atomicMax(&ctrl->max_devkey, md);
  }
  __syncthreads();
  uint32_t run = s_base + excl;
#pragma unroll
  for (uint32_t k = 0; k < C_ROWS; k++) {
    uint32_t i = i0 + k;
    if (i < n_tiles) tile_off[i] = run;
    run += v[k];
  }
}

// dense, order-preserving pack: CTA = one tile, 16-byte units, fully coalesced on both sides
template <int UNITS_PER_ITEM>
__global__ void __launch_bounds__(128) k_pack_survivors(const uint4* __restrict__ ragged,
                                                        const uint32_t* __restrict__ tile_off,
                                                        uint32_t tile_items, uint4* __restrict__ dense) {
  pdl_enter();
  const uint32_t tile = blockIdx.x;
  const uint32_t o0 = tile_off[tile], o1 = tile_off[tile + 1];
  const uint32_t units = (o1 - o0) * UNITS_PER_ITEM;
  const uint4* src = ragged + (size_t)tile * tile_items * UNITS_PER_ITEM;
  uint4* dst = dense + (size_t)o0 * UNITS_PER_ITEM;
  for (uint32_t u = threadIdx.x; u < units; u += blockDim.x) st_stream(dst + u, ld_stream(src + u));
}

}  // namespace kvg
