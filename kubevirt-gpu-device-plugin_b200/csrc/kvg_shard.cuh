// kvg_shard.cuh — the exchange step of the sharded scan (BASELINE.json config 4): one process per GPU,
// records range-sharded in Walk order, results partitioned BY KEY.
//
// Rank r classifies its shard (K3 / K5).  Its survivors stay on rank r (that is the rank's part of
// bdfToIommuMap: concatenating the shards in rank order is Walk order).  For the two group-by maps every
// survivor is sent to the OWNER of its key, owner = key % P, once per ordering:
//   ordering 0  device id (deviceMap)  /  mdev type   (vGpuMap)
//   ordering 1  iommu group (iommuMap) /  parent GPU  (gpuVgpuMap)
// so a rank sends 2 records per survivor whatever P is (constant volume per GPU: weak scaling can hold),
// and receives only the members of the keys it owns.  The first version replicated the whole survivor
// list on every rank: inbound bytes grew with P and efficiency fell to 0.385 at 8 GPUs.
//
// Transport: peer memory (CUDA IPC over NVLink / NVSwitch).  Every rank owns a receive WINDOW
//   [parity w][ordering o][source rank s][cap records]
// mapped by every peer.  The multisplit is stable and its stores ARE the collective:
//   k_shard_send    per 2048-survivor tile: counts per (ordering, owner), 2P chained scans over the tiles, then
//                   every survivor is stored at its final position of region `me` in its owner's window
//                   (match.any ranks: stable), once per ordering; the last CTA to finish publishes the
//                   region counts and a release flag (st.release.sys) in every peer's control block
//                   (count / scan / send as three launches cost two more reads of the list and two more
//                   launch gaps)
//   k_shard_gather  waits for the P flags of the step (ld.acquire.sys), concatenates the P regions of each
//                   ordering — source-rank order == Walk order — into the dense OWNED list the orderings
//                   read, reduces the largest owned keys (radix plan), and the last CTA acknowledges the
//                   window parity to every peer
// Nothing returns to the host between the classify launch and the last ordering kernel.  Spin loops carry
// a ~10 s clock bound and raise an error flag that the fetch turns into KVG_ENCCL.
//
// NCCL fallback (no peer access): the survivors are all-gathered with NCCL (grouped broadcasts — NCCL has no
// allgatherv) and the SAME kernels run in local mode on the gathered list: one source, only the records
// this rank owns are kept.
#pragma once
#include "kvg_common.cuh"
#include "kvg_order.cuh"

namespace kvg {

constexpr int SH_MAX_RANKS = 16;
constexpr uint32_t SH_ALL = 0xffffffffu;
constexpr long long SH_SPIN_LIMIT = 20000000000ll;  // ~10 s of SM clocks, then give up loudly

struct ShardCtrl {  // lives at the head of every rank's window allocation; written by the peers
  unsigned long long flag[2][SH_MAX_RANKS];  // [parity][source rank] = step whose regions are complete
  unsigned long long ack[SH_MAX_RANKS];      // [rank] = last step that rank has consumed
  uint32_t count[2][2][SH_MAX_RANKS];        // [parity][ordering][source rank] records in the region
};
struct ShardPeers {
  uint4* win[SH_MAX_RANKS];        // window base (16-byte units) of every rank, peer-mapped
  ShardCtrl* ctrl[SH_MAX_RANKS];   // control block of every rank, peer-mapped
};
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
#ifndef KVG_HOST_EMU
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
#else
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#endif
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
#ifndef KVG_HOST_EMU
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
  __atomic_store_n(p, v, __ATOMIC_RELEASE);
#endif
}

// record kinds: U = 16-byte units per survivor; keys of ordering 0 / 1
//   PCI  (U = 1)  {addr, iommu_group, device | numa<<16, name_slot}
//   mdev (U = 2)  {uuid[16]}, {parent, type_key | numa<<16, src, pad}
template <int U>
__device__ __forceinline__ uint2 shard_keys(const uint4* rec) {
  if (U == 1) return make_uint2(rec[0].z & 0xffffu, rec[0].y);
  return make_uint2(rec[1].y & 0xffffu, rec[1].x);
}

struct ShardArgs {
  const uint4* list;       // dense survivor list of this rank (NCCL mode: the gathered list)
  const uint32_t* n_ptr;   // its length (device)
  uint64_t* state;         // [2 orderings * P][T] chained-scan words of the per-tile counts (epoch-tagged)
  uint32_t* totals;        // [2][P]
  uint32_t* ticket;        // self-resetting "last CTA" counters: [0] send, [1] gather
  uint32_t T;              // row pitch of state (tiles the launch covers)
  uint32_t P;              // owners (key % P)
  uint32_t Pm;             // floor(2^32 / P) (P = 1: 2^32 - 1): key % P without a division (shard_owner)
  uint32_t me;             // this rank
  uint32_t only;           // SH_ALL: send to every owner; else keep only records owned by `only` (local mode)
  uint32_t n_src;          // regions per (parity, ordering): P, or 1 in local mode
  uint32_t src;            // my region index in the peers' windows: me, or 0 in local mode
  uint64_t region_cap;     // records per region
  uint32_t parity;
  unsigned long long step;
};

// owner of a key = key % P.  A runtime 32-bit modulo is ~20 instructions and every survivor needs four of them;
// with m = floor(2^32 / P) the estimate hi(key * m) is the quotient or one less, so one multiply-high, one
// multiply-subtract and one conditional subtract are exact.
__host__ __device__ __forceinline__ uint32_t shard_magic(uint32_t P) {
  return P <= 1 ? 0xffffffffu : (uint32_t)(0x100000000ull / P);
}
__device__ __forceinline__ uint32_t shard_owner(uint32_t key, const ShardArgs& A) {
#ifdef __CUDA_ARCH__
  const uint32_t qd = __umulhi(key, A.Pm);
#else
  const uint32_t qd = (uint32_t)(((uint64_t)key * A.Pm) >> 32);
#endif
  const uint32_t r = key - qd * A.P;
  return r >= A.P ? r - A.P : r;
}

// window addressing (16-byte units): region (parity, ordering, source) of a window
__device__ __forceinline__ size_t shard_region(const ShardArgs& A, uint32_t o, uint32_t s, int U) {
  return (((size_t)A.parity * 2 + o) * A.n_src + s) * A.region_cap * (size_t)U;
}
// store a record (U units) at position `at` of my region of ordering o in owner q's window
template <int U>
__device__ __forceinline__ void shard_store(const ShardPeers& peers, const ShardArgs& A, uint32_t q, uint32_t o, uint32_t at,
                                            const uint4* rec) {
  uint4* dst = peers.win[q] + shard_region(A, o, A.src, U) + (size_t)at * U;
#pragma unroll
  for (int u = 0; u < U; u++) dst[u] = rec[u];  // NVLink store (or local)
}

// The window parity of this step is rewritten: every owner must have consumed the step that used it two steps
// ago.  Thread q < P waits for owner q's acknowledgement; after SH_SPIN_LIMIT clocks it raises *err and goes on.
__device__ __forceinline__ void shard_wait_acks(const ShardArgs& A, const ShardCtrl* mine, uint32_t* err) {
  const uint32_t q = threadIdx.x;
  if (q >= A.P || A.step <= 2) return;
  const long long t0 = clock64();
  while (ld_acquire_sys(&mine->ack[q]) < A.step - 2) {
    if (clock64() - t0 > SH_SPIN_LIMIT) {
      atomicExch(err, 1u);
      break;
    }
  }
}

// Stable rank of the lane's survivor among the survivors of its warp that go to owner q in ordering o (called by
// the whole warp, one row at a time; q == SH_ALL: no survivor in this lane): the warp's earlier rows counted in
// wcnt[o][q], plus the lanes before it in this row.  One lane per owner then advances wcnt[o][q].
__device__ __forceinline__ uint32_t shard_warp_rank(uint32_t (*wcnt)[SH_MAX_RANKS], uint32_t o, uint32_t q) {
  const uint32_t same = __match_any_sync(KVG_FULL, q);
  const uint32_t before = __popc(same & lanemask_lt());
  const uint32_t prior = q != SH_ALL ? wcnt[o][q] : 0;
  const uint32_t rank = prior + before;
  __syncwarp();
  if (q != SH_ALL && before == 0) wcnt[o][q] = prior + __popc(same);
  __syncwarp();
  return rank;
}

// One launch: count, chained scan, send.  A CTA owns a 2048-survivor tile.  Ranks inside a warp come from
// match.any (one instruction per row and ordering whatever P is); the 2P per-tile counts are combined over the
// tiles by 2P chained scans (look-back), warp c of the CTA running counter c — so the survivor list is read once
// and nothing but the stores stands between the classify kernel and the windows.
template <int U>
__global__ void __launch_bounds__(KVG_BLOCK) k_shard_send(ShardArgs A, ShardPeers peers, const ShardCtrl* mine,
                                                          uint32_t* err, uint32_t epoch) {
  pdl_enter();
  const uint32_t n = *A.n_ptr;
  const uint32_t Tu = (n + C_TILE - 1) / C_TILE;
  const uint32_t tile = blockIdx.x;
  __shared__ uint32_t s_wcnt[KVG_WARPS][2][SH_MAX_RANKS];  // per warp: survivors of every (ordering, owner) -> prefix over the warps
  __shared__ uint32_t s_base[2][SH_MAX_RANKS];             // the tile's position in every (ordering, owner) region
  const uint32_t lane = lane_id(), warp = warp_id();
  const uint32_t active = max(Tu, 1u);  // CTAs that take part (tile 0 also stands for the empty list)
  if (tile >= active) return;
  if (A.only == SH_ALL) shard_wait_acks(A, mine, err);
  if (tile < Tu) {
    const uint32_t base = tile * C_TILE + warp * C_WARP_ITEMS;
    uint4 rec[C_ROWS][U];
    uint32_t q0[C_ROWS], q1[C_ROWS];
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++) {  // all loads in flight first
      const uint32_t i = base + k * 32 + lane;
      q0[k] = q1[k] = SH_ALL;
      if (i < n) {
#pragma unroll
        for (int u = 0; u < U; u++) rec[k][u] = A.list[(size_t)i * U + u];
        const uint2 key = shard_keys<U>(rec[k]);
        q0[k] = shard_owner(key.x, A);
        q1[k] = shard_owner(key.y, A);
      }
    }
    static_assert(2 * SH_MAX_RANKS == 32, "one lane per counter");
    (&s_wcnt[warp][0][0])[lane] = 0;
    __syncwarp();
    // stable position of every survivor among those of my warp that go to the same (ordering, owner)
    uint32_t pos[C_ROWS][2];
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++) {
#pragma unroll
      for (uint32_t o = 0; o < 2; o++) pos[k][o] = shard_warp_rank(s_wcnt[warp], o, o ? q1[k] : q0[k]);
    }
    __syncthreads();
    // warp c: counter c = (ordering, owner) — prefix over the warps in place, tile aggregate, chained scan
    for (uint32_t c = warp; c < 2 * A.P; c += KVG_WARPS) {
      const uint32_t o = c / A.P, q = c - o * A.P;
      const uint32_t v = lane < KVG_WARPS ? s_wcnt[lane][o][q] : 0;
      const uint32_t incl = warp_incl_sum(v);
      const uint32_t agg = __shfl_sync(KVG_FULL, incl, KVG_WARPS - 1);
      if (lane < KVG_WARPS) s_wcnt[lane][o][q] = incl - v;
      const uint32_t excl = lookback_sum(A.state + (size_t)c * A.T, tile, agg, epoch);
      if (lane == 0) {
        s_base[o][q] = excl;
        if (tile == Tu - 1) A.totals[c] = excl + agg;
      }
    }
    __syncthreads();
#pragma unroll
    for (uint32_t k = 0; k < C_ROWS; k++) {
#pragma unroll
      for (uint32_t o = 0; o < 2; o++) {
        const uint32_t q = o ? q1[k] : q0[k];
        if (q != SH_ALL && (A.only == SH_ALL || q == A.only)) {
          shard_store<U>(peers, A, q, o, s_base[o][q] + s_wcnt[warp][o][q] + pos[k][o], rec[k]);
        }
      }
    }
  } else if (n == 0 && tile == 0 && threadIdx.x < 2 * A.P) {
    A.totals[threadIdx.x] = 0;
  }
  // nothing is published here: the grid's completion is the fence (see k_shard_gather)
}

// ---- classify + send in ONE kernel (latency-bound shard sizes) ------------------------------------------------
// The classify kernel already holds every survivor in registers together with its position in the rank's dense
// list; it now also knows its position in the owner's window and stores it there itself.  Per 1024-record tile
// the CTA counts 1 + 2P things — survivors, and survivors per (ordering, owner) — and needs their totals over
// all earlier tiles.  With ~1000 tiles that all start together a chained scan is a chain of dependent L2 round
// trips per counter; instead every tile publishes its COUNTS only (one 32-bit word each: epoch << 11 | count,
// count <= 1024) and sums the words of ALL earlier tiles itself, a thread per earlier tile, every load
// independent: O(T^2 (1 + 2P)) loads from L2 in total — nothing at T ~ 1000 — and no chain.  (The standalone
// k_shard_send keeps the chained scan: it serves the sizes where T^2 is not nothing.)
// CW4 = uint4 loads per tile row: 4 * CW4 >= 1 + 2P.
constexpr uint32_t CS_COUNT_BITS = 11;
#ifndef KVG_CS_MINB_WIDE
#define KVG_CS_MINB_WIDE 7  // P >= 4 (more counters: more registers in the prefix loop); 8 would cap it at 64 registers
#endif
#ifndef KVG_CS_MINB
#define KVG_CS_MINB 8  // CTAs per SM asked of the P <= 3 instantiation: 8 x 132 SMs >= the 977 tiles of a 1 M-record shard (one wave)
#endif
template <class Op, int THREADS, int ROWS, int CW4>
__global__ void __launch_bounds__(THREADS, CW4 <= 2 ? KVG_CS_MINB : KVG_CS_MINB_WIDE) k_classify_send(Op op, ShardArgs A, ShardPeers peers, const ShardCtrl* mine,
                                                           uint32_t* err, uint32_t* tile_words, uint32_t epoch) {
  pdl_enter();
  constexpr int U = Op::UNITS;
  constexpr uint32_t TILE = THREADS * ROWS;
  constexpr uint32_t NW = THREADS / 32;
  constexpr uint32_t CW = 4 * CW4;
  static_assert(TILE < (1u << CS_COUNT_BITS), "a tile count fits the count field");
  static_assert(ROWS <= 8, "warp-local positions (< 32 x ROWS) are packed in bytes");
  __shared__ uint32_t s_wcnt[NW][2][SH_MAX_RANKS];  // per warp: survivors of every (ordering, owner) -> prefix over the warps
  __shared__ uint32_t s_wtot[NW];
  __shared__ uint32_t s_agg[CW], s_excl[CW];
  __shared__ uint32_t s_part[NW][CW];
  // the tile's survivors, staged in tile order: the registers that held the records are free during the prefix
  // below (the P = 8 instantiation needed 118 registers = 4 CTAs per SM = two waves of tiles without this), and
  // the rank's own list is then written with consecutive threads on consecutive records
  __shared__ uint4 s_rec[TILE * U];
  __shared__ uint32_t s_meta[TILE];  // warp | position among the warp's survivors of the same (ordering, owner): 2 + 8 + 8 bits
  static_assert(NW <= 4, "the warp index has two bits in s_meta");
  const uint32_t n_tiles = (op.n + TILE - 1) / TILE;
  const uint32_t active = max(n_tiles, 1u);  // tile 0 also stands for the empty shard
  const uint32_t tile = blockIdx.x;
  if (tile >= active) return;
  const uint32_t lane = lane_id(), warp = threadIdx.x >> 5, tid = threadIdx.x;
  const uint32_t C = 1 + 2 * A.P;  // counters in use: [0] survivors, [1 + o*P + q] survivors of ordering o owned by q
  const uint32_t ep = epoch << CS_COUNT_BITS;
  shard_wait_acks(A, mine, err);
  if (n_tiles == 0) {
    if (tid == 0) op.finish(0);
    if (tid < 2 * A.P) A.totals[tid] = 0;
  } else {
    ClassifyTile<Op, THREADS, ROWS> ct;
    ct.classify(op, tile);
    static_assert(2 * SH_MAX_RANKS == 32, "one lane per counter");
    (&s_wcnt[warp][0][0])[lane] = 0;
    __syncwarp();
    // stable position of every survivor among those of my warp that go to the same (ordering, owner): a byte each
    uint32_t pos0[2] = {0, 0}, pos1[2] = {0, 0};
#pragma unroll
    for (int k = 0; k < ROWS; k++) {
      const bool p = (ct.bal[k] >> lane) & 1u;
      const uint2 key = op.keys(ct.item[k], ct.aux[k]);
      pos0[k >> 2] |= shard_warp_rank(s_wcnt[warp], 0, p ? shard_owner(key.x, A) : SH_ALL) << (8 * (k & 3));  // < 256
      pos1[k >> 2] |= shard_warp_rank(s_wcnt[warp], 1, p ? shard_owner(key.y, A) : SH_ALL) << (8 * (k & 3));
    }
    if (lane == 0) s_wtot[warp] = ct.wtot;
    __syncthreads();
    {
      uint32_t l = 0;
#pragma unroll
      for (uint32_t w = 0; w < NW; w++)
        if (w < warp) l += s_wtot[w];
      ct.emit(l, [&](uint32_t my, const typename Op::Item& r, uint32_t i, uint32_t a) {
        uint4 rec[U];
        op.make(r, i, a, rec);
#pragma unroll
        for (int u = 0; u < U; u++) s_rec[my * U + u] = rec[u];
        const uint32_t k = (i - ct.base) / 32;  // the record's row
        s_meta[my] = warp | (((pos0[k >> 2] >> (8 * (k & 3))) & 0xffu) << 2) | (((pos1[k >> 2] >> (8 * (k & 3))) & 0xffu) << 10);
      });
    }
    // counts of the tile -> published words; the warps' counts become prefixes over the warps in place
    if (warp == 0) {
      for (uint32_t c = lane; c < CW; c += 32) {
        uint32_t agg = 0;
        if (c == 0) {
#pragma unroll
          for (uint32_t w = 0; w < NW; w++) agg += s_wtot[w];
        } else if (c < C) {
          const uint32_t o = (c - 1) / A.P, q = (c - 1) - o * A.P;
#pragma unroll
          for (uint32_t w = 0; w < NW; w++) {
            const uint32_t v = s_wcnt[w][o][q];
            s_wcnt[w][o][q] = agg;
            agg += v;
          }
        }
        s_agg[c] = agg;
        st_relaxed_u32(&tile_words[(size_t)tile * CW + c], ep | agg);
      }
    }
    // totals of all earlier tiles: a thread per earlier tile, CW4 independent 16-byte loads each (fetching 2 or 4
    // earlier tiles per round instead of one was measured: no gain)
    uint32_t acc[CW];
#pragma unroll
    for (uint32_t c = 0; c < CW; c++) acc[c] = 0;
    const uint32_t cmask = (1u << CS_COUNT_BITS) - 1;
    for (uint32_t j = tid; j < tile; j += THREADS) {
      const uint4* row = reinterpret_cast<const uint4*>(tile_words + (size_t)j * CW);
      uint4 x[CW4];
      bool ok;
      long long t0 = 0;
      do {
        ok = true;
#pragma unroll
        for (uint32_t v = 0; v < CW4; v++) {
          x[v] = ld_volatile_v4(row + v);
          ok = ok && ((x[v].x & ~cmask) == ep) && ((x[v].y & ~cmask) == ep) && ((x[v].z & ~cmask) == ep) &&
               ((x[v].w & ~cmask) == ep);
        }
        if (!ok) {  // tile j has not published yet
          if (t0 == 0) t0 = clock64();
          if (clock64() - t0 > SH_SPIN_LIMIT) {
            atomicExch(err, 1u);
            break;
          }
        }
      } while (!ok);
#pragma unroll
      for (uint32_t v = 0; v < CW4; v++) {
        acc[4 * v + 0] += x[v].x & cmask;
        acc[4 * v + 1] += x[v].y & cmask;
        acc[4 * v + 2] += x[v].z & cmask;
        acc[4 * v + 3] += x[v].w & cmask;
      }
    }
#pragma unroll
    for (uint32_t c = 0; c < CW; c++) {
      const uint32_t v = warp_sum(acc[c]);
      if (lane == 0) s_part[warp][c] = v;
    }
    __syncthreads();
    if (tid < CW) {
      uint32_t e = 0;
#pragma unroll
      for (uint32_t w = 0; w < NW; w++) e += s_part[w][tid];
      s_excl[tid] = e;
      if (tile == n_tiles - 1) {
        if (tid == 0) op.finish(e + s_agg[0]);
        else if (tid < C) A.totals[tid - 1] = e + s_agg[tid];
      }
    }
    __syncthreads();
    // survivors: to the rank's dense list (Walk order; consecutive threads, consecutive records) and, once per
    // ordering, to the owner's window
    {
      const uint32_t tile_total = s_agg[0];
      const size_t out0 = s_excl[0];
      uint32_t mx0 = 0, mx1 = 0;
      for (uint32_t l = tid; l < tile_total; l += THREADS) {
        uint4 rec[U];
#pragma unroll
        for (int u = 0; u < U; u++) rec[u] = s_rec[l * U + u];
        const uint32_t meta = s_meta[l];
#pragma unroll
        for (int u = 0; u < U; u++) st_stream(op.out + (out0 + l) * U + u, rec[u]);
        const uint2 key = shard_keys<U>(rec);
        mx0 = max(mx0, key.x);
        mx1 = max(mx1, key.y);
#pragma unroll
        for (uint32_t o = 0; o < 2; o++) {
          const uint32_t q = shard_owner(o ? key.y : key.x, A);
          shard_store<U>(peers, A, q, o, s_excl[1 + o * A.P + q] + s_wcnt[meta & 3u][o][q] + ((meta >> (2 + 8 * o)) & 0xffu), rec);
        }
      }
      // largest keys of the shard (the radix plans): ordering 0 -> max_devkey, ordering 1 -> max_group
      mx0 = warp_max(mx0);
      mx1 = warp_max(mx1);
      if (lane == 0) {
        if (mx0) atomicMax(&op.ctrl->max_devkey, mx0);
        if (mx1) atomicMax(&op.ctrl->max_group, mx1);
      }
    }
  }
  // nothing is published here: the grid's completion is the fence (see k_shard_gather)
}

struct GatherArgs {
  const uint4* window;     // my window (16-byte units)
  uint4* owned[2];         // dense owned list of ordering 0 / 1
  uint32_t* n_own;         // [2] -> ScanCtrl::n_own
  uint32_t* max_key;       // [2]: {max_devkey, max_group} of ScanCtrl (pre-zeroed)
};

// phase bit 0: publish my regions, bit 1: gather.  The product launches both at once; a sequential emulation of
// P ranks has to publish for every rank before any rank can gather.
//
// Publishing lives HERE, not at the end of the send kernel: a kernel boundary is a fence.  This kernel starts
// (griddepcontrol.wait returns) when the send grid has completed and all its stores — the NVLink ones included —
// are performed, so one CTA can publish the counts and the release flags at once.  The send kernels used to end
// with a system-scope fence + ticket per CTA: the fence alone was 45 % of the warp time of k_classify_send.
template <int U>
__global__ void __launch_bounds__(KVG_BLOCK) k_shard_gather(ShardArgs A, GatherArgs G, ShardPeers peers,
                                                            const ShardCtrl* mine, uint32_t* err, uint32_t phase) {
  pdl_enter();
  __shared__ uint32_t s_cnt[2][SH_MAX_RANKS], s_off[2][SH_MAX_RANKS + 1];
  __shared__ uint32_t s_last;
  const uint32_t tid = threadIdx.x;
  if ((phase & 1u) && blockIdx.x == 0 && blockIdx.y == 0 && tid < A.P && (A.only == SH_ALL || tid == A.only)) {
    ShardCtrl* c = peers.ctrl[tid];
    c->count[A.parity][0][A.src] = A.totals[tid];
    c->count[A.parity][1][A.src] = A.totals[A.P + tid];
    __threadfence_system();
    st_release_sys(&c->flag[A.parity][A.src], A.step);
  }
  if (!(phase & 2u)) return;
  if (tid < A.n_src) {  // wait for every source's regions of this step
    const long long t0 = clock64();
    bool ok = true;
    while (ld_acquire_sys(&mine->flag[A.parity][tid]) != A.step) {
      if (clock64() - t0 > SH_SPIN_LIMIT) {
        atomicExch(err, 1u);
        ok = false;
        break;
      }
    }
    s_cnt[0][tid] = ok ? *((volatile const uint32_t*)&mine->count[A.parity][0][tid]) : 0;
    s_cnt[1][tid] = ok ? *((volatile const uint32_t*)&mine->count[A.parity][1][tid]) : 0;
  }
  __syncthreads();
  if (tid < 2) {
    uint32_t run = 0;
    for (uint32_t s = 0; s < A.n_src; s++) {
      s_off[tid][s] = run;
      run += s_cnt[tid][s];
    }
    s_off[tid][A.n_src] = run;
    if (blockIdx.x == 0) G.n_own[tid] = run;
  }
  __syncthreads();
  // blockIdx.y = ordering; regions in source order == Walk order.  The P regions are walked as ONE index space
  // (a record's region = the last one that starts at or before it), four records of a thread in flight per
  // round: region by region and one record at a time, a 1 M-record shard was 13 rounds of a dependent
  // load -> store, and 8 regions at P = 8 were 8 rounds even when each was short.
  const uint32_t o = blockIdx.y;
  uint32_t mx = 0;
  {
    constexpr uint32_t GB = 4;
    const uint32_t total = s_off[o][A.n_src];
    const uint32_t stride = gridDim.x * KVG_BLOCK;
    uint4* dst = G.owned[o];
    for (uint32_t i0 = blockIdx.x * KVG_BLOCK + tid; i0 < total; i0 += GB * stride) {
      uint4 rec[GB][U];
#pragma unroll
      for (uint32_t k = 0; k < GB; k++) {
        const uint32_t i = i0 + k * stride;
        if (i < total) {
          uint32_t sreg = 0;
          for (uint32_t t = 1; t < A.n_src; t++)
            if (i >= s_off[o][t]) sreg = t;
          const uint4* src = G.window + shard_region(A, o, sreg, U) + (size_t)(i - s_off[o][sreg]) * U;
#pragma unroll
          for (int u = 0; u < U; u++) rec[k][u] = ld_stream(src + u);
        }
      }
#pragma unroll
      for (uint32_t k = 0; k < GB; k++) {
        const uint32_t i = i0 + k * stride;
        if (i < total) {
#pragma unroll
          for (int u = 0; u < U; u++) st_stream(dst + (size_t)i * U + u, rec[k][u]);
          const uint2 key = shard_keys<U>(rec[k]);
          mx = max(mx, o ? key.y : key.x);
        }
      }
    }
  }
  mx = warp_max(mx);
  if (lane_id() == 0 && mx) atomicMax(&G.max_key[o], mx);
  // the last CTA acknowledges the window parity to every source
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(&A.ticket[1], 1u) == gridDim.x * gridDim.y - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  if (tid < A.P && A.only == SH_ALL) st_release_sys(&peers.ctrl[tid]->ack[A.me], A.step);
  if (tid == 0) A.ticket[1] = 0;
}

}  // namespace kvg
