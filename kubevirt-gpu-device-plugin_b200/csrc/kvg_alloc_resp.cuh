// kvg_alloc_resp.cuh — the passthrough plugin's AllocateResponse from the raw reads (kvg_pci_allocate_response):
// generic_device_plugin.go:352-444 after the decisions of kvg_alloc_raw.cuh.
//
//   k_aresp_members   one thread per member: its vfio-dev listing (readVFIODev :702-716: the byte-wise least name of
//                     an entry that IsDir (links not followed) and has the prefix "vfio"), reached only with iommufd
//                     on and a member that passed k_araw_members' rule; dev.addr against its DevicesID into the ID's
//                     found flag (requestedDeviceFound, compared as bytes); the member's group string against the
//                     ID's first member's (they name one group, and a link basename never holds '/'); the member's
//                     address into the joined env string.  Threads below n_egm - 1 check that the EGM entry names
//                     ascend strictly byte-wise (ReadDir order).
//   k_aresp_requests  one CTA per request: the first error in the reference's order, then the device specs in append
//                     order, each host path kept at its first occurrence (appendDeviceSpec :108-118) through a key
//                     table of exact path strings, compacted with block scans and written with the EGM paths the
//                     request takes; also the env value's length and key.
// Event order within a request: member p's own events (its re-check failure, or its listing) at 2p, its DevicesID's
// "not found" at 2 * (the ID's last member) + 1, the lookup error after the visited IDs at 2 * n_members + 1.  One
// 64-bit word per event, (order << 8) | kind, so the smallest word is the reference's first error.
#pragma once
#include "kvg_alloc_raw.cuh"
#include "kvg_snap.cuh"

namespace kvg {

constexpr uint32_t ARESP_THREADS = 256;
constexpr uint32_t ARESP_REQ_THREADS = PREF_THREADS;  // pref_excl_sum scans the block
constexpr uint32_t ARESP_MAX_GRID = 65535;             // more requests than this: each CTA takes several in turn
constexpr uint32_t ARESP_NONE = 0xffffffffu;           // a member without a picked vfio-dev entry
constexpr uint32_t ARESP_EV_MISS = 7;                  // a reached listing that was not made: a refusal, not a kind
static_assert(KVG_ARESP_VFIO_NONE < ARESP_EV_MISS, "event kinds");

// One request of the call (host-built): members, visited IDs, candidates, key table and output places
struct ArespReq {
  uint32_t m0, n_mem;   // first member (call-wide), members
  uint32_t v0, n_vis;   // first visited ID (call-wide index into the visit table), visited IDs
  uint32_t lookup;      // 1: a lookup error follows the visited IDs
  uint32_t c0, n_cand;  // first candidate slot (call-wide), candidate paths
  uint32_t t0, mask;    // the key table's first word and mask (n_cand > 0)
  uint32_t s0;          // first spec slot of the result
  uint32_t b0;          // first byte of the spec pool
  uint32_t pad;
};
static_assert(sizeof(ArespReq) == 48, "layout");

// The call's places (host side): per request its ArespReq, per visited ID its visit, and the totals of candidates,
// key-table words, spec slots and pool bytes, each spec bound taken from the inputs.  false: a total exceeds uint32.
struct ArespTotals {
  uint64_t cand, words, slots, bytes;
};
inline bool aresp_plan(const kvg_alloc_req* reqs, uint32_t n_reqs, const kvg_alloc_raw* raw, const kvg_alloc_resp_in* in,
                       ArespReq* rq, uint4* visit, ArespTotals* tot) {
  const uint32_t iommufd = in->iommufd, n_egm = raw->n_egm;
  const size_t n_ent = raw->n_members ? in->vfio_first[raw->n_members] : 0;
  uint64_t egm_bytes = 0;
  for (uint32_t e = 0; e < n_egm; e++)
    egm_bytes += 5 + raw->egm_off[(size_t)e * KVG_AEGM_FIELDS + 1] - raw->egm_off[(size_t)e * KVG_AEGM_FIELDS];
  *tot = ArespTotals{0, 0, 0, 0};
  for (uint32_t r = 0, m = 0, v = 0, id_at = 0; r < n_reqs; id_at += reqs[r].n_ids, r++) {
    ArespReq& q = rq[r];
    q = ArespReq{m, reqs[r].n_members, v, in->n_visited[r], in->lookup_error[r], 0, 0, 0, 0, 0, 0, 0};
    uint64_t bytes = egm_bytes;  // /dev/<name> of every entry
    for (uint32_t k = 0; k < q.n_vis; k++, v++) {
      visit[v] = make_uint4(m, in->id_members[v], id_at + k, r);
      const uint32_t* g = raw->member_off + (size_t)m * KVG_AMEM_FIELDS + KVG_AMEM_GROUP;
      bytes += 14 + 10 + (g[1] - g[0]) + 10ull * iommufd;  // /dev/vfio/vfio, /dev/vfio/<group>, /dev/iommu
      m += in->id_members[v];
    }
    if (iommufd) bytes += 18ull * q.n_mem;  // /dev/vfio/devices/ and a name of the member's listing
    if (iommufd && q.n_mem && n_ent)
      bytes += in->vfio_off[in->vfio_first[q.m0 + q.n_mem]] - in->vfio_off[in->vfio_first[q.m0]];
    const uint64_t n_cand = (uint64_t)iommufd * q.n_mem + (uint64_t)q.n_vis * (2 + iommufd);
    const uint64_t slots = n_cand ? raw_slots(n_cand) : 0;
    if (tot->cand + n_cand > UINT32_MAX || tot->words + slots > UINT32_MAX ||
        tot->slots + n_cand + n_egm > UINT32_MAX || tot->bytes + bytes > UINT32_MAX)
      return false;
    q.c0 = (uint32_t)tot->cand;
    q.n_cand = (uint32_t)n_cand;
    q.t0 = (uint32_t)tot->words;
    q.mask = (uint32_t)(slots ? slots - 1 : 0);
    q.s0 = (uint32_t)tot->slots;
    q.b0 = (uint32_t)tot->bytes;
    tot->cand += n_cand;
    tot->words += slots;
    tot->slots += n_cand + n_egm;
    tot->bytes += bytes;
  }
  return true;
}

// the visit table: per visited ID {first member (call-wide), members, ID index (call-wide), request}
struct ArespArgs {
  const ArespReq* req;
  const uint4* visit;
  uint32_t n_reqs, n_visit, n_mem, iommufd;
  const uint32_t* moff;  // kvg_alloc_raw's member table: the group string is field KVG_AMEM_GROUP
  const uint8_t* mbytes;
  const uint32_t* id_off;
  const uint8_t* id_bytes;
  const uint32_t* aoff;  // [n_mem + 1] dev.addr
  const uint8_t* abytes;
  const uint32_t* lfirst;  // [n_mem + 1] each member's listing entries
  const uint32_t* loff;    // [entries + 1] their names
  const uint8_t* lbytes;
  const uint8_t* ldir;
  const uint8_t* lstate;
  const uint32_t* eoff;  // kvg_alloc_raw's EGM table
  const uint8_t* ebytes;
  uint32_t n_egm;
  const uint4* recs;            // k_araw_members' records: passed iff {.., 0x10de, 0, ..}
  const uint32_t* first_bad;    // k_pci_allocate_check's, per request
  const uint8_t* code_host;     // k_araw_members' codes
  const uint8_t* take;          // k_pci_allocate_check's, [n_reqs * n_egm]
  uint32_t* found;              // [n_visit], zeroed
  unsigned long long* ev;       // [n_reqs], ~0
  uint32_t* pick;               // [n_mem] the picked listing entry, or ARESP_NONE
  uint32_t* cslot;              // the key-table slot of every candidate
  uint64_t* table;
  unsigned long long* verdict_host;  // {group: lowest member, EGM order: lowest entry}; ~0 = none
  uint8_t* env_host;
  uint8_t* error_host;
  uint32_t* error_at_host;
  uint32_t* n_specs_host;
  uint32_t* spec_span_host;
  uint8_t* spec_host;
  uint32_t* env_len_host;
  uint8_t* env_key_host;
  uint32_t* done;  // zeroed; the last CTA of k_aresp_requests writes the sequence word
  uint32_t* seq_host;
  uint32_t seq;
};

// byte-wise order of two strings (Go's string <): -1, 0, 1
__device__ __forceinline__ int aresp_cmp(const uint8_t* x, uint32_t nx, const uint8_t* y, uint32_t ny) {
  for (uint32_t k = 0; k < nx && k < ny; k++)
    if (x[k] != y[k]) return x[k] < y[k] ? -1 : 1;
  return nx == ny ? 0 : (nx < ny ? -1 : 1);
}

// the visit (or candidate block) that holds call-wide member i: the last j with key(j) <= i
template <class K>
__device__ __forceinline__ uint32_t aresp_find(uint32_t lo, uint32_t hi, uint32_t i, K key) {
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (key(mid) <= i) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(ARESP_THREADS) k_aresp_members(ArespArgs a) {
  pdl_enter();
  const uint32_t i = blockIdx.x * ARESP_THREADS + threadIdx.x;
  if (i + 1 < a.n_egm) {  // ReadDir order of the EGM class entries
    const uint32_t* o = a.eoff + (size_t)i * KVG_AEGM_FIELDS;
    const uint32_t* p = o + KVG_AEGM_FIELDS;
    if (aresp_cmp(a.ebytes + o[0], o[1] - o[0], a.ebytes + p[0], p[1] - p[0]) >= 0)
      atomicMin(&a.verdict_host[1], (unsigned long long)(i + 1));
  }
  if (i >= a.n_mem) return;
  const uint32_t j = aresp_find(0, a.n_visit, i, [&](uint32_t k) { return a.visit[k].x; });
  const uint4 v = a.visit[j];
  const ArespReq q = a.req[v.w];
  // the group string: that of the ID's first member, and no '/'
  const uint32_t* mo = a.moff + (size_t)i * KVG_AMEM_FIELDS + KVG_AMEM_GROUP;
  const uint32_t* fo = a.moff + (size_t)v.x * KVG_AMEM_FIELDS + KVG_AMEM_GROUP;
  bool bad_group = !raw_same(a.mbytes, make_uint2(mo[0], mo[1]), make_uint2(fo[0], fo[1]));
  for (uint32_t k = mo[0]; k < mo[1]; k++) bad_group |= a.mbytes[k] == '/';
  if (bad_group) atomicMin(&a.verdict_host[0], (unsigned long long)i);
  // requestedDeviceFound (:401-403)
  const uint32_t a0 = a.aoff[i], a1 = a.aoff[i + 1], d0 = a.id_off[v.z], d1 = a.id_off[v.z + 1];
  if (aresp_cmp(a.abytes + a0, a1 - a0, a.id_bytes + d0, d1 - d0) == 0) a.found[j] = 1;
  // envList: the addresses of every member so far, joined by ','
  volatile uint8_t* env = a.env_host + a0 + i;
  if (i) env[-1] = ',';
  for (uint32_t k = a0; k < a1; k++) env[k - a0] = a.abytes[k];
  // readVFIODev (:404-410), reached only after the member's re-check passed
  uint32_t pick = ARESP_NONE;
  const uint4 rec = a.recs[i];
  if (a.iommufd && rec.y == 0x10deu && rec.z == 0) {
    const uint32_t st = a.lstate[i];
    uint32_t kind = KVG_ARESP_OK;
    if (!(st & KVG_AVFIO_MADE)) {
      kind = ARESP_EV_MISS;
    } else if (st & KVG_AVFIO_FAILED) {
      kind = KVG_ARESP_VFIO_READ;
    } else {
      for (uint32_t e = a.lfirst[i]; e < a.lfirst[i + 1]; e++) {
        const uint32_t n0 = a.loff[e], n1 = a.loff[e + 1];
        if (!a.ldir[e] || n1 - n0 < 4 || a.lbytes[n0] != 'v' || a.lbytes[n0 + 1] != 'f' || a.lbytes[n0 + 2] != 'i' ||
            a.lbytes[n0 + 3] != 'o')
          continue;
        if (pick == ARESP_NONE ||
            aresp_cmp(a.lbytes + n0, n1 - n0, a.lbytes + a.loff[pick], a.loff[pick + 1] - a.loff[pick]) < 0)
          pick = e;
      }
      if (pick == ARESP_NONE) kind = KVG_ARESP_VFIO_NONE;
    }
    if (kind != KVG_ARESP_OK) atomicMin(&a.ev[v.w], ((unsigned long long)(i - q.m0) << 9) | kind);
  }
  a.pick[i] = pick;
}

// ---- request: the specs -------------------------------------------------------------------------------------------
// One host path: a constant prefix and a suffix of input bytes
struct ArespPath {
  const char* pre;
  const uint8_t* suf;
  uint32_t npre, nsuf;
  __device__ __forceinline__ uint32_t len() const { return npre + nsuf; }
  __device__ __forceinline__ uint8_t at(uint32_t k) const { return k < npre ? (uint8_t)pre[k] : suf[k - npre]; }
};
__device__ __forceinline__ ArespPath aresp_path(const char* pre, uint32_t npre, const uint8_t* suf, uint32_t nsuf) {
  ArespPath p;
  p.pre = pre;
  p.npre = npre;
  p.suf = suf;
  p.nsuf = nsuf;
  return p;
}
__device__ __forceinline__ uint64_t aresp_hash(const ArespPath& p) {
  uint64_t h = 1469598103934665603ull;
  for (uint32_t k = 0; k < p.len(); k++) h = (h ^ p.at(k)) * 1099511628211ull;
  return h;
}
__device__ __forceinline__ bool aresp_same(const ArespPath& x, const ArespPath& y) {
  if (x.len() != y.len()) return false;
  for (uint32_t k = 0; k < x.len(); k++)
    if (x.at(k) != y.at(k)) return false;
  return true;
}

// first member of request q's visited ID k, relative to the request
__device__ __forceinline__ uint32_t aresp_cand_base(const ArespArgs& a, const ArespReq& q, uint32_t k) {
  return (a.iommufd ? a.visit[q.v0 + k].x - q.m0 : 0) + k * (2 + a.iommufd);
}
// candidate c of request q in append order: per visited ID its members' /dev/vfio/devices/<vfio> (iommufd), then
// /dev/vfio/vfio, filepath.Join("/dev/vfio", group) and /dev/iommu (iommufd)
__device__ __forceinline__ ArespPath aresp_cand(const ArespArgs& a, const ArespReq& q, uint32_t c) {
  const uint32_t k = aresp_find(0, q.n_vis, c, [&](uint32_t x) { return aresp_cand_base(a, q, x); });
  const uint4 v = a.visit[q.v0 + k];
  uint32_t o = c - aresp_cand_base(a, q, k);
  if (a.iommufd) {
    if (o < v.y) {
      const uint32_t e = a.pick[v.x + o];
      return aresp_path("/dev/vfio/devices/", 18, a.lbytes + a.loff[e], a.loff[e + 1] - a.loff[e]);
    }
    o -= v.y;
  }
  if (o == 0) return aresp_path("/dev/vfio/vfio", 14, nullptr, 0);
  if (o == 2) return aresp_path("/dev/iommu", 10, nullptr, 0);
  const uint32_t* g = a.moff + (size_t)v.x * KVG_AMEM_FIELDS + KVG_AMEM_GROUP;
  const uint8_t* gb = a.mbytes + g[0];
  const uint32_t gl = g[1] - g[0];
  if (gl == 0 || (gl == 1 && gb[0] == '.')) return aresp_path("/dev/vfio", 9, nullptr, 0);  // Join cleans the path
  if (gl == 2 && gb[0] == '.' && gb[1] == '.') return aresp_path("/dev", 4, nullptr, 0);
  return aresp_path("/dev/vfio/", 10, gb, gl);
}

// one spec: slot x of the request, pool bytes at y
__device__ __forceinline__ void aresp_emit(const ArespArgs& a, const ArespReq& q, uint32_t x, uint32_t y,
                                           const ArespPath& p) {
  volatile uint32_t* sp = a.spec_span_host + 2 * ((size_t)q.s0 + x);
  sp[0] = q.b0 + y;
  sp[1] = p.len();
  volatile uint8_t* out = a.spec_host + q.b0 + y;
  for (uint32_t k = 0; k < p.len(); k++) out[k] = p.at(k);
}

__global__ void __launch_bounds__(ARESP_REQ_THREADS) k_aresp_requests(ArespArgs a) {
  pdl_enter();
  __shared__ uint32_t s[ARESP_REQ_THREADS / 32 + 1];
  __shared__ unsigned long long s_ev;
  __shared__ uint32_t s_at;
  const uint32_t t = threadIdx.x;
  for (uint32_t r = blockIdx.x; r < a.n_reqs; r += gridDim.x) {
    const ArespReq q = a.req[r];
    if (t == 0) {
      unsigned long long e = a.ev[r];
      const uint32_t fb = a.first_bad[r];
      if (fb < q.n_mem) {
        const uint32_t kind =
            ((volatile const uint8_t*)a.code_host)[q.m0 + fb] == ARAW_PANIC ? KVG_ARESP_PANIC : KVG_ARESP_UNKNOWN_MEMBER;
        e = min(e, ((unsigned long long)fb << 9) | kind);
      }
      if (q.lookup) e = min(e, ((2ull * q.n_mem + 1) << 8) | KVG_ARESP_UNKNOWN_ID);
      s_ev = e;
      s_at = q.n_vis;
      const uint32_t m_end = q.m0 + q.n_mem;  // envList holds every member of requests 0..r
      ((volatile uint32_t*)a.env_len_host)[r] = m_end ? a.aoff[m_end] + m_end - 1 : 0;
      ((volatile uint8_t*)a.env_key_host)[r] = m_end ? 1 : 0;
    }
    __syncthreads();
    // requestedDeviceFound: an ID none of whose members is the ID itself
    for (uint32_t k = t; k < q.n_vis; k += ARESP_REQ_THREADS) {
      const uint4 v = a.visit[q.v0 + k];
      if (!a.found[q.v0 + k])
        atomicMin(&s_ev, ((2ull * (v.x + v.y - 1 - q.m0) + 1) << 8) | KVG_ARESP_UNKNOWN_ID);
    }
    __syncthreads();
    const unsigned long long ev = s_ev;
    const uint32_t kind = ev == ~0ull ? KVG_ARESP_OK : (uint32_t)(ev & 0xffu);
    if (kind == KVG_ARESP_UNKNOWN_ID) {  // its DevicesID: the one whose last member is at the event, else the lookup
      for (uint32_t k = t; k < q.n_vis; k += ARESP_REQ_THREADS) {
        const uint4 v = a.visit[q.v0 + k];
        if (!a.found[q.v0 + k] && ev >> 8 == 2ull * (v.x + v.y - 1 - q.m0) + 1) s_at = k;
      }
    }
    __syncthreads();
    if (t == 0) {
      ((volatile uint8_t*)a.error_host)[r] = (uint8_t)kind;
      ((volatile uint32_t*)a.error_at_host)[r] =
          kind == KVG_ARESP_OK ? 0u : kind == KVG_ARESP_UNKNOWN_ID ? s_at : (uint32_t)(ev >> 9);
    }
    uint32_t n_out = 0;
    if (kind == KVG_ARESP_OK) {
      uint64_t* table = a.table + q.t0;
      if (q.n_cand)
        for (uint32_t k = t; k <= q.mask; k += ARESP_REQ_THREADS) table[k] = 0;
      __syncthreads();
      // every candidate into the table: the slot of its path, whose word ends as the lowest candidate with it
      for (uint32_t c = t; c < q.n_cand; c += ARESP_REQ_THREADS) {
        const ArespPath p = aresp_cand(a, q, c);
        const unsigned long long mine = (1ull << 32) | c;
        unsigned long long* cas = reinterpret_cast<unsigned long long*>(table);
        for (uint32_t slot = (uint32_t)aresp_hash(p) & q.mask;; slot = (slot + 1) & q.mask) {
          unsigned long long w = ld_relaxed_u64(table + slot);
          if (w == 0) {
            w = atomicCAS(cas + slot, 0ull, mine);
            if (w == 0) {
              a.cslot[q.c0 + c] = slot;
              break;
            }
          }
          if (aresp_same(p, aresp_cand(a, q, (uint32_t)w))) {
            atomicMin(cas + slot, mine);
            a.cslot[q.c0 + c] = slot;
            break;
          }
        }
      }
      __syncthreads();
      // first occurrences in append order, then the EGM paths the request takes (ascending names, all distinct, and
      // none of them /dev, /dev/iommu or under /dev/vfio, so no earlier path can equal one)
      uint32_t bytes = 0;
      for (uint32_t c0 = 0; c0 < q.n_cand; c0 += ARESP_REQ_THREADS) {
        const uint32_t c = c0 + t;
        ArespPath p = aresp_path("", 0, nullptr, 0);
        const bool first = c < q.n_cand && (uint32_t)ld_relaxed_u64(table + a.cslot[q.c0 + c]) == c;
        if (first) p = aresp_cand(a, q, c);
        uint32_t tn, tb;
        const uint32_t x = n_out + pref_excl_sum(first ? 1u : 0u, s, tn);
        const uint32_t y = bytes + pref_excl_sum(p.len(), s, tb);
        if (first) aresp_emit(a, q, x, y, p);
        n_out += tn;
        bytes += tb;
      }
      for (uint32_t e0 = 0; e0 < a.n_egm; e0 += ARESP_REQ_THREADS) {
        const uint32_t e = e0 + t;
        ArespPath p = aresp_path("", 0, nullptr, 0);
        const bool take = e < a.n_egm && a.take[(size_t)r * a.n_egm + e];
        if (take) {
          const uint32_t* o = a.eoff + (size_t)e * KVG_AEGM_FIELDS + KVG_AEGM_NAME;
          p = aresp_path("/dev/", 5, a.ebytes + o[0], o[1] - o[0]);
        }
        uint32_t tn, tb;
        const uint32_t x = n_out + pref_excl_sum(take ? 1u : 0u, s, tn);
        const uint32_t y = bytes + pref_excl_sum(p.len(), s, tb);
        if (take) aresp_emit(a, q, x, y, p);
        n_out += tn;
        bytes += tb;
      }
    }
    if (t == 0) ((volatile uint32_t*)a.n_specs_host)[r] = n_out;
    __syncthreads();  // s_ev, s_at and the scan words are read before the next request resets them
  }
  __threadfence_system();  // this CTA's results are on their way before it counts itself done
  __syncthreads();
  if (t == 0 && atomicAdd(a.done, 1u) == gridDim.x - 1) {
    __threadfence_system();
    *((volatile uint32_t*)a.seq_host) = a.seq;
  }
}

}  // namespace kvg
