// kvg_parse_k1.cuh — K1, the pci.ids parse: text -> device id -> line offset of the lines under vendor 10de.
// Reference semantics: getDeviceName / locateVendor, pkg/device_plugin/device_plugin.go:371-438.
//
// A WARP owns a 4 KiB span of text end to end and never waits for another warp or CTA:
//
//   (no clearing launch: the table and the accumulators are SELF-CLEANING — k_pciids_names resets every
//   dev_off slot it reads, the finalize CTAs consume and reset the two per-image accumulators kept in
//   PciIdsInfo::pad, the resolve CTAs zero the name pool of the parse they belong to, and nv_index is written
//   whole.  Fresh allocations are filled once by the host.)
//   k_pciids_scan      persistent warps; every warp streams a contiguous run of spans through a PRIVATE two-stage ring of
//                      TMA bulk copies (cp.async.bulk ... mbarrier::complete_tx::bytes -> SASS UBLKCP) into
//                      shared memory.  Per span, 4 rows of 1 KiB: two conflict-free LDS.128 per lane and
//                      row -> exact SWAR newline flags -> ONE 32-bit line-start mask per lane and row ->
//                      line count -> first byte of every line start -> header-type lines (neither '\t'
//                      nor '#'): first header, LAST header (the vendor context the span hands to its
//                      successors), "10de" headers (v_off).  Device lines are looked at ONLY in a span that
//                      itself holds a valid "10de" header (one span per image): only vendor 10de is ever
//                      looked up (:424-431), so nothing else is recorded.  One 16-byte summary store per
//                      span; no block barrier, no cross-CTA wait, no epochs.
//   k_pciids_resolve_finalize
//                      CTAs [0, n_files): section end + bufio.Scanner 64 KiB limit of one image (from the
//                      span summaries).  Remaining CTAs, one warp per span: device lines in FRONT of the
//                      span's first header take their context from the nearest earlier span that has a
//                      header (plain loads: the scan kernel has completed); if that context is a valid
//                      "10de" the warp re-reads its span (TMA) and records those lines.  In the shipped
//                      file that is the ~28 spans of the NVIDIA block, 7 % of the text, re-read from L2.
//   k_pciids_names     K2 for image 0: one thread per device id; every id recorded inside the first "10de"
//                      section gets nv_index[id] = line offset - v_off and its sanitised name (:404-414)
//                      at that slot of the pool (warp-cooperative per line).
//
// The table: vendor is fixed (10de) by construction, so the (vendor, device) -> line map is an
// open-addressed table with the IDENTITY hash over the 16-bit device id: capacity equals the key space,
// every probe sequence has length one, and "first line wins" is a fire-and-forget atomicMin (RED.MIN) on
// the slot — no compare-and-swap round trips (the CAS chains of a smaller hashed table were the critical
// path of the single-image parse: chains of dependent L2 atomics in the one span that holds the NVIDIA
// header).
#pragma once
#include "kvg_parse.cuh"

namespace kvg {

#ifndef KVG_K1_SPAN
#define KVG_K1_SPAN 4096
#endif
#ifndef KVG_K1_STAGES
#define KVG_K1_STAGES 1
#endif
constexpr uint32_t K1_SPAN = KVG_K1_SPAN;          // text bytes owned by one warp iteration
constexpr uint32_t K1_HALO = 16;                   // a line starting on the span's last byte is classified
constexpr uint32_t K1_STAGE = K1_SPAN + K1_HALO;   // one TMA transaction (multiple of 16)
constexpr uint32_t K1_STAGES = KVG_K1_STAGES;
constexpr uint32_t K1_WARPS = 4;                   // warps (independent span streams) per CTA
constexpr uint32_t K1_ROWS = K1_SPAN / 1024;       // 4 rows; a lane owns bytes [l*16, +16) of both row halves
constexpr uint32_t K1_SMEM = K1_WARPS * K1_STAGES * K1_STAGE;
constexpr uint32_t K1_VALID_10DE = 0x10000u | 0x10deu;
constexpr uint32_t K1_IDS = 65536;                 // slots of one image's table
static_assert(K1_STAGE % 16 == 0, "bulk copies move multiples of 16 bytes");
static_assert(P_TILE % K1_SPAN == 0, "kvg_text_pad covers whole spans + halo");

// per-span summary (one 16-byte store by lane 0; read by the resolve / finalize CTAs)
//   x  file offset of the first header-type line owned, or NONE
//   y  1: the span holds at least one '\n' inside the file, else 0
//   z  unused
//   w  0: no header in the span, else 0x80000000 | valid<<16 | vendor of the LAST header
struct K1Args {
  const uint8_t* text;  // image 0; image f at text + f*stride
  uint64_t stride;
  uint32_t len;
  uint32_t n_files;
  uint32_t spans_per_file;
  uint32_t n_spans;
  uint32_t* dev_off;  // [n_files][K1_IDS] line offset of the FIRST "\t<id>" line under a 10de header, or NONE
  PciIdsInfo* info;   // [n_files]; pad[0] = max over ~offset of the "10de" headers seen (0: none), pad[1] = newlines:
                      // accumulators of the scan kernel, consumed and reset by the finalize CTA of the image
  uint4* span_sum;    // [n_spans]
  uint4* pool;        // name pool of image 0 (pool16 x 16 bytes): zeroed by the resolve CTAs, filled by k_pciids_names
  uint32_t pool16;
};

// bit 7 of byte b is CLEAR iff the LOW SEVEN bits of byte b of w are those of '\n' — true for '\n' and for
// 0x8A.  Three instructions per word ((w ^ c) & m as ONE LOP3 with a constant in a register, an add, and the
// shift that the combine needs anyway); the exact test costs one more per word, and bytes >= 0x80 are rare in
// pci.ids, so k1_row_mask pays for them only in the cells that have one.
__device__ __forceinline__ uint32_t k1_lo7(uint32_t w) {
#ifndef KVG_HOST_EMU
  uint32_t t;
  asm("lop3.b32 %0, %1, 0x0A0A0A0A, 0x7F7F7F7F, 0x28;" : "=r"(t) : "r"(w));  // (w ^ 0x0A..) & 0x7F..
  return t + 0x7F7F7F7Fu;
#else
  return ((w ^ 0x0A0A0A0Au) & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;
#endif
}
// bit 7 of every byte of word k -> bit position 8*b + k
#define K1_GATHER(f, va, vb)                                                                                   \
  ((((f(va.x)) >> 7) & 0x01010101u) | (((f(va.y)) >> 6) & 0x02020202u) | (((f(va.z)) >> 5) & 0x04040404u) |    \
   (((f(va.w)) >> 4) & 0x08080808u) | (((f(vb.x)) >> 3) & 0x10101010u) | (((f(vb.y)) >> 2) & 0x20202020u) |    \
   (((f(vb.z)) >> 1) & 0x40404040u) | ((f(vb.w)) & 0x80808080u))
#define K1_IDENT(w) (w)
// Line-start mask of one lane and row: the lane's 16 bytes of the row's first half (words k = 0..3) and of
// its second half (words k = 4..7).  Bit t = 8*b + k is set iff byte b of word k is '\n'.  Exact.
__device__ __forceinline__ uint32_t k1_row_mask(const uint4& va, const uint4& vb) {
  uint32_t m = K1_GATHER(k1_lo7, va, vb);  // bit set: NOT a newline (low seven bits differ)
  const uint32_t hi = (va.x | va.y | va.z | va.w | vb.x | vb.y | vb.z | vb.w) & 0x80808080u;
  if (hi) m |= K1_GATHER(K1_IDENT, va, vb);  // a byte >= 0x80 is not a newline whatever its low bits are
  return ~m;
}
// offset (inside the lane's row: + r * 1024 + lane * 16) of the byte behind mask bit t
__host__ __device__ __forceinline__ uint32_t k1_bit_off(uint32_t t) {
  const uint32_t k = t & 7u, b = t >> 3;
  return ((k & 4u) << 7) + ((k & 3u) << 2) + b;
}

// header-type line at span-relative offset p (0 .. 4096): (p+1)<<17 | valid<<16 | vendor   (never 0;
// keys ascend with p, so "max" == "latest")
__device__ __forceinline__ uint32_t k1_header_key(const uint8_t* sm, uint32_t p) {
  return ((p + 1) << 17) | parse_hex4(sm + p);
}

// A span whose tail lies beyond EOF (the last span of an image): padding bytes become 0 in shared memory, so
// that no mask needs an EOF case (the one remaining rule — a '\n' that is the file's LAST byte is counted but
// starts no line — is applied to the masks by the callers).
__device__ __forceinline__ void k1_patch_eof(uint8_t* sm, uint32_t a, uint32_t len, uint32_t lane) {
  const uint32_t inside = len - a;  // <= K1_SPAN here
  for (uint32_t p = inside + lane; p < K1_STAGE; p += 32) sm[p] = 0;
#ifndef KVG_HOST_EMU
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes; TMA refills the stage later
#endif
  __syncwarp();
}

// Device lines ("\t" + 4 lower hex) of the span whose vendor context is a valid "10de" -> table.
//   ctx_in     context carried INTO the span (valid<<16 | vendor, or 0 = unknown)
//   only_head  true: stop at the span's first header (the resolve pass: the lines behind it were
//              handled by the scan pass); false: lines in front of the first header are skipped
//              when ctx_in is unknown
// Rare path (the one span per image that holds a "10de" header, and the spans of the NVIDIA block), written
// for clarity: 512-byte rows in order with natural-order masks, one warp scan per row that has a header.
__device__ __noinline__ void k1_record_lines(const uint8_t* sm, uint32_t* dev_off, uint32_t len, uint32_t a,
                                             uint32_t lane, bool extra, uint32_t ctx_in, bool only_head) {
  uint32_t carry = ctx_in ? (ctx_in & 0x1ffffu) : 0u;  // key of the latest header so far (in-span keys carry
                                                       // position bits: they always beat the carried-in one)
  bool stop = false;                                   // only_head: a header has been seen in an earlier row
#pragma unroll 1
  for (uint32_t r = 0; r < K1_SPAN / 512; r++) {
    const uint32_t cell = r * 512 + lane * 16;
    uint32_t ls = nl_mask16(*reinterpret_cast<const uint4*>(sm + cell));
    // a '\n' that is the file's last byte starts no line (bytes beyond EOF were patched to 0 already)
    if (a + cell < len && a + cell + 16 >= len) ls &= ~(1u << (len - 1 - a - cell));
    const bool first_cell = r == 0 && extra;
    // last header among this lane's lines of the row, and whether the row holds any header
    uint32_t hk = 0;
    if (first_cell) {
      const uint32_t b0 = sm[0];
      if (b0 != '\t' && b0 != '#') hk = k1_header_key(sm, 0);
    }
    for (uint32_t mm = ls; mm; mm &= mm - 1) {
      const uint32_t p = cell + (uint32_t)__ffs(mm);
      const uint32_t b0 = sm[p];
      if (b0 != '\t' && b0 != '#') hk = k1_header_key(sm, p);
    }
    uint32_t before = carry;
    bool hdr_before_me = stop;  // only_head: is there a header of this span in front of my cell?
    if (__any_sync(KVG_FULL, hk != 0)) {
      const uint32_t incl = warp_incl_max(hk);
      uint32_t excl = __shfl_up_sync(KVG_FULL, incl, 1);
      if (lane == 0) excl = 0;
      if (excl) {
        before = excl;
        hdr_before_me = true;
      }
      carry = __shfl_sync(KVG_FULL, incl, 31);
      stop = true;
    }
    if (only_head && hdr_before_me) continue;
    // walk my lines of the row in order with the running context
    uint32_t ctx = before;
    bool done = false;
    bool first_iter = first_cell;
    uint32_t mm = ls;
    while (!done && (first_iter || mm)) {
      uint32_t p;
      if (first_iter) {
        p = 0;
        first_iter = false;
      } else {
        p = cell + (uint32_t)__ffs(mm);
        mm &= mm - 1;
      }
      const uint32_t b0 = sm[p];
      if (b0 == '\t') {
        if ((ctx & 0x1ffffu) == K1_VALID_10DE) {
          const uint32_t dv = parse_hex4(sm + p + 1);
          if (dv & 0x10000u) atomicMin(&dev_off[dv & 0xffffu], a + p);  // first line wins (:388-402)
        }
      } else if (b0 != '#') {
        if (only_head) done = true;  // the span's first header: the scan pass owns everything behind it
        ctx = k1_header_key(sm, p);
      }
    }
  }
}

#ifndef KVG_K1_MINCTAS
#define KVG_K1_MINCTAS 1
#endif
#ifndef KVG_K1_UNROLL
#define KVG_K1_UNROLL 4  // rows of a span unrolled in the scan loop (measured at 256 images: 4 is faster than 1 or 2)
#endif
constexpr int K1_UNROLL = KVG_K1_UNROLL;
__global__ void __launch_bounds__(K1_WARPS * 32, KVG_K1_MINCTAS) k_pciids_scan(K1Args A) {
  pdl_enter();
#ifndef KVG_HOST_EMU
  extern __shared__ __align__(128) uint8_t k1_smem[];
#else
  static __attribute__((aligned(128))) uint8_t k1_smem[K1_SMEM];
#endif
  __shared__ __align__(8) uint64_t bar[K1_WARPS][K1_STAGES];
  __shared__ uint16_t s_off[32];  // mask bit -> byte offset + 1 (the line start behind the newline)
  const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
  if (threadIdx.x < 32) s_off[threadIdx.x] = (uint16_t)(k1_bit_off(threadIdx.x) + 1);
  __syncthreads();  // the only block-wide barrier: before any warp can leave
  // every warp owns a CONTIGUOUS run of spans (of the concatenated images): the next span is the next 4 KiB
  const uint32_t GW = gridDim.x * K1_WARPS, gw = blockIdx.x * K1_WARPS + warp;
  const uint32_t per = (A.n_spans + GW - 1) / GW;
  const uint32_t s0 = gw * per;
  if (s0 >= A.n_spans) return;  // warp-uniform
  const uint32_t my_count = min(per, A.n_spans - s0);
  uint8_t* ring = k1_smem + warp * (K1_STAGES * K1_STAGE);
  const uint32_t spf = A.spans_per_file;

  // (image, span-in-image) of my next span to FETCH (ff, fj) and to PROCESS (f, j): one division per warp
  uint32_t ff = s0 / spf, fj = s0 - ff * spf;
  uint32_t f = ff, j = fj;
  auto issue = [&](uint32_t i) {  // lane 0: bulk copy of my i-th span into stage i % 2
    const uint8_t* src = A.text + (uint64_t)ff * A.stride + (uint64_t)fj * K1_SPAN;
    uint64_t* b = &bar[warp][i % K1_STAGES];
    mbar_arrive_expect_tx(b, K1_STAGE);
    tma_load_1d(ring + (i % K1_STAGES) * K1_STAGE, src, K1_STAGE, b);
    if (++fj == spf) {
      fj = 0;
      ff++;
    }
  };
  if (lane == 0) {
    for (uint32_t s = 0; s < K1_STAGES; s++) mbar_init(&bar[warp][s], 1);
    mbar_fence_init();
    for (uint32_t s = 0; s < K1_STAGES && s < my_count; s++) issue(s);
  }
  __syncwarp();

  for (uint32_t i = 0; i < my_count; i++) {
    const uint32_t a = j * K1_SPAN;
    uint8_t* sm = ring + (i % K1_STAGES) * K1_STAGE;
    mbar_wait(&bar[warp][i % K1_STAGES], (i / K1_STAGES) & 1);
    const bool full = a + K1_SPAN < A.len;  // every byte of the span and its successor lie inside the file
    if (!full) k1_patch_eof(sm, a, A.len, lane);

    uint32_t n_nl = 0, any = 0;
    const bool extra = j == 0 && lane == 0 && A.len > 0;  // the line at offset 0 of the image
    // a '\n' that is the file's last byte is counted but starts no line: its row and mask bit (this lane's, else none)
    uint32_t eof_row = K1_ROWS, eof_bit = 0;
    if (!full) {
      const uint32_t q = A.len - 1 - a;  // span-relative position of the last byte (< K1_SPAN)
      const uint32_t h = (q >> 9) & 1u, l = (q >> 4) & 31u, o = q & 15u;
      if (l == lane) {
        eof_row = q >> 10;
        eof_bit = 1u << (((o & 3u) << 3) | (h << 2) | (o >> 2));
      }
    }

    // header-type lines: first byte of every line start
    uint32_t last_key = 0, first_hdr = P_NONE;
    bool saw_10de = false;
    if (extra) {
      const uint32_t b0 = sm[0];
      if (b0 != '\t' && b0 != '#') {
        last_key = k1_header_key(sm, 0);
        first_hdr = 0;
        if ((last_key & 0x1ffffu) == K1_VALID_10DE) {
          saw_10de = true;
          atomicMax(&A.info[f].pad[0], ~a);
        }
      }
    }
    const uint8_t* cell = sm + lane * 16;
    auto header_at = [&](uint32_t po) {  // a header-type line starts at cell + po
      const uint32_t p = po + lane * 16;
      const uint32_t k = k1_header_key(sm, p);
      last_key = max(last_key, k);  // mask bits are not in position order: keys carry the position
      first_hdr = min(first_hdr, p);
      if ((k & 0x1ffffu) == K1_VALID_10DE) {
        saw_10de = true;
        atomicMax(&A.info[f].pad[0], ~(a + p));
      }
    };
    // One row (1 KiB) per iteration: the row's mask is consumed where it is made (51 registers instead of 72 when
    // the four masks were kept for a second loop).  Fully unrolled by default: instruction-level parallelism across
    // rows beats the smaller code (11 % of the samples are instruction-cache misses either way).
#pragma unroll K1_UNROLL
    for (uint32_t r = 0; r < K1_ROWS; r++) {
      const uint4 va = *reinterpret_cast<const uint4*>(sm + r * 1024 + lane * 16);
      const uint4 vb = *reinterpret_cast<const uint4*>(sm + r * 1024 + 512 + lane * 16);
      uint32_t ls = k1_row_mask(va, vb);
      n_nl += (uint32_t)__popc(ls);
      any |= ls;
      if (r == eof_row) ls &= ~eof_bit;
      // A lane's row is two 16-byte cells and a 16-byte cell rarely holds more than one line start (the shortest
      // lines of the file are about that long).  The FIRST line start of each cell is handled without a loop —
      // independent chains (find bit -> offset -> first byte) in flight together; what is left (a cell with two
      // or more newlines) goes through the loop below.
      uint32_t rest = 0;
#pragma unroll
      for (uint32_t h = 0; h < 2; h++) {
        const uint32_t m = ls & (h ? 0xF0F0F0F0u : 0x0F0F0F0Fu);  // mask bit 8b + k: k < 4 is the first cell
        const uint32_t t = (uint32_t)__ffs((int)(m | 0x80000000u)) - 1;  // m == 0: any valid index
        const uint32_t po = r * 1024 + s_off[t];
        const uint32_t b0 = cell[po];
        if (m != 0 && b0 != '\t' && b0 != '#') header_at(po);
        rest |= m & (m - 1);
      }
      for (uint32_t mm = rest; mm; mm &= mm - 1) {
        const uint32_t po = r * 1024 + s_off[(uint32_t)__ffs(mm) - 1];
        const uint32_t b0 = cell[po];
        if (b0 != '\t' && b0 != '#') header_at(po);
      }
    }
    last_key = warp_max(last_key);
    first_hdr = warp_min(first_hdr);
    n_nl = warp_sum(n_nl);
    const bool has_nl = __any_sync(KVG_FULL, any != 0);
    if (__any_sync(KVG_FULL, saw_10de))
      k1_record_lines(sm, A.dev_off + (size_t)f * K1_IDS, A.len, a, lane, extra, 0u, false);
    if (lane == 0) {
      if (n_nl) atomicAdd(&A.info[f].pad[1], n_nl);
      A.span_sum[s0 + i] = make_uint4(first_hdr == P_NONE ? P_NONE : a + first_hdr, has_nl ? 1u : 0u, 0u,
                                      last_key ? (0x80000000u | (last_key & 0x1ffffu)) : 0u);
    }
    __syncwarp();  // every lane is done with the stage before it is refilled
    if (lane == 0 && i + K1_STAGES < my_count) issue(i + K1_STAGES);
    if (++j == spf) {
      j = 0;
      f++;
    }
  }
}

// CTAs [0, n_files): section end + scanner limit of one image.  Remaining CTAs: resolve, one warp per span.
constexpr uint32_t K1_RWARPS = KVG_BLOCK / 32;
__global__ void __launch_bounds__(KVG_BLOCK) k_pciids_resolve_finalize(K1Args A) {
  pdl_enter();
#ifndef KVG_HOST_EMU
  extern __shared__ __align__(128) uint8_t k1r_smem[];
#else
  static __attribute__((aligned(128))) uint8_t k1r_smem[K1_RWARPS * K1_STAGE];
#endif
  __shared__ __align__(8) uint64_t bar[K1_RWARPS];
  __shared__ uint32_t s_end, s_limit, s_hdr_span;
  if (blockIdx.x < A.n_files) {
    // ---------------------------------------------------------------- finalize image f
    const uint32_t f = blockIdx.x;
    const uint8_t* text = A.text + (uint64_t)f * A.stride;
    const uint4* sum = A.span_sum + (size_t)f * A.spans_per_file;
    PciIdsInfo* info = &A.info[f];
    const uint32_t acc_v = info->pad[0], acc_lines = info->pad[1];  // complete: the scan kernel has finished
    const uint32_t V = acc_v ? ~acc_v : P_NONE;
    // stage the span that owns the line starting at V (the byte scan below reads neighbours)
    const uint32_t tv = (V == P_NONE || V == 0) ? 0 : (V - 1) / K1_SPAN;
    if (V != P_NONE) {
      const uint4* src = reinterpret_cast<const uint4*>(text + (size_t)tv * K1_SPAN);
      for (uint32_t i = threadIdx.x; i < K1_STAGE / 16; i += blockDim.x)
        reinterpret_cast<uint4*>(k1r_smem)[i] = src[i];
    }
    if (threadIdx.x == 0) {
      s_end = A.len;
      s_limit = A.len;
      s_hdr_span = P_NONE;
    }
    __syncthreads();
    // bufio.Scanner: a line with no '\n' in its first 64 KiB ends the scan (ErrTooLong).  Two newlines
    // inside one span are < 4 KiB apart and newlines of neighbouring spans < 8 KiB, so only a run of
    // newline-free spans can make a line that long: a thread per span that HAS a newline (plus the virtual
    // span behind the last, standing for EOF) looks back; only if >= 14 spans in between are empty does it
    // locate the two newlines exactly.
    for (uint32_t t = threadIdx.x; t <= A.spans_per_file; t += blockDim.x) {
      if (t < A.spans_per_file && sum[t].y == 0) continue;
      int u = (int)t - 1;
      while (u >= 0 && sum[u].y == 0) u--;
      if (((uint32_t)((int)t - u) + 1) * K1_SPAN < SCAN_TOKEN_MAX) continue;  // that line cannot reach 64 KiB
      uint32_t fn = A.len;            // first newline at or after span t
      if (t < A.spans_per_file) {
        fn = t * K1_SPAN;
        while (text[fn] != '\n') fn++;
      }
      uint32_t line_start = 0;
      if (u >= 0) {
        uint32_t q = min(A.len, ((uint32_t)u + 1) * K1_SPAN) - 1;  // last newline of span u
        while (text[q] != '\n') q--;
        line_start = q + 1;
      }
      if (line_start < A.len && fn - line_start >= SCAN_TOKEN_MAX) atomicMin(&s_limit, line_start);
    }
    __syncthreads();
    const uint32_t limit = s_limit;
    if (V == P_NONE || V >= limit) {  // vendor line never reached (:382-385)
      if (threadIdx.x == 0) {
        PciIdsInfo z;
        z.v_off = z.sec_end = P_NONE;
        z.n_entries = 0;
        z.n_lines = acc_lines;
        z.limit = limit;
        z.overflow = z.pad[0] = z.pad[1] = 0;  // accumulators back to "nothing seen" for the next parse
        *info = z;
      }
      return;
    }
    // first header-type line after V: inside V's span from the staged bytes, else from the span summaries
    const uint32_t a = tv * K1_SPAN;
    const uint32_t span_end = min(A.len, a + K1_SPAN + 1);  // line starts owned by the span: <= a + SPAN
    for (uint32_t p = V + 1 + threadIdx.x; p < span_end; p += blockDim.x) {
      if (k1r_smem[p - 1 - a] == '\n') {
        const uint8_t b0 = k1r_smem[p - a];
        if (b0 != '\t' && b0 != '#') atomicMin(&s_end, p);
      }
    }
    for (uint32_t t = tv + 1 + threadIdx.x; t < A.spans_per_file; t += blockDim.x)
      if (sum[t].x != P_NONE) atomicMin(&s_hdr_span, t);
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t e = s_end;
      if (e == A.len && s_hdr_span != P_NONE) e = sum[s_hdr_span].x;
      PciIdsInfo z;
      z.v_off = V;
      z.sec_end = min(e, limit);
      z.n_entries = 0;  // counted by k_pciids_names
      z.n_lines = acc_lines;
      z.limit = limit;
      z.overflow = z.pad[0] = z.pad[1] = 0;  // accumulators back to "nothing seen" for the next parse
      *info = z;
    }
    return;
  }
  // ------------------------------------------------------------------ resolve: one warp per span
  // first the name pool of this parse (k_pciids_names, the next kernel, is its only writer)
  for (uint32_t i = (blockIdx.x - A.n_files) * KVG_BLOCK + threadIdx.x; i < A.pool16; i += (gridDim.x - A.n_files) * KVG_BLOCK)
    A.pool[i] = make_uint4(0, 0, 0, 0);
  const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
  const uint32_t span = (blockIdx.x - A.n_files) * K1_RWARPS + warp;
  if (span >= A.n_spans) return;  // warp-uniform; no block barrier on this path
  const uint32_t f = span / A.spans_per_file, j = span - f * A.spans_per_file;
  if (j == 0) return;  // nothing in front of the image's first span
  const uint4 mine = A.span_sum[span];
  const uint32_t a = j * K1_SPAN;
  // the span's first owned line start is already a header: no line of it depends on earlier spans
  // (offset a+1 is the earliest line start a span with j > 0 can own)
  if (mine.x == a + 1) return;
  uint32_t ctx = 0;  // no header before this span: no vendor context, nothing is recorded
  for (int base = (int)j - 1; base >= 0; base -= 32) {
    const int u = base - (int)lane;  // lane 0 looks at the nearest span
    const uint32_t st = u >= 0 ? A.span_sum[(size_t)f * A.spans_per_file + (uint32_t)u].w : 0u;
    const uint32_t m = __ballot_sync(KVG_FULL, st != 0);
    if (m) {
      ctx = __shfl_sync(KVG_FULL, st, (uint32_t)__ffs(m) - 1);
      break;
    }
  }
  if ((ctx & 0x1ffffu) != K1_VALID_10DE) return;
  uint8_t* sm = k1r_smem + warp * K1_STAGE;
  if (lane == 0) {
    mbar_init(&bar[warp], 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(&bar[warp], K1_STAGE);
    tma_load_1d(sm, A.text + (uint64_t)f * A.stride + (uint64_t)a, K1_STAGE, &bar[warp]);
  }
  __syncwarp();
  mbar_wait(&bar[warp], 0);
  if (!(a + K1_SPAN < A.len)) k1_patch_eof(sm, a, A.len, lane);
  k1_record_lines(sm, A.dev_off + (size_t)f * K1_IDS, A.len, a, lane, false, ctx & 0x1ffffu, true);
}

// K2 for image 0: thread per device id (strided so that runs of consecutive ids — the shipped file has
// many — spread over the warps); every id recorded inside the first "10de" section publishes
// nv_index[id] = slot (= line offset - v_off) and, warp-cooperatively, its sanitised name at pool + slot
// (u16 length + bytes); every other id publishes NONE, so nv_index never needs clearing.  Counts the ids
// recorded.  Every slot read is reset (the table is self-cleaning), the tables of the other images included.
// Launch with K1_NAME_CTAS CTAs (image 0), plus any number of further CTAs that only reset the tables of the
// other images.
constexpr uint32_t K1_NAME_CTAS = K1_IDS / 32 / KVG_WARPS;
__global__ void __launch_bounds__(KVG_BLOCK) k_pciids_names(uint32_t* __restrict__ dev_off, uint32_t n_files,
                                                            const uint8_t* __restrict__ text, uint32_t len,
                                                            PciIdsInfo* __restrict__ info,
                                                            uint32_t* __restrict__ nv_index,
                                                            uint8_t* __restrict__ pool) {
  pdl_enter();
  if (blockIdx.x >= K1_NAME_CTAS) {
    // the tables of images 1 .. n_files - 1 (throughput runs parse many images; nothing reads their slots)
    uint4* rest = reinterpret_cast<uint4*>(dev_off + K1_IDS);
    const size_t rest16 = (size_t)(n_files - 1) * (K1_IDS / 4);
    const size_t nth = (size_t)(gridDim.x - K1_NAME_CTAS) * KVG_BLOCK;
    const uint4 none = make_uint4(P_NONE, P_NONE, P_NONE, P_NONE);
    for (size_t i0 = (size_t)(blockIdx.x - K1_NAME_CTAS) * KVG_BLOCK + threadIdx.x; i0 < rest16; i0 += 4 * nth) {
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; u++)  // four loads in flight per thread
        v[u] = i0 + u * nth < rest16 ? rest[i0 + u * nth] : none;
#pragma unroll
      for (int u = 0; u < 4; u++)
        if ((v[u].x & v[u].y & v[u].z & v[u].w) != P_NONE) rest[i0 + u * nth] = none;
    }
    return;
  }
  const uint32_t V = info->v_off, E = info->sec_end;
  const uint32_t lane = lane_id();
  const uint32_t n_warps = K1_NAME_CTAS * KVG_WARPS;
  const uint32_t w = blockIdx.x * KVG_WARPS + warp_id();
  const uint32_t id = lane * n_warps + w;
  const uint32_t off = id < K1_IDS ? dev_off[id] : P_NONE;
  if (off != P_NONE) dev_off[id] = P_NONE;
  const uint32_t recorded = __ballot_sync(KVG_FULL, off != P_NONE);
  if (lane == 0 && recorded) atomicAdd(&info->n_entries, (uint32_t)__popc(recorded));
  const bool ok = V != P_NONE && off != P_NONE && off > V && off < E;
  if (id < K1_IDS && nv_index) nv_index[id] = ok ? off - V : P_NONE;
  for (uint32_t todo = __ballot_sync(KVG_FULL, ok); todo; todo &= todo - 1) {
    const uint32_t slot = __shfl_sync(KVG_FULL, off, (uint32_t)__ffs(todo) - 1) - V;
    sanitise_line_warp(text, len, V + slot + 5, pool + slot, lane);  // first byte after "\t" + 4 hex
  }
}

}  // namespace kvg
