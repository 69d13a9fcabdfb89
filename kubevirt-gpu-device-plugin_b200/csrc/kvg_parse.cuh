// kvg_parse.cuh — pci.ids on the GPU, shared pieces: getDeviceName / locateVendor of the reference
// (pkg/device_plugin/device_plugin.go:371-438) turned into a build-once table.
//
//   (K1 lives in kvg_parse_k1.cuh: scan -> resolve + finalize -> names, self-cleaning)
//   SWAR newline masks, lower-hex field parse
//   the name transform of :404-414 (serial exact routine + warp-cooperative fast path)
//   k_section_lines / k_lookup_general / k_sanitise_matches   exact prefix semantics of :388-402 for
//                                                             arbitrary key bytes
#pragma once
#include "kvg_common.cuh"

namespace kvg {

constexpr uint32_t P_TILE = 8192;             // padding granule of a text image (kvg_text_pad)
constexpr uint32_t P_HALO = 16;               // readable bytes behind the padded image (TMA halo)
constexpr uint32_t P_NONE = 0xffffffffu;
constexpr uint32_t SCAN_TOKEN_MAX = 65536;  // bufio.MaxScanTokenSize

// per-image facts; v_off / n_lines are accumulated by the scan kernel, n_entries by k_pciids_names,
// the rest by the finalize CTAs
struct PciIdsInfo {
  uint32_t v_off;     // offset of the first line with prefix "10de" (locateVendor :424-431)
  uint32_t sec_end;   // first header-type line after it / EOF / scanner failure point
  uint32_t n_entries; // distinct device ids recorded under a 10de header (image 0 only)
  uint32_t n_lines;
  uint32_t limit;     // start of the first line bufio.Scanner would reject (>= 64 KiB), or len
  uint32_t overflow;  // unused (the table cannot overflow: capacity == key space)
  uint32_t pad[2];
};

// 0x80 in every byte of w that equals '\n' (exact, no cross-byte carries)
__device__ __forceinline__ uint32_t nl_flags(uint32_t w) {
  uint32_t x = w ^ 0x0A0A0A0Au;
  uint32_t t = (x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;
  return ~(t | x | 0x7F7F7F7Fu);
}
// gather the four 0x80 flags into a 4-bit mask (bit i = byte i)
__device__ __forceinline__ uint32_t nl_nibble(uint32_t w) { return (nl_flags(w) * 0x00204081u) >> 28; }
__device__ __forceinline__ uint32_t nl_mask16(const uint4& v) {
  return nl_nibble(v.x) | (nl_nibble(v.y) << 4) | (nl_nibble(v.z) << 8) | (nl_nibble(v.w) << 12);
}

// lower-case hex digit value, or 16 for anything else (upper-case is NOT hex here: the keys the
// reference builds come from sysfs "0x%04x" and the match is a byte compare, :388/:400)
__device__ __forceinline__ uint32_t hexval(uint32_t c) {
  uint32_t d = c - '0';
  uint32_t a = c - 'a';
  return d <= 9 ? d : (a <= 5 ? a + 10 : 16);
}
// parse 4 bytes at p -> (valid<<16)|value
__device__ __forceinline__ uint32_t parse_hex4(const uint8_t* p) {
  uint32_t h0 = hexval(p[0]), h1 = hexval(p[1]), h2 = hexval(p[2]), h3 = hexval(p[3]);
  uint32_t bad = (h0 | h1 | h2 | h3) & 16;
  return bad ? 0u : (0x10000u | (h0 << 12) | (h1 << 8) | (h2 << 4) | h3);
}

// ------------------------------------------------------------------------------------------------
// The name transform (:404-414) as one left-to-right pass.
//   TrimSpace (unicode.IsSpace, with Go's ASCII fast path) -> ToUpper (simple mapping: only U+0131
//   and U+017F land in ASCII) -> '/'->'_' -> '.'->'_' -> RE2 \s+ ([\t\n\f\r ]) -> '_' ->
//   delete [^a-zA-Z0-9_.]+.   Output alphabet is [A-Z0-9_].
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool d_ascii_space(uint32_t c) {
  return c == ' ' || (c >= 9 && c <= 13);
}
__device__ __forceinline__ bool d_re2_space(uint32_t c) {
  return c == ' ' || c == '\t' || c == '\n' || c == '\f' || c == '\r';
}
__device__ uint32_t d_decode_rune(const uint8_t* p, uint32_t n, uint32_t* width) {
  *width = 1;
  if (n == 0) {
    *width = 0;
    return 0xFFFD;
  }
  uint32_t b0 = p[0];
  if (b0 < 0x80) return b0;
  if (b0 < 0xC2 || b0 > 0xF4) return 0xFFFD;
  if (b0 < 0xE0) {
    if (n < 2 || (p[1] & 0xC0) != 0x80) return 0xFFFD;
    *width = 2;
    return ((b0 & 0x1F) << 6) | (p[1] & 0x3F);
  }
  if (b0 < 0xF0) {
    if (n < 3) return 0xFFFD;
    uint32_t lo = b0 == 0xE0 ? 0xA0 : 0x80, hi = b0 == 0xED ? 0x9F : 0xBF;
    if (p[1] < lo || p[1] > hi || (p[2] & 0xC0) != 0x80) return 0xFFFD;
    *width = 3;
    return ((b0 & 0x0F) << 12) | ((p[1] & 0x3F) << 6) | (p[2] & 0x3F);
  }
  if (n < 4) return 0xFFFD;
  uint32_t lo = b0 == 0xF0 ? 0x90 : 0x80, hi = b0 == 0xF4 ? 0x8F : 0xBF;
  if (p[1] < lo || p[1] > hi || (p[2] & 0xC0) != 0x80 || (p[3] & 0xC0) != 0x80) return 0xFFFD;
  *width = 4;
  return ((b0 & 0x07) << 18) | ((p[1] & 0x3F) << 12) | ((p[2] & 0x3F) << 6) | (p[3] & 0x3F);
}
__device__ uint32_t d_decode_last_rune(const uint8_t* p, uint32_t n, uint32_t* width) {
  *width = 1;
  if (n == 0) {
    *width = 0;
    return 0xFFFD;
  }
  int end = (int)n, start = end - 1;
  if (p[start] < 0x80) return p[start];
  int lim = end - 4 < 0 ? 0 : end - 4;
  for (start--; start >= lim; start--)
    if ((p[start] & 0xC0) != 0x80) break;
  if (start < 0) start = 0;
  uint32_t w;
  uint32_t r = d_decode_rune(p + start, (uint32_t)(end - start), &w);
  if (start + (int)w != end) return 0xFFFD;
  *width = w;
  return r;
}
__device__ __forceinline__ bool d_is_space_rune(uint32_t r) {
  if (r < 0x80) return d_ascii_space(r);
  return r == 0x85 || r == 0xA0 || r == 0x1680 || (r >= 0x2000 && r <= 0x200A) || r == 0x2028 ||
         r == 0x2029 || r == 0x202F || r == 0x205F || r == 0x3000;
}
__device__ void d_trim_space(const uint8_t* s, uint32_t n, uint32_t* pa, uint32_t* pb) {
  uint32_t a = 0, b = n;
  int uni = 0;
  for (; a < n; a++) {
    uint32_t c = s[a];
    if (c >= 0x80) {
      uni = 1;
      break;
    }
    if (!d_ascii_space(c)) break;
  }
  if (!uni) {
    for (; b > a; b--) {
      uint32_t c = s[b - 1];
      if (c >= 0x80) {
        uni = 2;
        break;
      }
      if (!d_ascii_space(c)) break;
    }
  }
  if (uni == 1) {
    while (a < n) {
      uint32_t w;
      uint32_t r = d_decode_rune(s + a, n - a, &w);
      if (!d_is_space_rune(r)) break;
      a += w;
    }
    b = n;
  }
  if (uni) {
    while (b > a) {
      uint32_t w;
      uint32_t r = d_decode_last_rune(s + a, b - a, &w);
      if (!d_is_space_rune(r)) break;
      b -= w;
    }
  }
  *pa = a;
  *pb = b;
}
// returns the output length; writes at most `cap` bytes (the caller sizes cap >= n)
__device__ uint32_t d_sanitise_name(const uint8_t* s, uint32_t n, uint8_t* out, uint32_t cap) {
  uint32_t a, b;
  d_trim_space(s, n, &a, &b);
  uint32_t o = 0;
  bool prev_ws = false;
  for (uint32_t i = a; i < b;) {
    uint32_t c = s[i];
    uint32_t e = 0;
    if (c < 0x80) {
      i++;
      if (d_re2_space(c)) {
        if (!prev_ws) e = '_';
        prev_ws = true;
      } else {
        prev_ws = false;
        if (c >= 'a' && c <= 'z')
          e = c - 32;
        else if ((c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_')
          e = c;
        else if (c == '/' || c == '.')
          e = '_';
      }
    } else {
      prev_ws = false;
      if (c == 0xC4 && i + 1 < b && s[i + 1] == 0xB1) {
        e = 'I';
        i += 2;
      } else if (c == 0xC5 && i + 1 < b && s[i + 1] == 0xBF) {
        e = 'S';
        i += 2;
      } else {
        i++;
      }
    }
    if (e) {
      if (o < cap) out[o] = (uint8_t)e;
      o++;
    }
  }
  return o;
}


// K2 for one line, executed by a full warp: lanes classify 32 characters at a time.  ASCII-only lines
// (every line of the shipped file's NVIDIA block) take the lane-parallel path; a line with any byte
// >= 0x80 falls back to the exact serial routine (Unicode TrimSpace / ToUpper rules).
//   s0   offset of the first byte after "\t" + key;   out   u16 length, then the sanitised bytes
__device__ __forceinline__ void sanitise_line_warp(const uint8_t* __restrict__ text, uint32_t len, uint32_t s0,
                                                   uint8_t* __restrict__ out, uint32_t lane) {
  // line end and ASCII test
  uint32_t n = 0;
  bool ascii = true;
  for (uint32_t c0 = 0;; c0 += 32) {
    uint32_t pos = s0 + c0 + lane;
    uint32_t c = pos < len ? text[pos] : '\n';
    uint32_t nl = __ballot_sync(KVG_FULL, c == '\n');
    uint32_t hi = __ballot_sync(KVG_FULL, c >= 0x80);
    if (nl) {
      uint32_t k = (uint32_t)__ffs(nl) - 1;
      n = c0 + k;
      if (hi & ((1u << k) - 1)) ascii = false;
      break;
    }
    if (hi) ascii = false;
  }
  if (!ascii) {
    if (lane == 0) {
      uint32_t m = d_sanitise_name(text + s0, n, out + 2, n);
      out[0] = (uint8_t)(m & 0xff);
      out[1] = (uint8_t)(m >> 8);
    }
    return;
  }
  // trim: first / last byte that is not ASCII white space (TrimSpace; includes \v)
  uint32_t first = n, last = 0;
  for (uint32_t c0 = 0; c0 < n; c0 += 32) {
    uint32_t i = c0 + lane;
    bool ns = i < n && !d_ascii_space(text[s0 + i]);
    uint32_t b = __ballot_sync(KVG_FULL, ns);
    if (b) {
      if (first == n) first = c0 + (uint32_t)__ffs(b) - 1;
      last = c0 + 32 - (uint32_t)__clz(b);  // one past the last non-space
    }
  }
  uint32_t o = 0;
  if (first < last) {
    for (uint32_t c0 = first; c0 < last; c0 += 32) {
      uint32_t i = c0 + lane;
      uint32_t e = 0;
      if (i < last) {
        uint32_t c = text[s0 + i];
        if (d_re2_space(c)) {
          if (!(i > first && d_re2_space(text[s0 + i - 1]))) e = '_';  // one '_' per run
        } else if (c >= 'a' && c <= 'z') {
          e = c - 32;
        } else if ((c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_') {
          e = c;
        } else if (c == '/' || c == '.') {
          e = '_';
        }
      }
      uint32_t b = __ballot_sync(KVG_FULL, e != 0);
      if (e) out[2 + o + __popc(b & lanemask_lt())] = (uint8_t)e;
      o += __popc(b);
    }
  }
  if (lane == 0) {
    out[0] = (uint8_t)(o & 0xff);
    out[1] = (uint8_t)(o >> 8);
  }
}

// every line start of the NVIDIA section that begins with '\t' (candidates of the prefix match),
// collected once per table load; order is irrelevant (matches are reduced with atomicMin)
__global__ void __launch_bounds__(KVG_BLOCK) k_section_lines(const uint8_t* __restrict__ text,
                                                             const PciIdsInfo* __restrict__ info,
                                                             uint32_t* __restrict__ lines,
                                                             uint32_t* __restrict__ n_lines, uint32_t cap) {
  pdl_enter();
  const uint32_t V = info->v_off, E = info->sec_end;
  if (V == P_NONE) return;
  for (uint32_t b = V + 1 + blockIdx.x * blockDim.x + threadIdx.x; b < E; b += gridDim.x * blockDim.x) {
    if (text[b - 1] == '\n' && text[b] == '\t') {
      uint32_t k = atomicAdd(n_lines, 1u);
      if (k < cap) lines[k] = b;
    }
  }
}

// Exact :388-402 for arbitrary keys.  grid.y = key index; threads sweep the section's '\t' lines
// (E already excludes everything past the first non-'\t' non-'#' line; '#' lines are not listed).
//   match = HasPrefix(line, "\t"+key) on the token bufio.ScanLines returns (one trailing '\r'
//   dropped); the first matching line wins (atomicMin on its offset).
__global__ void __launch_bounds__(KVG_BLOCK) k_lookup_general(const uint8_t* __restrict__ text,
                                                              uint32_t len,
                                                              const uint32_t* __restrict__ lines,
                                                              const uint32_t* __restrict__ n_lines_ptr,
                                                              const uint8_t* __restrict__ keys,
                                                              const uint32_t* __restrict__ key_off,
                                                              uint32_t* __restrict__ match_off) {
  pdl_enter();
  const uint32_t n_lines = *n_lines_ptr;
  const uint32_t kidx = blockIdx.y;
  const uint8_t* key = keys + key_off[kidx];
  const uint32_t klen = key_off[kidx + 1] - key_off[kidx];
  for (uint32_t li = blockIdx.x * blockDim.x + threadIdx.x; li < n_lines; li += gridDim.x * blockDim.x) {
    const uint32_t b = lines[li];
    bool ok = true;
    for (uint32_t k = 0; k < klen && ok; k++) {
      uint32_t pos = b + 1 + k;
      if (pos >= len) {
        ok = false;
        break;
      }
      uint8_t c = text[pos];
      if (c == '\n' || c != key[k]) ok = false;
      // a '\r' that is the last byte of the line is not part of the token
      else if (c == '\r' && (pos + 1 >= len || text[pos + 1] == '\n'))
        ok = false;
    }
    if (ok) atomicMin(&match_off[kidx], b);
  }
}
// one thread per key: sanitise the remainder of the matched line into out[k*cap ...], or, with out_off, into
// out[out_off[k] .. out_off[k+1]); out_len[k] is the name's full length either way
__global__ void k_sanitise_matches(const uint8_t* __restrict__ text, uint32_t len,
                                   const uint32_t* __restrict__ key_off,
                                   const uint32_t* __restrict__ match_off, uint32_t n_keys,
                                   uint8_t* __restrict__ out, uint32_t cap,
                                   uint32_t* __restrict__ out_len, const uint64_t* __restrict__ out_off) {
  pdl_enter();
  uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_keys) return;
  uint32_t b = match_off[k];
  if (b == P_NONE) {
    out_len[k] = 0;
    return;
  }
  uint32_t s = b + 1 + (key_off[k + 1] - key_off[k]);
  uint32_t e = s;
  while (e < len && text[e] != '\n') e++;
  if (e > s && text[e - 1] == '\r') e--;  // ScanLines dropCR (TrimSpace would drop it anyway)
  const size_t o = out_off ? out_off[k] : (size_t)k * cap;
  const uint32_t c = out_off ? (uint32_t)(out_off[k + 1] - out_off[k]) : cap;
  out_len[k] = d_sanitise_name(text + s, e - s, out + o, c);
}

}  // namespace kvg
