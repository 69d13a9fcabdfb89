// alloc_raw_emu.cpp — kvg_pci_allocate_raw's kernels (csrc/kvg_alloc_raw.cuh) compiled for the CPU from their real
// source on top of warp_emu.h, in the library's order and launch shapes: k_araw_members, k_araw_keys, then
// k_pci_allocate_check on what they wrote, the key kernel sized and its arguments built by araw_keys_size /
// araw_keys_args (kvg_alloc_raw.cuh) and the request table by allocate_check_reqs (kvg_scan.cuh), as the library
// builds them; and unicode.ToLower of the device (case_lower) over any runes.
#define KVG_HOST_EMU 1
#include <algorithm>
#include <vector>
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_scan.cuh"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_alloc_raw.cuh"
using namespace kvg;

extern "C" {

// reqs: n_reqs x {n_members, n_ids}; the member, ID and EGM tables as kvg_alloc_raw has them (bytes readable one past
// their end).  first_bad_out [n_reqs]; code_out [n_members] (ARAW_*); kept_out [n_egm]; take_out [n_reqs * n_egm];
// verdict_out {miss, range} as the key kernel leaves them (~0 = none, and when n_egm = 0).
int emu_pci_allocate_raw(const uint32_t* reqs, uint32_t n_reqs, const uint32_t* moff, const uint16_t* mst,
                         const uint8_t* mb, uint32_t n_mem, const uint32_t* ioff, const uint8_t* ib, uint32_t n_ids,
                         const uint32_t* eoff, const uint16_t* est, const uint8_t* eb, uint32_t n_egm,
                         uint32_t* first_bad_out, uint8_t* code_out, uint8_t* kept_out, uint8_t* take_out,
                         uint64_t* verdict_out) {
  std::vector<uint4> recs(n_mem + 1);
  std::vector<uint32_t> want(n_mem + 1), ids(n_ids + 1);
  memset(code_out, ARAW_PASS, n_mem);
  verdict_out[0] = verdict_out[1] = ~0ull;
  uint32_t seq = 0;
  if (n_mem)
    emu_launch(k_araw_members, dim3((n_mem + ARAW_THREADS - 1) / ARAW_THREADS), ARAW_THREADS, moff, mst, mb, n_mem,
               recs.data(), want.data(), code_out);
  const ArawKeysSize ks = araw_keys_size(n_egm, n_egm ? eoff[(size_t)n_egm * KVG_AEGM_FIELDS] : 0);
  const size_t n_list = ks.n_list;
  std::vector<uint32_t> list_off(n_egm + 1), list(n_list + 1), tok_entry(n_list + 1), rank(n_list + 1, 0xdeadbeefu);
  std::vector<uint2> tok(n_list + 1);
  std::vector<uint64_t> table(ks.slots, 0x5a5a5a5a5a5a5a5aull);  // the kernel clears its table
  if (n_egm)
    emu_launch(k_araw_keys, dim3(1), ARAW_KEY_THREADS,
               araw_keys_args(ks, eoff, est, eb, n_egm, ioff, ib, n_ids, list_off.data(), list.data(), tok.data(),
                              tok_entry.data(), rank.data(), table.data(), ids.data(), kept_out,
                              (unsigned long long*)verdict_out, n_reqs, &seq, 7));
  if (n_reqs) {
    std::vector<uint4> req(n_reqs);
    allocate_check_reqs((const kvg_alloc_req*)reqs, n_reqs, req.data());
    uint32_t done = 0;
    emu_launch(k_pci_allocate_check, dim3(std::min(n_reqs, ALLOC_CHECK_MAX_GRID)), GROUP_CHECK_THREADS,
               (const uint4*)req.data(), (const uint4*)recs.data(), (const uint32_t*)want.data(),
               (const uint32_t*)ids.data(), (const uint32_t*)list_off.data(), (const uint32_t*)list.data(), n_reqs,
               n_egm, n_egm ? (uint32_t)KVG_ALLOC_MAX_EGM_GPUS : 0u, &done, first_bad_out, take_out, &seq, 7u);
  }
  return (n_reqs || n_egm) && seq != 7 ? -2 : 0;
}

// out[k] = case_lower(runes[k])
void emu_case_lower(const uint32_t* runes, uint32_t* out, uint64_t n) {
  for (uint64_t k = 0; k < n; k++) out[k] = case_lower(runes[k]);
}

}  // extern "C"
