// alloc_resp_emu.cpp — kvg_pci_allocate_response's kernels (csrc/kvg_alloc_resp.cuh, after those of
// kvg_alloc_raw.cuh) compiled for the CPU from their real source on top of warp_emu.h, in the library's order and
// launch shapes: k_araw_members, k_aresp_members, k_araw_keys, k_pci_allocate_check, k_aresp_requests, with the
// request places built by aresp_plan and the key kernel's work by araw_keys_size / araw_keys_args, as the library
// builds them.  The host keeps the library's zeroed and ~0 initial words.
#define KVG_HOST_EMU 1
#include <algorithm>
#include <vector>
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_scan.cuh"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_alloc_resp.cuh"
using namespace kvg;

extern "C" {

// The call's kernels on kvg_alloc_raw / kvg_alloc_resp_in (bytes readable one past their end).  Outputs, sized by
// the caller: first_bad/error/error_at/n_specs/env_len/env_key [n_reqs], spec_first [n_reqs], span [2 * slots],
// pool [bytes], env [addresses + n_members], code [n_members], verdicts {raw miss, raw range, group, EGM order}.
// sizes_out = {slots, bytes} (call with span = NULL to size only).  Returns -1 when aresp_plan refuses, -2 when the
// sequence word was not written.
int emu_pci_allocate_response(const kvg_alloc_req* reqs, uint32_t n_reqs, const kvg_alloc_raw* raw,
                              const kvg_alloc_resp_in* in, uint64_t* sizes_out, uint32_t* first_bad, uint8_t* error,
                              uint32_t* error_at, uint32_t* spec_first, uint32_t* n_specs, uint32_t* span, uint8_t* pool,
                              uint32_t* env_len, uint8_t* env_key, uint8_t* env, uint8_t* code, uint64_t* verdict) {
  const uint32_t n_mem = (uint32_t)raw->n_members, n_ids = (uint32_t)raw->n_ids, n_egm = raw->n_egm;
  uint32_t n_vis = 0;
  for (uint32_t r = 0; r < n_reqs; r++) n_vis += in->n_visited[r];
  std::vector<ArespReq> rq(n_reqs + 1);
  std::vector<uint4> visit(n_vis + 1);
  ArespTotals tot;
  if (!aresp_plan(reqs, n_reqs, raw, in, rq.data(), visit.data(), &tot)) return -1;
  sizes_out[0] = tot.slots;
  sizes_out[1] = tot.bytes;
  if (!span) return 0;
  for (uint32_t r = 0; r < n_reqs; r++) spec_first[r] = rq[r].s0;
  std::vector<uint4> recs(n_mem + 1);
  std::vector<uint32_t> want(n_mem + 1), ids(n_ids + 1), found(n_vis + 1, 0), pick(n_mem + 1, 0xdeadbeefu),
      cslot(tot.cand + 1);
  std::vector<unsigned long long> ev(n_reqs + 1, ~0ull);
  std::vector<uint64_t> ktab(tot.words + 1, 0x5a5a5a5a5a5a5a5aull);  // the request kernel clears its table
  std::vector<uint8_t> kept(n_egm + 1), take((size_t)n_reqs * n_egm + 1);
  std::vector<uint4> req(n_reqs + 1);
  allocate_check_reqs(reqs, n_reqs, req.data());
  memset(code, ARAW_PASS, n_mem);
  for (int k = 0; k < 4; k++) verdict[k] = ~0ull;
  uint32_t seq = 0, dummy = 0, done[2] = {0, 0};
  const ArespArgs a = {rq.data(), visit.data(), n_reqs, n_vis, n_mem, in->iommufd, raw->member_off, raw->member_bytes,
                       raw->id_off, raw->id_bytes, in->addr_off, in->addr_bytes, in->vfio_first, in->vfio_off,
                       in->vfio_bytes, in->vfio_dir, in->vfio_state, raw->egm_off, raw->egm_bytes, n_egm, recs.data(),
                       first_bad, code, take.data(), found.data(), ev.data(), pick.data(), cslot.data(), ktab.data(),
                       (unsigned long long*)verdict + 2, env, error, error_at, n_specs, span, pool, env_len, env_key,
                       &done[1], &seq, 7u};
  if (n_mem)
    emu_launch(k_araw_members, dim3((n_mem + ARAW_THREADS - 1) / ARAW_THREADS), ARAW_THREADS, raw->member_off,
               raw->member_state, raw->member_bytes, n_mem, recs.data(), want.data(), code);
  const uint32_t n_thr = std::max(n_mem, n_egm > 1 ? n_egm - 1 : 0u);
  if (n_thr) emu_launch(k_aresp_members, dim3((n_thr + ARESP_THREADS - 1) / ARESP_THREADS), ARESP_THREADS, a);
  const ArawKeysSize ks = araw_keys_size(n_egm, n_egm ? raw->egm_off[(size_t)n_egm * KVG_AEGM_FIELDS] : 0);
  const size_t n_list = ks.n_list;
  std::vector<uint32_t> list_off(n_egm + 1), list(n_list + 1), tok_entry(n_list + 1), rank(n_list + 1, 0xdeadbeefu);
  std::vector<uint2> tok(n_list + 1);
  std::vector<uint64_t> table(ks.slots, 0x5a5a5a5a5a5a5a5aull);
  if (n_egm)
    emu_launch(k_araw_keys, dim3(1), ARAW_KEY_THREADS,
               araw_keys_args(ks, raw->egm_off, raw->egm_state, raw->egm_bytes, n_egm, raw->id_off, raw->id_bytes,
                              n_ids, list_off.data(), list.data(), tok.data(), tok_entry.data(), rank.data(),
                              table.data(), ids.data(), kept.data(), (unsigned long long*)verdict, n_reqs, &seq, 7));
  if (n_reqs) {
    emu_launch(k_pci_allocate_check, dim3(std::min(n_reqs, ALLOC_CHECK_MAX_GRID)), GROUP_CHECK_THREADS,
               (const uint4*)req.data(), (const uint4*)recs.data(), (const uint32_t*)want.data(),
               (const uint32_t*)ids.data(), (const uint32_t*)list_off.data(), (const uint32_t*)list.data(), n_reqs,
               n_egm, n_egm ? (uint32_t)KVG_ALLOC_MAX_EGM_GPUS : 0u, &done[0], first_bad, take.data(), &dummy, 7u);
    emu_launch(k_aresp_requests, dim3(std::min(n_reqs, ARESP_MAX_GRID)), ARESP_REQ_THREADS, a);
  }
  return (n_reqs || n_egm) && seq != 7 ? -2 : 0;
}

}  // extern "C"
