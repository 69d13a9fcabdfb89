// shard_emu.cpp — the exchange step of the sharded scan (csrc/kvg_shard.cuh: k_shard_send,
// k_shard_gather) compiled for the CPU from its real source on top of warp_emu.h.  P ranks are
// emulated in ONE process: every rank has its own window + control block, `peers` points at all of them, and the
// kernels of a step run rank after rank (all sends, then all gathers — the order the flags allow).
#define KVG_HOST_EMU 1
#include "warp_emu.h"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_scan.cuh"
#include "../../kubevirt-gpu-device-plugin_b200/csrc/kvg_shard.cuh"
using namespace kvg;

template <int U>
static int run(const uint4* const* lists, const uint32_t* n, uint32_t P, uint32_t steps, uint32_t cap, int local_mode,
               uint4* owned0_out, uint4* owned1_out, uint32_t* n_own_out, uint32_t* max_out) {
  // local_mode: NCCL path — lists[r] is the SAME gathered list on every rank, one source region
  const uint32_t n_src = local_mode ? 1 : P;
  const size_t region_cap = local_mode ? (size_t)P * cap : cap;
  const size_t win_units = 2 * 2 * (size_t)n_src * region_cap * U;
  std::vector<std::vector<uint4>> win(P, std::vector<uint4>(win_units, uint4{0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu}));
  std::vector<ShardCtrl> ctrl(P);
  memset(ctrl.data(), 0, sizeof(ShardCtrl) * P);
  ShardPeers peers;
  memset(&peers, 0, sizeof peers);
  for (uint32_t q = 0; q < P; q++) {
    peers.win[q] = win[q].data();
    peers.ctrl[q] = &ctrl[q];
  }
  uint32_t err = 0;
  std::vector<std::vector<uint64_t>> state(P);  // chained-scan words: epoch-tagged, reused by every step uncleared
  for (uint32_t step = 1; step <= steps; step++) {
    std::vector<std::vector<uint32_t>> cnt(P);
    for (uint32_t r = 0; r < P; r++) {
      const size_t T = (n[r] + C_TILE - 1) / C_TILE + 1;
      cnt[r].assign(64, 0);
      uint32_t nn = n[r];
      ShardArgs A;
      A.list = lists[r];
      A.n_ptr = &nn;
      if (state[r].empty()) state[r].assign(2 * (size_t)P * T, 0);
      A.state = state[r].data();
      A.totals = cnt[r].data();
      A.ticket = cnt[r].data() + 32;
      A.T = (uint32_t)T;
      A.P = P;
      A.Pm = shard_magic(P);
      A.me = r;
      A.only = local_mode ? r : SH_ALL;
      A.n_src = n_src;
      A.src = local_mode ? 0 : r;
      A.region_cap = region_cap;
      A.parity = step & 1;
      A.step = step;
      emu_launch(k_shard_send<U>, dim3((unsigned)T), KVG_BLOCK, A, peers, (const ShardCtrl*)&ctrl[r], &err, 100u + step);
    }
    for (int pass = 0; pass < 2; pass++)  // every rank publishes, then every rank gathers
    for (uint32_t r = 0; r < P; r++) {
      uint32_t nn = n[r];
      const size_t T = (n[r] + C_TILE - 1) / C_TILE + 1;
      ShardArgs A;
      A.list = lists[r];
      A.n_ptr = &nn;
      A.state = state[r].data();
      A.totals = cnt[r].data();
      A.ticket = cnt[r].data() + 32;
      A.T = (uint32_t)T;
      A.P = P;
      A.Pm = shard_magic(P);
      A.me = r;
      A.only = local_mode ? r : SH_ALL;
      A.n_src = n_src;
      A.src = local_mode ? 0 : r;
      A.region_cap = region_cap;
      A.parity = step & 1;
      A.step = step;
      const size_t owned_cap = (size_t)P * cap;
      GatherArgs G;
      G.window = win[r].data();
      G.owned[0] = owned0_out + (size_t)r * owned_cap * U;
      G.owned[1] = owned1_out + (size_t)r * owned_cap * U;
      G.n_own = n_own_out + 2 * r;
      max_out[2 * r] = max_out[2 * r + 1] = 0;
      G.max_key = max_out + 2 * r;
      if (pass == 0) {
        emu_launch(k_shard_gather<U>, dim3(1, 1), KVG_BLOCK, A, G, peers, (const ShardCtrl*)&ctrl[r], &err, 1u);  // publish
        continue;
      }
      emu_launch(k_shard_gather<U>, dim3(3, 2), KVG_BLOCK, A, G, peers, (const ShardCtrl*)&ctrl[r], &err, 2u);
      if (cnt[r][33] != 0) return -4;
    }
  }
  return err ? -5 : 0;
}

// k_classify_send: raw PCI records of P shards -> each rank's dense survivor list AND the owners' windows in one
// kernel per rank, then the gathers.  CW4 follows the host's choice for P.
template <int CW4>
static int run_fused(const uint4* const* recs, const uint32_t* n, uint32_t P, uint32_t steps, uint32_t cap, const uint32_t* nv_index,
                     uint4* surv_out, uint32_t* n_surv_out, uint4* owned0_out, uint4* owned1_out, uint32_t* n_own_out,
                     uint32_t* max_out) {
  constexpr int TH = 128, ROWS = 8, U = 1;
  const size_t win_units = 2 * 2 * (size_t)P * cap * U;
  std::vector<std::vector<uint4>> win(P, std::vector<uint4>(win_units, uint4{0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu, 0xdeadbeefu}));
  std::vector<ShardCtrl> ctrl(P);
  memset(ctrl.data(), 0, sizeof(ShardCtrl) * P);
  ShardPeers peers;
  memset(&peers, 0, sizeof peers);
  for (uint32_t q = 0; q < P; q++) {
    peers.win[q] = win[q].data();
    peers.ctrl[q] = &ctrl[q];
  }
  uint32_t err = 0;
  std::vector<std::vector<uint32_t>> words(P);  // published tile counts: epoch-tagged, reused uncleared
  std::vector<std::vector<uint32_t>> cnt(P, std::vector<uint32_t>(64, 0));
  std::vector<ScanCtrl> sc(P);
  auto args = [&](uint32_t r, uint32_t step) {
    ShardArgs A;
    A.list = nullptr;
    A.n_ptr = nullptr;
    A.state = nullptr;
    A.totals = cnt[r].data();
    A.ticket = cnt[r].data() + 32;
    A.T = 0;
    A.P = P;
    A.Pm = shard_magic(P);
    A.me = r;
    A.only = SH_ALL;
    A.n_src = P;
    A.src = r;
    A.region_cap = cap;
    A.parity = step & 1;
    A.step = step;
    return A;
  };
  for (uint32_t step = 1; step <= steps; step++) {
    for (uint32_t r = 0; r < P; r++) {
      const size_t tiles = std::max<size_t>(1, (n[r] + (size_t)TH * ROWS - 1) / ((size_t)TH * ROWS));
      if (words[r].empty()) words[r].assign(tiles * 4 * CW4, 0);
      memset(&sc[r], 0, sizeof(ScanCtrl));
      PciClassifyOp op;
      op.recs = recs[r];
      op.n = n[r];
      op.out = surv_out + (size_t)r * cap;
      op.ctrl = &sc[r];
      op.nv_index = nv_index;
      emu_launch(k_classify_send<PciClassifyOp, TH, ROWS, CW4>, dim3((unsigned)tiles), TH, op, args(r, step), peers,
                 (const ShardCtrl*)&ctrl[r], &err, words[r].data(), 40u + step);
      n_surv_out[r] = sc[r].n_surv;
    }
    for (int pass = 0; pass < 2; pass++)
    for (uint32_t r = 0; r < P; r++) {
      const size_t owned_cap = (size_t)P * cap;
      GatherArgs G;
      G.window = win[r].data();
      G.owned[0] = owned0_out + (size_t)r * owned_cap * U;
      G.owned[1] = owned1_out + (size_t)r * owned_cap * U;
      G.n_own = n_own_out + 2 * r;
      max_out[2 * r] = max_out[2 * r + 1] = 0;
      G.max_key = max_out + 2 * r;
      if (pass == 0) {
        emu_launch(k_shard_gather<U>, dim3(1, 1), KVG_BLOCK, args(r, step), G, peers, (const ShardCtrl*)&ctrl[r], &err, 1u);
        continue;
      }
      emu_launch(k_shard_gather<U>, dim3(3, 2), KVG_BLOCK, args(r, step), G, peers, (const ShardCtrl*)&ctrl[r], &err, 2u);
      if (cnt[r][33] != 0) return -4;
    }
  }
  return err ? -5 : 0;
}

extern "C" {
// recs: P pointers to raw PCI records (16 bytes each), n[P].  Outputs per rank r: surv_out + r * cap (dense
// survivor list, n_surv_out[r] long), owned lists as in emu_exchange.
int emu_classify_exchange(const uint4* const* recs, const uint32_t* n, uint32_t P, uint32_t steps, uint32_t cap,
                          const uint32_t* nv_index, uint4* surv_out, uint32_t* n_surv_out, uint4* owned0_out, uint4* owned1_out,
                          uint32_t* n_own_out, uint32_t* max_out) {
  const int C = 1 + 2 * (int)P;
#define KVG_RUN(W) run_fused<W>(recs, n, P, steps, cap, nv_index, surv_out, n_surv_out, owned0_out, owned1_out, n_own_out, max_out)
  return C <= 8 ? KVG_RUN(2) : C <= 16 ? KVG_RUN(4) : C <= 20 ? KVG_RUN(5) : KVG_RUN(9);
#undef KVG_RUN
}
// lists: P pointers to dense record lists (units x 16 bytes per record), n[P] their lengths.  Outputs per rank
// r at owned{0,1}_out + r * P * cap * units: the owned lists; n_own_out[2r + o], max_out[2r + o].
int emu_exchange(int units, const uint4* const* lists, const uint32_t* n, uint32_t P, uint32_t steps, uint32_t cap,
                 int local_mode, uint4* owned0_out, uint4* owned1_out, uint32_t* n_own_out, uint32_t* max_out) {
  if (units == 1) return run<1>(lists, n, P, steps, cap, local_mode, owned0_out, owned1_out, n_own_out, max_out);
  return run<2>(lists, n, P, steps, cap, local_mode, owned0_out, owned1_out, n_own_out, max_out);
}
}
