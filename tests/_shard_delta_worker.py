"""Worker for the sharded re-scan delta test (kvg_dev_scan_pci_shard_fetch_delta): rank r scans its shard of a
sequence of snapshots on GPU r (hot-adds, hot-removes, re-binds, regroups, device-id and NUMA changes at about 0.1 %
of the records per step; the record count changes, so shard boundaries move) and checks every step:
  - the result equals a plain kvg_dev_scan_pci_shard_fetch of the same scan;
  - its delta is exact: the local changes against delta_ref.expect_pci_delta of its previous and new local survivors,
    the owned key lists against the whole snapshot's delta restricted to the keys it owns;
  - the ranks' deltas merged by merge_pci_shard_deltas equal Context.scan_pci_delta of the whole snapshot on a
    second context, and the parts patched by apply_pci_shard_delta dump like the oracle;
  - plain sharded fetches, kvg_scan_pci_delta and kvg_scan_pci in between leave its previous result alone, and it
    leaves theirs alone;
  - the first call and a reset report everything as added; a refusal keeps the previous result, and a refusal on
    one rank makes ShardedScan.fetch_delta reset every rank;
  - the call costs exactly two launches beyond the plain fetch.

Arguments: n_per_rank mode (p2p | nccl | one-device: every rank on GPU 0, gloo, peer windows; tests/_one_device.py)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch
import torch.distributed as dist

import _one_device
import delta_ref
import kvgpu
import util
from oracle import oracle as O
from test_gpu_delta import KINDS, snapshot, step


def main():
    n_per_rank, mode = int(sys.argv[1]), sys.argv[2]
    one_device = mode == "one-device"
    if one_device:                     # every rank on GPU 0 over gloo: peer windows only
        rank, world, local_rank = _one_device.init()
    else:
        rank, world, local_rank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    text = util.pciids_text()
    ids = O.nv_ids(text)
    ctx = kvgpu.Context(local_rank)
    ctx.pciids_load(text)
    whole = kvgpu.Context(local_rank)          # the single-GPU delta of the whole snapshot
    whole.pciids_load(text)

    def bcast(b, src):
        t = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == src:
            t[:len(b)].copy_(torch.frombuffer(bytearray(b), dtype=torch.uint8))
        dist.broadcast(t, src)
        return bytes(t.cpu().numpy().tobytes())

    def allgather(b):
        t = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
        outs = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(outs, t)
        return [bytes(o.cpu().numpy().tobytes()) for o in outs]

    def gather(obj):
        if world == 1:
            return [obj]
        out = [None] * world
        dist.all_gather_object(out, obj)
        return out

    if one_device:
        bcast, allgather = _one_device.broadcast, _one_device.allgather

    n = n_per_rank * world
    cap = n_per_rank + n_per_rank // 50 + 64                 # room for hot-adds and moving boundaries
    sh = kvgpu.ShardedScan(ctx, rank, world, bcast, allgather if mode != "nccl" else None, cap)
    assert sh.mode == "p2p" or not one_device, "rank %d: no peer windows on one device" % rank
    if mode == "p2p" and sh.mode != "p2p" and rank == 0:
        print("note: peer windows unavailable, fell back to NCCL")
    buf = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(n_per_rank + world)

    def scan(recs):
        lo, hi = kvgpu.shard_range(len(recs), rank, world)
        part = np.ascontiguousarray(recs[lo:hi])
        assert hi - lo <= cap
        buf[:part.nbytes].copy_(torch.from_numpy(part.view(np.uint8)))
        torch.cuda.synchronize()
        # the ranks line up before every sharded scan: a rank's exchange waits at most ~10 s for its peers, and the
        # checks between two scans take longer on the ranks that own more keys
        dist.barrier()
        sh.scan_device_shard(buf.data_ptr(), hi - lo)
        return part

    def same_shard_result(a, b):
        assert a.n_records == b.n_records and np.array_equal(a.local, b.local)
        for x, y in ((a.dev, b.dev), (a.grp, b.grp)):
            for f in ("survivors", "dev_keys", "dev_off", "dev_perm", "dev_name_slot", "grp_keys", "grp_off",
                      "grp_perm", "name_pool"):
                u, v = getattr(x, f), getattr(y, f)
                assert (np.array_equal(u, v) if isinstance(u, np.ndarray) else u == v), f

    def owned(surv):
        return surv[surv["device"] % world == rank], surv[surv["iommu_group"] % world == rank]

    def check_rank(got, res, prev_local, prev_all, now_all):
        """This rank's delta: local changes, and the owned share of the whole snapshot's key lists."""
        loc = delta_ref.expect_pci_delta(prev_local, res.local, kvgpu.PCI_CHANGE)
        assert got.n_prev == len(prev_local)
        assert got.changes.tobytes() == loc["changes"].tobytes(), "local changes"
        want = delta_ref.expect_pci_delta(prev_all, now_all, kvgpu.PCI_CHANGE)
        for mine, want_own in zip((res.dev.survivors, res.grp.survivors), owned(now_all)):
            for f in ("addr", "iommu_group", "device", "numa"):
                assert np.array_equal(mine[f], want_own[f]), "owned lists: " + f
        dd = np.unique(now_all["device"])[want["dev_dirty"]]
        gd = np.unique(now_all["iommu_group"])[want["grp_dirty"]]
        assert np.array_equal(res.dev.dev_keys[got.dev_dirty], dd[dd % world == rank]), "dev_dirty"
        assert np.array_equal(res.grp.grp_keys[got.grp_dirty], gd[gd % world == rank]), "grp_dirty"
        assert np.array_equal(got.dev_gone, want["dev_gone"][want["dev_gone"] % world == rank]), "dev_gone"
        assert np.array_equal(got.grp_gone, want["grp_gone"][want["grp_gone"] % world == rank]), "grp_gone"

    def check_merged(got, res, recs):
        """All ranks: the merged delta equals the single-GPU delta of the whole snapshot on `whole`."""
        m = kvgpu.merge_pci_shard_deltas(gather(kvgpu.shard_delta_part(res, got)))
        r2, d2 = whole.scan_pci_delta(recs)
        assert m.n_prev == d2.n_prev and m.n_now == len(r2.survivors)
        assert m.changes.tobytes() == d2.changes.tobytes(), "merged changes"
        assert np.array_equal(m.dev_dirty, r2.dev_keys[d2.dev_dirty]) and np.array_equal(m.dev_gone, d2.dev_gone)
        assert np.array_equal(m.grp_dirty, r2.grp_keys[d2.grp_dirty]) and np.array_equal(m.grp_gone, d2.grp_gone)
        return r2.survivors

    recs = snapshot(n, ids, seed=7)
    sh.delta_reset()
    whole.scan_pci_delta_reset()
    part_maps = kvgpu.Maps()
    prev_local, prev_all = np.zeros(0, kvgpu.PCI_SURV), np.zeros(0, kvgpu.PCI_SURV)
    pci_prev = None                              # what ctx.scan_pci_delta last saw (interleaved, other direction)
    for s in range(len(KINDS) + 1):
        if s:
            recs = step(recs, KINDS[s - 1], rng, ids)
        part = scan(recs)
        res, got = sh.fetch_delta()
        same_shard_result(res, sh.fetch())       # the same scan again: identical, and the previous result stays
        now_all = check_merged(got, res, recs)
        check_rank(got, res, prev_local, prev_all, now_all)
        if s == 0:
            assert got.n_prev == 0 and (got.changes["what"] == delta_ref.CH_ADDED).all()
            assert len(got.dev_dirty) == len(res.dev.dev_keys) and len(got.grp_dirty) == len(res.grp.grp_keys)
        kvgpu.apply_pci_shard_delta(part_maps, res, got)
        # the patched maps against the oracle: every step up to 1 Mi records per rank, else the first and the last
        # (a patch rewrites a dirty key whole, so a wrong one stays wrong until its key is dirty again)
        if n_per_rank < 1 << 20 or s in (0, len(KINDS)):
            om = O.Maps()
            om.create_iommu_device_map_flat(np.ascontiguousarray(recs))
            assert kvgpu.canonical_dump(kvgpu.merge_parts(gather(part_maps))) == om.dump(text), "patched maps"
        # the other deltas and scans on this context, in between: neither disturbs the other's previous result
        r3, d3 = ctx.scan_pci_delta(part)
        if pci_prev is not None:
            want = delta_ref.expect_pci_delta(pci_prev, r3.survivors, kvgpu.PCI_CHANGE)
            assert d3.changes.tobytes() == want["changes"].tobytes(), "kvg_scan_pci_delta disturbed"
        pci_prev = r3.survivors
        ctx.scan_pci(recs[:1000])
        prev_local, prev_all = res.local, now_all

    # the launch budget, on an input whose orderings have settled: exactly two beyond the plain fetch
    scan(recs)
    sh.fetch()
    scan(recs)
    c0 = ctx.launch_count
    sh.fetch_delta()
    c1 = ctx.launch_count
    scan(recs)
    c2 = ctx.launch_count
    sh.fetch()
    c3 = ctx.launch_count
    assert (c1 - c0) - (c3 - c2) == 2, "launches beyond the plain fetch: %d" % ((c1 - c0) - (c3 - c2))

    # reset: everything added, then a plain diff again
    scan(recs)
    sh.delta_reset()
    res, got = sh.fetch_delta()
    check_rank(got, res, prev_local[:0], prev_all[:0], prev_all)
    assert got.n_prev == 0 and len(got.changes) == len(res.local)
    scan(recs)
    res, got = sh.fetch_delta()
    assert got.n_prev == len(res.local) and len(got.changes) == 0 and len(got.dev_dirty) == 0

    # refusal on every rank (a repeated address in each shard): the previous result stays
    lo, hi = kvgpu.shard_range(len(recs), rank, world)
    alive = lo + np.nonzero(util.pci_alive(recs[lo:hi]))[0]
    bad = recs.copy()
    bad["addr"][alive[len(alive) // 2]] = bad["addr"][alive[len(alive) // 2 - 1]]
    scan(bad)
    try:
        ctx.dev_scan_pci_shard_fetch_delta()
        raise AssertionError("non-ascending shard accepted")
    except kvgpu.KvgError as e:
        assert e.rc == -1 and "ascending" in str(e), e
    nxt = step(recs, "regroup", rng, ids)
    scan(nxt)
    res, got = sh.fetch_delta()
    now_all = check_merged(got, res, nxt)
    check_rank(got, res, prev_local, prev_all, now_all)

    # refusal on rank 0 only: ShardedScan.fetch_delta resets every rank, the next step is a full "added" step
    scan(bad if rank == 0 else nxt)
    try:
        sh.fetch_delta()
        raise AssertionError("fetch_delta did not raise")
    except kvgpu.KvgError as e:
        # rank 0 refused; an owner of the repeated address refuses too, every other rank is reset by the collective
        assert e.rc == -1 if rank == 0 else e.rc in (-1, -5), e
    scan(nxt)
    res, got = sh.fetch_delta()
    assert got.n_prev == 0 and len(got.changes) == len(res.local) and len(got.dev_gone) == 0
    assert len(got.dev_dirty) == len(res.dev.dev_keys) and len(got.grp_dirty) == len(res.grp.grp_keys)

    dist.barrier()
    if rank == 0:
        print("shard-delta-ok world=%d n=%d exchange=%s" % (world, n_per_rank, sh.mode))
    sh.close()
    ctx.close()
    whole.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    # a failing rank must take the job down instead of hanging in collective teardown
    import faulthandler
    import traceback
    faulthandler.dump_traceback_later(int(os.environ.get("KVG_WORKER_STALL_S", "300")), exit=True)
    try:
        main()
    except BaseException:
        traceback.print_exc()
        sys.stderr.flush()
        os._exit(1)
