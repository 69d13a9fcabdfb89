"""Worker for the sharded mdev re-scan delta test (kvg_dev_scan_mdev_shard_fetch_delta): rank r scans its shard of a
sequence of mdev snapshots on GPU r (creates, destroys, retypes, parent and NUMA moves at about 0.1 % of the records
per step, and a reordered dictionary that moves labels between ranks; the record count changes, so shard boundaries
move) and checks every step:
  - the result equals a plain kvg_dev_scan_mdev_shard_fetch of the same scan;
  - its delta is exact: the local changes against mdev_delta_ref.expect_mdev_delta of its previous and new local
    survivors, the four key lists against the same restatement of its previous and new owned lists;
  - the ranks' deltas merged by merge_mdev_shard_deltas equal Context.scan_mdev_delta of the whole snapshot on a
    second context, and the parts patched by apply_mdev_shard_delta dump like the oracle;
  - plain sharded fetches, kvg_scan_mdev_delta, kvg_dev_scan_pci_shard_fetch_delta and their resets in between leave
    its previous result alone, and it and its reset leave theirs alone;
  - the first call and a reset report everything as added; a refusal keeps the previous result, and a refusal on
    one rank makes ShardedScan.fetch_mdev_delta reset every rank;
  - the call costs exactly three launches beyond the plain fetch, under stable labels.

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
import mdev_delta_ref
import util
from oracle import oracle as O
from test_gpu_mdev_delta import KINDS, NT, snapshot, step


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
    shard_cap = n_per_rank + n_per_rank // 50 + 64           # room for creates and moving boundaries
    # p2p_cap counts PCI records and an mdev record takes two
    sh = kvgpu.ShardedScan(ctx, rank, world, bcast, allgather if mode != "nccl" else None, 2 * shard_cap)
    assert sh.mode == "p2p" or not one_device, "rank %d: no peer windows on one device" % rank
    if mode == "p2p" and sh.mode != "p2p" and rank == 0:
        print("note: peer windows unavailable, fell back to NCCL")
    buf = torch.empty(shard_cap * 32, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(n_per_rank + world)
    # a small PCI snapshot for the sharded PCI delta that runs in between
    n_pci = 4000 * world
    pci = O.gen_pci(3, n_pci, ids, 16)
    pci["addr"] = np.arange(n_pci, dtype=np.uint32) * 4
    plo, phi = kvgpu.shard_range(n_pci, rank, world)
    pbuf = torch.from_numpy(np.ascontiguousarray(pci[plo:phi]).view(np.uint8).ravel().copy()).cuda()

    def scan(recs, types):
        lo, hi = kvgpu.shard_range(len(recs), rank, world)
        part = np.ascontiguousarray(recs[lo:hi])
        assert hi - lo <= shard_cap
        buf[:part.nbytes].copy_(torch.from_numpy(part.view(np.uint8).ravel()))
        torch.cuda.synchronize()
        # the ranks line up before every sharded scan: a rank's exchange waits at most ~10 s for its peers, and the
        # checks between two scans take longer on the ranks that own more keys (at P = 2 rank 0 owns every vGpuMap
        # key: the canonical ids of the synthetic dictionary are even)
        dist.barrier()
        sh.scan_device_mdev_shard(buf.data_ptr(), hi - lo, types)
        return part

    def same_shard_result(a, b):
        assert a.n_records == b.n_records and np.array_equal(a.local, b.local)
        for x, y in ((a.by_type, b.by_type), (a.by_parent, b.by_parent)):
            for f in ("survivors", "type_keys", "type_off", "type_perm", "labels", "type_canon", "type_names",
                      "par_keys", "par_off", "par_perm"):
                u, v = getattr(x, f), getattr(y, f)
                assert (np.array_equal(u, v) if isinstance(u, np.ndarray) else u == v), f

    def owned(surv):
        return surv[surv["type_key"] % world == rank], surv[surv["parent"] % world == rank]

    def check_rank(got, res, prev, prev_labels, now_all):
        """This rank's delta: local changes, and the four key lists of its owned lists."""
        now = [res.local, res.by_type.survivors, res.by_parent.survivors]
        for mine, want_own in zip(now[1:], owned(now_all)):
            for f in ("uuid", "parent", "type_key", "numa"):
                assert np.array_equal(mine[f], want_own[f]), "owned lists: " + f
        labels = res.by_type.labels
        exp = lambda a, b: mdev_delta_ref.expect_mdev_delta(a, b, prev_labels, labels, kvgpu.MDEV_CHANGE)
        loc, by_type, by_par = exp(prev[0], now[0]), exp(prev[1], now[1]), exp(prev[2], now[2])
        assert got.n_prev == len(prev[0])
        assert got.changes.tobytes() == loc["changes"].tobytes(), "local changes"
        assert np.array_equal(got.type_dirty, by_type["type_dirty"]), "type_dirty"
        assert got.type_gone == by_type["type_gone"], "type_gone"
        assert np.array_equal(got.par_dirty, by_par["par_dirty"]), "par_dirty"
        assert np.array_equal(got.par_gone, by_par["par_gone"]), "par_gone"

    def check_merged(got, res, recs, types):
        """All ranks: the merged delta equals the single-GPU delta of the whole snapshot on `whole`."""
        m = sh.merge_mdev_deltas(gather(kvgpu.mdev_shard_delta_part(res, got)))
        r2, d2 = whole.scan_mdev_delta(recs, types)
        assert m.n_prev == d2.n_prev and m.n_now == len(r2.survivors)
        assert m.changes.tobytes() == d2.changes.tobytes(), "merged changes"
        assert np.array_equal(m.type_dirty, r2.type_keys[d2.type_dirty]), "merged type_dirty"
        assert m.type_gone == d2.type_gone, "merged type_gone"
        assert np.array_equal(m.par_dirty, r2.par_keys[d2.par_dirty]) and np.array_equal(m.par_gone, d2.par_gone)
        return r2.survivors

    def lists(res):
        return [res.local, res.by_type.survivors, res.by_parent.survivors]

    state = {"mdev": None, "pci": None}          # what the other deltas on ctx last saw

    def other_deltas(part, types, reset=False):
        """kvg_scan_mdev_delta and the sharded PCI delta on the same context: each still diffs against its own
        previous result.  reset: forget both first."""
        if reset:
            ctx.scan_mdev_delta_reset()
            sh.delta_reset()
            state["mdev"] = state["pci"] = None
        r3, d3 = ctx.scan_mdev_delta(part, types)
        pm = state["mdev"]
        want = mdev_delta_ref.expect_mdev_delta(pm.survivors if pm else r3.survivors[:0], r3.survivors,
                                                pm.labels if pm else [], r3.labels, kvgpu.MDEV_CHANGE)
        assert d3.changes.tobytes() == want["changes"].tobytes() and d3.type_gone == want["type_gone"], \
            "kvg_scan_mdev_delta disturbed"
        state["mdev"] = r3
        dist.barrier()                           # as in scan()
        sh.scan_device_shard(pbuf.data_ptr(), phi - plo)
        pres, pd = sh.fetch_delta()
        pp = state["pci"] if state["pci"] is not None else pres.local[:0]
        want = delta_ref.expect_pci_delta(pp, pres.local, kvgpu.PCI_CHANGE)
        assert pd.n_prev == len(pp) and pd.changes.tobytes() == want["changes"].tobytes(), \
            "kvg_dev_scan_pci_shard_fetch_delta disturbed"
        state["pci"] = pres.local

    recs, types = snapshot(n, seed=7), O.gen_type_names(NT)
    sh.mdev_delta_reset()
    whole.scan_mdev_delta_reset()
    part_maps = kvgpu.Maps()
    prev = [np.zeros(0, kvgpu.MDEV_SURV)] * 3
    prev_labels = []
    for s in range(len(KINDS) + 1):
        if s:
            recs, types = step(recs, types, KINDS[s - 1], rng)
        part = scan(recs, types)
        res, got = sh.fetch_mdev_delta()
        same_shard_result(res, sh.fetch_mdev())  # the same scan again: identical, and the previous result stays
        now_all = check_merged(got, res, recs, types)
        check_rank(got, res, prev, prev_labels, now_all)
        if s == 0:
            assert got.n_prev == 0 and (got.changes["what"] == delta_ref.CH_ADDED).all()
            assert len(got.type_dirty) == len(res.by_type.type_keys)
            assert len(got.par_dirty) == len(res.by_parent.par_keys)
        kvgpu.apply_mdev_shard_delta(part_maps, res, got)
        # the patched maps against the oracle: every step up to 1 Mi records per rank, else the first and the last
        if n_per_rank < 1 << 20 or s in (0, len(KINDS)):
            om = O.Maps()
            om.create_vgpu_id_map_flat(np.ascontiguousarray(recs), types)
            assert kvgpu.canonical_dump(kvgpu.merge_parts(gather(part_maps))) == om.dump(text), "patched maps"
        # the other deltas on this context, in between (and, once, their resets): neither disturbs the other
        other_deltas(part, types, reset=s == 3)
        prev, prev_labels = lists(res), res.by_type.labels

    # the launch budget, on an input whose orderings have settled: exactly three beyond the plain fetch
    scan(recs, types)
    sh.fetch_mdev()
    scan(recs, types)
    c0 = ctx.launch_count
    sh.fetch_mdev_delta()
    c1 = ctx.launch_count
    scan(recs, types)
    c2 = ctx.launch_count
    sh.fetch_mdev()
    c3 = ctx.launch_count
    assert (c1 - c0) - (c3 - c2) == 3, "launches beyond the plain fetch: %d" % ((c1 - c0) - (c3 - c2))
    ctx.set_kernel_timing(True)
    try:
        scan(recs, types)
        sh.fetch_mdev_delta()
        labels = [name for name, _ in ctx.kernel_times()]
    finally:
        ctx.set_kernel_timing(False)
    assert labels[-3:] == ["shard_mdev_delta_types", "shard_mdev_delta_merge", "shard_mdev_delta_lists"], labels[-6:]

    # reset: everything added, then a plain diff again; the reset leaves the other deltas alone
    scan(recs, types)
    sh.mdev_delta_reset()
    res, got = sh.fetch_mdev_delta()
    check_rank(got, res, [a[:0] for a in prev], [], np.concatenate(gather(res.local)))
    assert got.n_prev == 0 and len(got.changes) == len(res.local)
    other_deltas(part, types)
    scan(recs, types)
    res, got = sh.fetch_mdev_delta()
    assert got.n_prev == len(res.local) and len(got.changes) == 0 and len(got.type_dirty) == 0
    assert got.type_gone == [] and len(got.par_dirty) == 0
    prev, prev_labels = lists(res), res.by_type.labels

    # refusal on every rank (a repeated UUID in each shard): the previous result stays
    bad = recs.copy()
    for r in range(world):
        rlo, rhi = kvgpu.shard_range(len(recs), r, world)
        alive = rlo + np.nonzero((recs["flags"][rlo:rhi] & 3) == 0)[0]
        bad["uuid"][alive[len(alive) // 2]] = bad["uuid"][alive[len(alive) // 2 - 1]]
    scan(bad, types)
    try:
        ctx.dev_scan_mdev_shard_fetch_delta()
        raise AssertionError("non-ascending shard accepted")
    except kvgpu.KvgError as e:
        assert e.rc == -1 and "ascending" in str(e), e
    nxt, ntypes = step(recs, types, "retype", rng)
    scan(nxt, ntypes)
    res, got = sh.fetch_mdev_delta()
    now_all = check_merged(got, res, nxt, ntypes)
    check_rank(got, res, prev, prev_labels, now_all)

    # refusal on rank 0 only: ShardedScan.fetch_mdev_delta resets every rank, the next step is a full "added" step
    scan(bad if rank == 0 else nxt, ntypes)
    try:
        sh.fetch_mdev_delta()
        raise AssertionError("fetch_mdev_delta did not raise")
    except kvgpu.KvgError as e:
        # rank 0 refused; an owner of the repeated UUID refuses too, every other rank is reset by the collective
        assert e.rc == -1 if rank == 0 else e.rc in (-1, -5), e
    scan(nxt, ntypes)
    res, got = sh.fetch_mdev_delta()
    assert got.n_prev == 0 and len(got.changes) == len(res.local) and got.type_gone == []
    assert len(got.type_dirty) == len(res.by_type.type_keys) and len(got.par_dirty) == len(res.by_parent.par_keys)

    dist.barrier()
    if rank == 0:
        print("mdev-shard-delta-ok world=%d n=%d exchange=%s" % (world, n_per_rank, sh.mode))
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
