"""Worker for tests/test_gpu_exchange_one_device.py: P ranks of the sharded scan as P processes on ONE GPU
(tests/_one_device.py), exchanging through each other's peer windows.  Every rank checks every scan exactly:
  - its local survivors against util.expect_pci / util.expect_mdev of its shard;
  - both owned lists against the whole snapshot's survivors whose key % P == rank, in Walk order, field by field
    (an mdev survivor's src is its index in the shard it came from);
  - both orderings (util.check_ordering), and the name slots / type names against the name table and getDeviceName;
  - up to DUMP_MAX records, the union of all ranks' map parts against the oracle's dump.
A peer that never delivers makes the fetch raise KVG_ENCCL, which fails the job like any other error.

Argument 1, the job:
  steps    PCI and mdev scans on the same windows, some three times back to back with no fetch in between, so both
           parities are reused and the acknowledgements are waited for: shards on tile edges with an empty shard and one without survivors; one owner taking every
           key with every region exactly full; no key staying home; every shard empty (PCI) or without survivors
           (mdev); a merging dictionary with sparse canonical ids and parent 0xFFFFFFFF; keys widened on one rank
           behind a re-parse; then the first step again with the shard roles rotated
  mixed    P = 2, shards of FUSED_SEND_MAX - 1 and FUSED_SEND_MAX + 1 records: in every scan one rank classifies and
           sends in one kernel and the other classifies, then sends with k_shard_send
  big N    one owner takes every key of N-record shards: owned lists P times longer than the orderings expect"""
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
import kvgpu
import util
from oracle import oracle as O

FUSED_SEND_MAX = 2 << 20      # shard records below which classify and send are one kernel (kvg_api_shard.inc)
DUMP_MAX = 200_000            # snapshots up to this size are also compared with the oracle's dump
PCI_FIELDS = ("addr", "iommu_group", "device", "numa")
MDEV_FIELDS = ("uuid", "parent", "type_key", "numa", "src")


def same_fields(got, want, fields, what):
    n = len(want[fields[0]])
    assert len(got) == n, "%s: %d records, want %d" % (what, len(got), n)
    for f in fields:
        if not np.array_equal(got[f], want[f]):
            bad = np.nonzero((got[f] != want[f]).reshape(n, -1).any(axis=1))[0][0]
            raise AssertionError("%s: %s differs first at %d: %r, want %r" % (what, f, bad, got[bad], want[f][bad]))


class Job:
    def __init__(self, cap):
        """cap: PCI records per shard (an mdev record takes two)."""
        self.rank, self.world, dev = _one_device.init()
        self.text = util.pciids_text()
        self.ids = O.nv_ids(self.text)
        self.ctx = kvgpu.Context(dev)
        self.ctx.pciids_load(self.text)
        self.names = self.ctx.name_table()
        self.cap = cap
        self.sh = kvgpu.ShardedScan(self.ctx, self.rank, self.world, _one_device.broadcast, _one_device.allgather, cap)
        assert self.sh.mode == "p2p", "rank %d: no peer windows on one device" % self.rank
        self.buf = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
        pad = self.ctx.text_pad(len(self.text))
        h = np.full(pad + 16, 10, dtype=np.uint8)
        h[:len(self.text)] = np.frombuffer(self.text, dtype=np.uint8)
        self.d_text, self.text_stride = torch.from_numpy(h).cuda(), pad + 16
        self.type_names = {}
        self.step = 0

    def reparse(self):
        """Parse pci.ids again on the device: the next scan runs beside the parse and joins its names late."""
        self.ctx.dev_pciids_parse(self.d_text.data_ptr(), len(self.text), self.text_stride, 1)

    def _shard(self, recs, sizes):
        assert len(sizes) == self.world and sum(sizes) == len(recs)
        lo = sum(sizes[:self.rank])
        shard = np.ascontiguousarray(recs[lo:lo + sizes[self.rank]])
        assert shard.nbytes <= self.buf.numel()
        if len(shard):
            self.buf[:shard.nbytes].copy_(torch.from_numpy(shard.view(np.uint8).reshape(-1)))
        torch.cuda.synchronize()
        # the ranks line up before every scan: host-side checks of different lengths never keep a peer spinning
        dist.barrier()
        return shard

    def _tag(self, what):
        return "rank %d scan %d (%s)" % (self.rank, self.step, what)

    def _names(self, lst, name_at, what):
        """Every survivor's name slot resolves to the name of its device id (one slot per id)."""
        if not len(lst):
            return
        pairs = np.unique((lst["device"].astype(np.uint64) << np.uint64(32)) | lst["name_slot"].astype(np.uint64))
        dev, slot = (pairs >> np.uint64(32)).astype(np.int64), pairs & np.uint64(0xFFFFFFFF)
        assert len(np.unique(dev)) == len(dev), what + ": a device id with two name slots"
        assert [name_at(int(s)) for s in slot] == [self.names[int(d)] for d in dev], what + ": names"

    def pci(self, recs, sizes, what, repeat=1):
        """Scan this rank's shard of recs (shards of `sizes` records, rank order) `repeat` times back to back, with
        no fetch in between (each scan's send waits for the peers' acknowledgements of the scan two before it), and
        check the last result."""
        P, r, tag = self.world, self.rank, self._tag(what)
        recs = np.ascontiguousarray(recs)
        shard = self._shard(recs, sizes)
        for _ in range(repeat):
            self.sh.scan_device_shard(self.buf.data_ptr(), len(shard))
        res = self.sh.fetch()
        same_fields(res.local, util.expect_pci(shard), PCI_FIELDS, tag + " local")
        whole = util.expect_pci(recs)
        for part, key in ((res.dev, "device"), (res.grp, "iommu_group")):
            mine = whole[key] % P == r
            same_fields(part.survivors, {f: whole[f][mine] for f in PCI_FIELDS}, PCI_FIELDS, tag + " owned by " + key)
        d, g = res.dev, res.grp
        util.check_ordering(d.survivors["device"], d.dev_keys, d.dev_off, d.dev_perm, tag + " device ordering")
        util.check_ordering(g.survivors["iommu_group"], g.grp_keys, g.grp_off, g.grp_perm, tag + " group ordering")
        assert [d.name_at(int(s)) for s in d.dev_name_slot] == [self.names[int(k)] for k in d.dev_keys], \
            tag + ": device-id names"
        for lst, name in ((res.local, "local"), (d.survivors, "owned by device"), (g.survivors, "owned by group")):
            self._names(lst, d.name_at, "%s %s" % (tag, name))
        if len(recs) <= DUMP_MAX:
            parts = _one_device.gather(kvgpu.pci_maps_from_shard(res))
            om = O.Maps()
            om.create_iommu_device_map_flat(recs)
            assert kvgpu.canonical_dump(kvgpu.merge_parts(parts)) == om.dump(self.text), tag + ": merged dump"
        self.step += 1

    def mdev(self, recs, sizes, types, what, repeat=1):
        P, r, tag = self.world, self.rank, self._tag(what)
        recs = np.ascontiguousarray(recs)
        shard = self._shard(recs, sizes)
        for _ in range(repeat):
            self.sh.scan_device_mdev_shard(self.buf.data_ptr(), len(shard), types)
        res = self.sh.fetch_mdev()
        same_fields(res.local, util.expect_mdev(shard, types), MDEV_FIELDS, tag + " local")
        whole = util.expect_mdev(recs, types)
        starts = np.cumsum([0] + list(sizes))
        src_shard = np.searchsorted(starts, whole["src"], side="right") - 1
        whole["src"] = (whole["src"] - starts[src_shard]).astype(np.uint32)   # the index in its own shard
        for part, key in ((res.by_type, "type_key"), (res.by_parent, "parent")):
            mine = whole[key] % P == r
            same_fields(part.survivors, {f: whole[f][mine] for f in MDEV_FIELDS}, MDEV_FIELDS, tag + " owned by " + key)
        t, p = res.by_type, res.by_parent
        util.check_ordering(t.survivors["type_key"], t.type_keys, t.type_off, t.type_perm, tag + " type ordering")
        util.check_ordering(p.survivors["parent"], p.par_keys, p.par_off, p.par_perm, tag + " parent ordering")
        labels, canon = util.mdev_labels(types)
        assert t.labels == labels and np.array_equal(t.type_canon.astype(np.int64), canon), tag + ": dictionary"
        key = tuple(types)
        if key not in self.type_names:
            self.type_names[key] = [O.get_device_name(self.text, lb) for lb in labels]
        assert t.type_names == self.type_names[key], tag + ": type names"
        if len(recs) <= DUMP_MAX:
            parts = _one_device.gather(kvgpu.mdev_maps_from_shard(res))
            om = O.Maps()
            om.create_vgpu_id_map_flat(recs, types)
            assert kvgpu.canonical_dump(kvgpu.merge_parts(parts)) == om.dump(self.text), tag + ": merged dump"
        self.step += 1

    # ---- synthetic snapshots (the same on every rank: seeded) -------------------------------------------------
    def ids_owned_by(self, q):
        s = self.ids[self.ids % self.world == q]
        assert len(s), "no device id of the table is owned by %d" % q
        return s

    def pci_owned(self, sizes, owner, rng):
        """Every record survives; shard q's device ids and groups are owned by owner(q).  addr = Walk index."""
        recs = np.zeros(sum(sizes), dtype=kvgpu.PCI_REC)
        recs["addr"] = np.arange(len(recs))
        recs["vendor"] = 0x10DE
        recs["driver"] = rng.integers(1, 3, len(recs))                 # vfio-pci or nvgrace
        recs["flags"] = np.where(rng.random(len(recs)) < 0.05, 16, 0)   # NUMA unreadable: still a survivor
        recs["numa"] = rng.integers(-1, 4, len(recs))
        lo = 0
        for q, n in enumerate(sizes):
            o = owner(q)
            recs["device"][lo:lo + n] = rng.choice(self.ids_owned_by(o), n)
            recs["iommu_group"][lo:lo + n] = rng.integers(0, 256, n) * self.world + o
            lo += n
        return recs

    def mdev_owned(self, sizes, owner, types, rng):
        """Every record survives; shard q's canonical types and parents are owned by owner(q)."""
        _, canon = util.mdev_labels(types)
        recs = np.zeros(sum(sizes), dtype=kvgpu.MDEV_REC)
        idx = np.arange(len(recs), dtype=np.uint32)
        recs["uuid"][:, :4] = idx.astype(">u4").view(np.uint8).reshape(-1, 4)
        recs["uuid"][:, 4:] = rng.integers(0, 256, (len(recs), 12))
        recs["parent_numa"] = rng.integers(-1, 4, len(recs))
        lo = 0
        for q, n in enumerate(sizes):
            o = owner(q)
            recs["type_idx"][lo:lo + n] = rng.choice(np.nonzero(canon % self.world == o)[0], n)
            recs["parent"][lo:lo + n] = rng.integers(0, 256, n) * self.world + o
            lo += n
        return recs

    def close(self):
        dist.barrier()
        self.sh.close()
        self.ctx.close()


def sparse_dictionary():
    """300 raw types whose labels merge (white-space variants of 12 names) and whose canonical ids are sparse."""
    first = [0, 5, 6, 40, 41, 99, 128, 200, 255, 256, 298, 299]
    forms = (lambda b: b + b"\n", lambda b: b.replace(b" ", b"  ") + b"\n", lambda b: b.replace(b" ", b"\t"),
             lambda b: b"\n" + b.replace(b" ", b" \t ") + b"\n")
    out = []
    for i in range(300):
        j = max(k for k, f in enumerate(first) if f <= i)
        out.append(forms[i % 4](b"GRID A100-%dC" % j if j % 3 else b"NVIDIA SYN%02X-1Q" % j))
    return out


def steps_job():
    P = int(os.environ["WORLD_SIZE"])
    cap = 1026                                            # PCI records per shard; an mdev shard holds up to 513
    J = Job(cap)
    rng = np.random.default_rng(4321)                     # the same snapshots on every rank
    types = O.gen_type_names(256)
    own_types = [b"OWNER %d\n" % k for k in range(64)]    # distinct labels: canonical id == index, any residue

    def natural(shift):
        """Shard sizes on tile edges (1024 PCI / 512 mdev records a tile): role P-1 is empty, role P-2 (P >= 3) has
        records but no survivors; roles rotate with `shift`."""
        role = [(q + shift) % P for q in range(P)]
        ps = [0 if k == P - 1 else (1023, 1024, 1025)[k % 3] for k in role]
        ms = [0 if k == P - 1 else (511, 512, 513)[(k + 2) % 3] for k in role]
        prec = O.gen_pci(0, sum(ps), J.ids, 12)
        mrec = O.gen_mdev(0, sum(ms))
        dead = [q for q in range(P) if role[q] == P - 2 and P >= 3]
        for q in dead:
            prec["driver"][sum(ps[:q]):sum(ps[:q + 1])] = 3           # neither vfio-pci nor nvgrace
            mrec["flags"][sum(ms[:q]):sum(ms[:q + 1])] |= 1           # type unreadable
        J.pci(prec, ps, "tile edges, shift %d" % shift, repeat=3)
        J.mdev(mrec, ms, types, "tile edges, shift %d" % shift, repeat=3)

    # 1: natural data
    natural(0)
    # 2: one owner takes every key; every region of its window exactly full
    J.pci(J.pci_owned([cap] * P, lambda q: P - 1, rng), [cap] * P, "one owner", repeat=3)
    J.mdev(J.mdev_owned([cap // 2] * P, lambda q: P - 1, own_types, rng), [cap // 2] * P, own_types, "one owner")
    # 3: nothing stays home
    ps = [700 + 37 * q % 300 for q in range(P)]
    ms = [300 + 11 * q % 200 for q in range(P)]
    J.pci(J.pci_owned(ps, lambda q: (q + 1) % P, rng), ps, "nothing home")
    J.mdev(J.mdev_owned(ms, lambda q: (q + 1) % P, own_types, rng), ms, own_types, "nothing home")
    # 4: every PCI shard empty, every mdev shard without survivors
    J.pci(np.zeros(0, kvgpu.PCI_REC), [0] * P, "all empty")
    dead = O.gen_mdev(0, 100 * P)
    dead["flags"] |= 2                                    # parent unreadable
    J.mdev(dead, [100] * P, types, "no survivors")
    # 5: a merging dictionary with sparse canonical ids; parents 0xFFFFFFFF; a shard of exactly cap / 2 records
    ms = [(513, 511, 512)[q % 3] for q in range(P)]
    sd = sparse_dictionary()
    mrec = O.gen_mdev(1_000_000, sum(ms))
    mrec["type_idx"] = rng.integers(0, len(sd) + 20, len(mrec))       # some outside the dictionary
    top = np.nonzero((mrec["flags"] & 3) == 0)[0][[0, len(mrec) // 2, -1]]
    mrec["parent"][top] = 0xFFFFFFFF
    mrec["type_idx"][top] = 299
    J.mdev(mrec, ms, sd, "sparse dictionary")
    # 6: widened keys on one rank only (group 0xFFFFFFFF, device 0xFFFF), behind a re-parse
    ps = [900 + 7 * q for q in range(P)]
    prec = O.gen_pci(10_000, sum(ps), J.ids, 12)
    w = P // 2
    lo = sum(ps[:w])
    for i, (f, v) in ((lo, ("iommu_group", 0xFFFFFFFF)), (lo + ps[w] - 1, ("device", 0xFFFF))):
        prec["vendor"][i], prec["driver"][i], prec["flags"][i] = 0x10DE, 1, 0
        prec[f][i] = v
    J.reparse()
    J.pci(prec, ps, "wide keys")
    # 7: the first step again, roles rotated
    natural(1)
    J.close()
    return "steps=%d" % J.step


def mixed_job():
    assert int(os.environ["WORLD_SIZE"]) == 2
    lo, hi = FUSED_SEND_MAX - 1, FUSED_SEND_MAX + 1
    J = Job(2 * hi)
    prec = O.gen_pci(0, lo + hi, J.ids, 17)
    mrec = O.gen_mdev(0, lo + hi)
    types = O.gen_type_names(256)
    J.pci(prec, [lo, hi], "fused | standalone send")
    J.mdev(mrec, [hi, lo], types, "standalone | fused send")
    J.pci(prec, [hi, lo], "standalone | fused send")
    J.mdev(mrec, [lo, hi], types, "fused | standalone send")
    J.close()
    return "steps=%d" % J.step


def big_job(n):
    P = int(os.environ["WORLD_SIZE"])
    J = Job(n)
    rng = np.random.default_rng(n + P)
    for o in (P - 1, 0):
        J.pci(J.pci_owned([n] * P, lambda q: o, rng), [n] * P, "owner %d takes all" % o, repeat=2)
    J.close()
    return "steps=%d n=%d" % (J.step, n)


def main():
    job = sys.argv[1]
    if job == "steps":
        info = steps_job()
    elif job == "mixed":
        info = mixed_job()
    elif job == "big":
        info = big_job(int(sys.argv[2]))
    else:
        raise SystemExit("unknown job " + job)
    if dist.get_rank() == 0:
        print("exchange-ok job=%s world=%d %s exchange=p2p" % (job, dist.get_world_size(), info), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    # a failing rank must take the job down instead of leaving its peers to time out in the exchange
    import faulthandler
    import traceback
    faulthandler.dump_traceback_later(int(os.environ.get("KVG_WORKER_STALL_S", "300")), exit=True)
    try:
        main()
    except BaseException:
        traceback.print_exc()
        sys.stderr.flush()
        os._exit(1)
