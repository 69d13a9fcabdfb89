"""Multi-GPU sharding of the scan (BASELINE.json config 4): one process per GPU.

Records are range-partitioned in Walk order, rank r owns [r*N/P, (r+1)*N/P).  Every rank classifies its
shard; its survivors stay local (rank order == Walk order: the host concatenates them for bdfToIommuMap).
ONE exchange step sends every survivor to the OWNER of its key (key % P), once per group-by map, so each
rank ends up with all members of the keys it owns — constant volume per GPU whatever P is.  Transport:
stores into the owners' peer windows over NVLink (CUDA IPC), or — fallback — one NCCL allgatherv of the
survivor lists followed by a local select.  The pci.ids table is parsed by every rank itself.

Re-scan deltas (Context.dev_scan_pci_shard_fetch_delta): each rank diffs its own shard and the keys it owns with no
communication; apply_pci_shard_delta patches its part of the maps, and merge_pci_shard_deltas over the ranks'
shard_delta_part summaries gives the delta of the whole snapshot.  The mdev form (dev_scan_mdev_shard_fetch_delta,
apply_mdev_shard_delta, mdev_shard_delta_part, merge_mdev_shard_deltas) works the same way; a vGpuMap label whose owner
moved between two scans (the dictionary renumbered) is gone on one rank and dirty on the other, and the merge derives
the global type lists from the fused changes.

`ShardedScan` needs only byte collectives (broadcast for the 128-byte NCCL unique id, all-gather for the
64-byte IPC handles), so the same class is driven by torch.distributed (bench.py) or any other launcher.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import _lib as L
from .context import Context, MdevShardResult, PciShardResult
from .plugin import (Maps, MdevMapsTouched, PciMapsTouched, _fully_numeric, _mdev_maps, _numeric_mdev, _patch_mdev_maps,
                     _patch_pci_maps, _pci_maps, _rebuild_into, _rebuild_mdev_maps)


def shard_range(n: int, rank: int, world: int) -> tuple[int, int]:
    """[lo, hi) of rank's contiguous shard; shards tile [0, n) exactly, sizes differ by <= 1."""
    if world < 1 or not 0 <= rank < world:
        raise ValueError("bad rank/world")
    return (n * rank) // world, (n * (rank + 1)) // world


def concat_in_rank_order(parts: list) -> list:
    """The host-side statement of what the allgatherv does: shard outputs concatenated in rank
    order are the global Walk-order list (used by the gloo CPU tests)."""
    out = []
    for p in parts:
        out.extend(p)
    return out


def allgatherv_torch(local, dist_mod=None):
    """Backend-agnostic statement of the exchange step (same algorithm as the NCCL path in
    kvg_dev_scan_pci_sharded): all-gather the per-rank counts, then one broadcast per root into the
    rank-ordered output.  `local` is a 1-D torch tensor; works on gloo (CPU tests) and nccl."""
    import torch
    import torch.distributed as dist
    dist = dist_mod or dist
    world, rank = dist.get_world_size(), dist.get_rank()
    cnt = torch.tensor([local.numel()], dtype=torch.int64, device=local.device)
    counts = [torch.zeros_like(cnt) for _ in range(world)]
    dist.all_gather(counts, cnt)
    counts = [int(c.item()) for c in counts]
    out = torch.empty(sum(counts), dtype=local.dtype, device=local.device)
    off = 0
    for root in range(world):
        seg = out[off:off + counts[root]]
        if root == rank:
            seg.copy_(local)
        if counts[root]:
            dist.broadcast(seg, root)
        off += counts[root]
    return out, counts


def pci_maps_from_shard(sh: PciShardResult) -> Maps:
    """This rank's part of the three PCI maps: deviceMap / iommuMap for the keys it owns (all members),
    bdfToIommuMap for its own shard's survivors."""
    return _pci_maps(Maps(), sh.dev, sh.grp, sh.local)


def mdev_maps_from_shard(sh: MdevShardResult) -> Maps:
    """This rank's part of vGpuMap (type labels it owns) and gpuVgpuMap (parents it owns)."""
    return _mdev_maps(Maps(), sh.by_type, sh.by_parent)


def apply_pci_shard_delta(part: Maps, res: PciShardResult, delta, snap=None, prev_snap=None) -> PciMapsTouched:
    """Patch one rank's part of the maps (pci_maps_from_shard of its previous fetch_delta result) into what
    pci_maps_from_shard(res) builds: the owned deviceMap / iommuMap keys that are dirty or gone and the local
    bdfToIommuMap entries of changed addresses, nothing else.  As in apply_pci_delta, a snapshot that is not fully
    numeric has no stable handles: the part is then rebuilt and every key is reported."""
    if not (_fully_numeric(snap) and _fully_numeric(prev_snap)):
        def build(m):
            fresh = pci_maps_from_shard(res)
            for key in set(m.deviceMap) - set(fresh.deviceMap):
                m.deviceNames.pop(key, None)
            m.deviceMap, m.iommuMap, m.bdfToIommuMap = fresh.deviceMap, fresh.iommuMap, fresh.bdfToIommuMap
            m.deviceNames.update(fresh.deviceNames)
        return _rebuild_into(part, build)
    return _patch_pci_maps(part, res.dev, res.grp, delta)


@dataclass
class PciShardDelta:
    """A re-scan delta with its keys as values: one rank's part (shard_delta_part; indices local to its shard) or
    the whole snapshot's (merge_pci_shard_deltas; indices into the concatenated survivor lists)."""
    n_prev: int                 # survivors of the previous result
    n_now: int                  # survivors now
    changes: np.ndarray         # PCI_CHANGE, ascending addr
    dev_dirty: np.ndarray       # u16 device ids whose (addr, numa) member sequence changed, ascending
    dev_gone: np.ndarray        # u16 device ids absent now, ascending
    grp_dirty: np.ndarray       # u32 groups, ascending
    grp_gone: np.ndarray        # u32 groups absent now, ascending


def shard_delta_part(res: PciShardResult, delta) -> PciShardDelta:
    """The small summary of one rank's fetch_delta that the merge needs: counts, changes and key values (no member
    arrays, so all_gather_object ships little)."""
    return PciShardDelta(int(delta.n_prev), len(res.local), delta.changes,
                         res.dev.dev_keys[delta.dev_dirty].astype(np.uint16), delta.dev_gone,
                         res.grp.grp_keys[delta.grp_dirty].astype(np.uint32), delta.grp_gone)


def _merge_shard_changes(parts: list, dtype, key_name: str, key, bits) -> tuple:
    """The ranks' changes (rank order) as those of the whole snapshot -> (changes, n_prev, n_now).  Local indices
    become global through prefix sums of the per-rank counts, and the changes are sorted by key(changes), an (n, w)
    array of unsigned words, most significant first.  A key seen twice must be REMOVED on one rank and ADDED on
    another (it crossed a shard boundary): the pair fuses into one entry with the previous side of the REMOVED one and
    the new side of the ADDED one, whose bits(fused) compare the two survivors (none: no entry)."""
    none = np.uint32(0xFFFFFFFF)
    prev_off = np.cumsum([0] + [p.n_prev for p in parts])
    now_off = np.cumsum([0] + [p.n_now for p in parts])
    chs = []
    for r, p in enumerate(parts):
        c = p.changes.copy()
        c["prev_index"] = np.where(c["prev_index"] == none, none, c["prev_index"] + np.uint32(prev_off[r]))
        c["now_index"] = np.where(c["now_index"] == none, none, c["now_index"] + np.uint32(now_off[r]))
        chs.append(c)
    ch = np.concatenate(chs) if chs else np.zeros(0, dtype)
    k = key(ch)
    order = np.lexsort(k.T[::-1])
    ch, k = ch[order], k[order]
    dup = np.nonzero((k[1:] == k[:-1]).all(axis=1))[0]          # pairs: i (one side), i + 1 (the other)
    if len(dup):
        rem = (ch["what"][dup] & L.CH_REMOVED) != 0             # which of the two is the REMOVED entry
        gone_, new_ = ch[np.where(rem, dup, dup + 1)], ch[np.where(rem, dup + 1, dup)]
        if not ((gone_["what"] == L.CH_REMOVED) & (new_["what"] == L.CH_ADDED)).all():
            raise ValueError("one %s twice, not as REMOVED + ADDED: the shards overlap" % key_name)
        f = new_.copy()
        for side in (name for name in dtype.names if name.startswith("prev_")):
            f[side] = gone_[side]
        f["what"] = bits(f).astype(np.uint32)
        keep = np.ones(len(ch), dtype=bool)
        keep[dup + 1] = False
        ch[dup] = f
        keep[dup[f["what"] == 0]] = False
        ch = ch[keep]
    return np.ascontiguousarray(ch), int(prev_off[-1]), int(now_off[-1])


def merge_pci_shard_deltas(parts: list) -> PciShardDelta:
    """The delta of the whole snapshot from the ranks' shard_delta_part summaries (rank order): equal to
    kvg_scan_pci_delta on the concatenated snapshot (changes byte for byte, dirty keys as values).  Changes are
    sorted by address; an address that crossed a shard boundary is REMOVED on one rank and ADDED on another, and
    the pair fuses into one entry whose bits compare the two survivors (none: no entry).  Local indices become
    global through prefix sums of the per-rank counts; the key lists are unions (ranks own disjoint keys)."""
    bits = lambda f: ((f["prev_group"] != f["now_group"]) * L.CH_GROUP
                      | (f["prev_device"] != f["now_device"]) * L.CH_DEVICE | (f["prev_numa"] != f["now_numa"]) * L.CH_NUMA)
    ch, n_prev, n_now = _merge_shard_changes(parts, L.PCI_CHANGE, "address", lambda ch: ch["addr"][:, None], bits)
    cat = lambda name, dt: np.unique(np.concatenate([getattr(p, name) for p in parts] + [np.zeros(0, dt)])).astype(dt)
    return PciShardDelta(n_prev, n_now, ch, cat("dev_dirty", np.uint16),
                         cat("dev_gone", np.uint16), cat("grp_dirty", np.uint32), cat("grp_gone", np.uint32))


def apply_mdev_shard_delta(part: Maps, res: MdevShardResult, delta, snap=None, prev_snap=None) -> MdevMapsTouched:
    """Patch one rank's part of the mdev maps (mdev_maps_from_shard of its previous fetch_mdev_delta result) IN PLACE
    into what mdev_maps_from_shard(res) builds: the owned vGpuMap / gpuVgpuMap keys that are dirty or gone, nothing
    else.  As in apply_mdev_delta, a snapshot without canonical UUIDs and packed-BDF parents has no stable handles: the
    part is then rebuilt (in place) and every key is reported."""
    if not (_numeric_mdev(snap) and _numeric_mdev(prev_snap)):
        return _rebuild_mdev_maps(part, res.by_type, res.by_parent, snap)
    return _patch_mdev_maps(part, res.by_type, res.by_parent, delta)


@dataclass
class MdevShardDelta:
    """An mdev re-scan delta with its keys as values: one rank's part (mdev_shard_delta_part; indices local to its
    shard, key lists over the keys it owns) or the whole snapshot's (merge_mdev_shard_deltas; indices into the
    concatenated survivor lists)."""
    n_prev: int                 # survivors of the previous result
    n_now: int                  # survivors now
    changes: np.ndarray         # MDEV_CHANGE, ascending UUID
    type_keys: np.ndarray       # u16 canonical ids of the vGpuMap keys now (a part: the ones the rank owns), ascending
    type_dirty: np.ndarray      # u16 canonical ids (this result's dictionary) whose (uuid, numa) sequence changed
    type_gone: list             # labels (bytes) absent now, ascending previous canonical id
    par_dirty: np.ndarray       # u32 parent handles whose uuid sequence changed, ascending
    par_gone: np.ndarray        # u32 parent handles absent now, ascending


def mdev_shard_delta_part(res: MdevShardResult, delta) -> MdevShardDelta:
    """The small summary of one rank's fetch_mdev_delta that the merge needs: counts, changes, the owned type keys and
    the key values (no member arrays)."""
    keys = res.by_type.type_keys.astype(np.uint16)
    return MdevShardDelta(int(delta.n_prev), len(res.local), delta.changes, keys, keys[delta.type_dirty],
                          list(delta.type_gone), res.by_parent.par_keys[delta.par_dirty].astype(np.uint32),
                          np.asarray(delta.par_gone, np.uint32))


def _canonical_ids(labels: list) -> dict:
    """label -> canonical id (the smallest raw index with that label) of one dictionary"""
    out = {}
    for i, lb in enumerate(labels):
        out.setdefault(bytes(lb), i)
    return out


def merge_mdev_shard_deltas(parts: list, prev_labels: list, now_labels: list) -> MdevShardDelta:
    """The delta of the whole snapshot from the ranks' mdev_shard_delta_part summaries (rank order): equal to
    kvg_scan_mdev_delta on the concatenated snapshot.  prev_labels / now_labels: the labels of the previous and the new
    dictionary (MdevResult.labels; every rank loads the same dictionary).  Changes are fused as in
    merge_pci_shard_deltas (KVG_CH_TYPE compares the labels through the two dictionaries) and come out byte for byte.
    The vGpuMap lists follow from the fused changes by the rule of the kernels: a change dirties the label it joined,
    and the label it left if that label is still a key somewhere (some rank owns it now), else that label is gone.  They
    are not the union of the ranks' lists: a label that moved between ranks with unchanged members is gone on one rank
    and dirty on the other, yet neither in the whole snapshot's delta.  Parent handles never change owner, so the
    gpuVgpuMap lists are unions."""
    prev_lab = [bytes(b) for b in prev_labels]
    now_lab = [bytes(b) for b in now_labels]
    key = lambda ch: np.ascontiguousarray(ch["uuid"]).reshape(-1, 16).view(">u8").astype(np.uint64)
    relabel = lambda f: np.array([prev_lab[int(a)] != now_lab[int(b)] for a, b in zip(f["prev_type"], f["now_type"])],
                                 bool)
    bits = lambda f: (relabel(f) * L.CH_TYPE | (f["prev_parent"] != f["now_parent"]) * L.CH_PARENT
                      | (f["prev_numa"] != f["now_numa"]) * L.CH_NUMA)
    ch, n_prev, n_now = _merge_shard_changes(parts, L.MDEV_CHANGE, "UUID", key, bits)
    type_keys = np.unique(np.concatenate([p.type_keys for p in parts] + [np.zeros(0, np.uint16)])).astype(np.uint16)
    now_id = _canonical_ids(now_lab)
    live = set(type_keys.tolist())
    dirty, gone = set(), set()
    for c in ch[(ch["what"] & (L.CH_ADDED | L.CH_REMOVED | L.CH_TYPE | L.CH_NUMA)) != 0]:
        has_now, has_prev = c["now_index"] != L.NO_INDEX, c["prev_index"] != L.NO_INDEX
        if has_now:
            dirty.add(int(c["now_type"]))
        if has_prev:
            label = prev_lab[int(c["prev_type"])]
            if has_now and label == now_lab[int(c["now_type"])]:
                continue
            same = now_id.get(label)
            if same is not None and same in live:
                dirty.add(same)
            else:
                gone.add(int(c["prev_type"]))
    cat = lambda name: np.unique(np.concatenate([getattr(p, name) for p in parts] + [np.zeros(0, np.uint32)]))
    return MdevShardDelta(n_prev, n_now, ch, type_keys,
                          np.array(sorted(dirty), np.uint16), [prev_lab[c] for c in sorted(gone)],
                          cat("par_dirty").astype(np.uint32), cat("par_gone").astype(np.uint32))


def merge_parts(parts: list) -> Maps:
    """Union of the ranks' parts (rank order): key sets are disjoint, bdfToIommuMap concatenates in rank
    order == Walk order."""
    out = Maps()
    for p in parts:
        for name in ("deviceMap", "iommuMap", "vGpuMap", "gpuVgpuMap"):
            mine, theirs = getattr(out, name), getattr(p, name)
            clash = set(mine) & set(theirs)
            if clash:
                raise ValueError("%s: key owned by two ranks: %r" % (name, sorted(clash)[:3]))
            mine.update(theirs)
        out.bdfToIommuMap.update(p.bdfToIommuMap)
        out.deviceNames.update(p.deviceNames)
    return out


class ShardedScan:
    def __init__(self, ctx: Context, rank: int, world: int, broadcast_bytes, allgather_bytes=None,
                 p2p_cap: int = 0):
        """broadcast_bytes(b: bytes | None, src=0) -> bytes : collective byte broadcast (NCCL unique id).
        allgather_bytes(b: bytes) -> list[bytes] (rank order) + p2p_cap (PCI records per shard; an mdev
        record takes two): set up the peer windows (CUDA IPC over NVLink) first; only if that fails on any
        rank is the NCCL communicator created.  Every rank takes the same decision (it follows from the
        all-gathered status bytes), so libnccl is never loaded when the peer windows work — and ranks that
        share one GPU, which NCCL refuses, can still exchange."""
        self.ctx, self.rank, self.world = ctx, rank, world
        self._bcast, self._allgather = broadcast_bytes, allgather_bytes
        self.mdev_prev_labels, self.mdev_labels = [], []   # dictionaries of the last fetch_mdev_delta: before, now
        self.mode = "nccl"
        if allgather_bytes is not None and p2p_cap > 0:
            try:
                mine = ctx.comm_p2p_export(rank, world, p2p_cap)
                ok = b"\1"
            except Exception:
                mine, ok = b"\0" * 64, b"\0"
            blobs = allgather_bytes(mine + ok)            # every rank learns whether all exported
            if all(b[64:65] == b"\1" for b in blobs):
                try:
                    ctx.comm_p2p_import(b"".join(b[:64] for b in blobs))
                    good = b"\1"
                except Exception:
                    good = b"\0"
                if all(g == b"\1" for g in allgather_bytes(good)):
                    ctx.comm_p2p_enable(True)
                    self.mode = "p2p"
        if self.mode == "nccl":
            uid = ctx.comm_unique_id() if rank == 0 else None
            uid = broadcast_bytes(uid, 0)
            ctx.comm_init(rank, world, uid)

    def scan_device_shard(self, d_recs: int, n_local: int):
        self.ctx.dev_scan_pci_sharded(d_recs, n_local)

    def fetch(self) -> PciShardResult:
        return self.ctx.dev_scan_pci_shard_fetch()

    def fetch_delta(self):
        """fetch plus this rank's share of the re-scan delta -> (PciShardResult, PciDelta), see
        Context.dev_scan_pci_shard_fetch_delta.  Collective here (not in the library): every rank learns every
        rank's status.  If any rank's call failed, EVERY rank resets its previous result and raises KvgError, so that
        the ranks never diff against previous results of different steps; the next step then reports everything as
        added on every rank."""
        return self._collective(self.ctx.dev_scan_pci_shard_fetch_delta, self.ctx.dev_scan_pci_shard_delta_reset,
                                "fetch_delta")

    def delta_reset(self):
        """Forget this rank's previous result (call it on every rank)."""
        self.ctx.dev_scan_pci_shard_delta_reset()

    def _collective(self, call, reset, name: str):
        """call() on this rank.  If it raised KvgError on any rank, every rank calls reset() and raises: the rank's own
        error, or KVG_ESTATE for a failure elsewhere."""
        err, out = None, None
        try:
            out = call()
        except L.KvgError as e:
            err = e
        if all(s[:1] == b"\1" for s in self._statuses(b"\0" if err else b"\1")):
            return out
        reset()
        if err is not None:
            raise err
        raise L.KvgError(L.KVG_ESTATE, "%s failed on another rank; every rank's previous result is reset" % name)

    def _statuses(self, mine: bytes) -> list:
        """every rank's status byte, in rank order"""
        if self._allgather is not None:
            return self._allgather(mine)
        return [self._bcast(mine if q == self.rank else None, q) for q in range(self.world)]

    def scan_device_mdev_shard(self, d_recs: int, n_local: int, raw_types: list):
        self.ctx.dev_scan_mdev_sharded(d_recs, n_local, raw_types)

    def fetch_mdev(self) -> MdevShardResult:
        return self.ctx.dev_scan_mdev_shard_fetch()

    def fetch_mdev_delta(self):
        """fetch_mdev plus this rank's share of the mdev re-scan delta -> (MdevShardResult, MdevDelta), see
        Context.dev_scan_mdev_shard_fetch_delta.  Collective here exactly like fetch_delta: if any rank's call failed,
        EVERY rank resets its previous result and raises KvgError.  The labels of the dictionary the delta was taken
        against are kept, so that merge_mdev_deltas needs only the ranks' parts."""
        out = self._collective(self.ctx.dev_scan_mdev_shard_fetch_delta, self.mdev_delta_reset, "fetch_mdev_delta")
        self.mdev_prev_labels, self.mdev_labels = self.mdev_labels, list(out[0].by_type.labels)
        return out

    def mdev_delta_reset(self):
        """Forget this rank's previous mdev result (call it on every rank)."""
        self.ctx.dev_scan_mdev_shard_delta_reset()
        self.mdev_labels = []

    def merge_mdev_deltas(self, parts: list) -> MdevShardDelta:
        """merge_mdev_shard_deltas of the ranks' parts of the last fetch_mdev_delta, with the labels it kept."""
        return merge_mdev_shard_deltas(parts, self.mdev_prev_labels, self.mdev_labels)

    def close(self):
        self.ctx.comm_destroy()
