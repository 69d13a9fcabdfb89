"""Context: thin object wrapper over the C-ABI (one CUDA stream, single-threaded)."""
from __future__ import annotations

import ctypes as C
import os
import threading
from dataclasses import dataclass

import numpy as np

from . import _lib as L


@dataclass
class PciResult:
    """Flat output of kvg_scan_pci (see include/kvgpu.h kvg_pci_result)."""
    n_records: int
    survivors: np.ndarray       # PCI_SURV, Walk order
    dev_keys: np.ndarray        # u16 ascending
    dev_off: np.ndarray
    dev_perm: np.ndarray
    dev_name_slot: np.ndarray
    grp_keys: np.ndarray        # u32 ascending
    grp_off: np.ndarray
    grp_perm: np.ndarray
    name_pool: bytes

    def name_at(self, slot: int) -> str:
        if slot == L.KVG_NO_NAME:
            return ""
        n = self.name_pool[slot] | (self.name_pool[slot + 1] << 8)
        return self.name_pool[slot + 2:slot + 2 + n].decode("latin-1")


@dataclass
class MdevResult:
    n_records: int
    survivors: np.ndarray       # MDEV_SURV
    type_keys: np.ndarray
    type_off: np.ndarray
    type_perm: np.ndarray
    labels: list                # sanitised label per raw dictionary entry (bytes)
    type_canon: np.ndarray
    type_names: list            # getDeviceName(label) per raw entry (str, "" = miss)
    par_keys: np.ndarray
    par_off: np.ndarray
    par_perm: np.ndarray


@dataclass
class PciShardResult:
    """One rank's part of a sharded PCI scan (include/kvgpu.h kvg_pci_shard_result): its own shard's
    survivors, and ALL members of the device ids / iommu groups it owns (key % nranks == rank)."""
    n_records: int
    local: np.ndarray           # PCI_SURV, this shard's survivors, Walk order
    dev: PciResult              # deviceMap part: survivors = the owned members (grp_* arrays empty)
    grp: PciResult              # iommuMap part:  survivors = the owned members (dev_* arrays empty)


@dataclass
class MdevShardResult:
    n_records: int
    local: np.ndarray           # MDEV_SURV
    by_type: MdevResult         # vGpuMap part (par_* empty)
    by_parent: MdevResult       # gpuVgpuMap part (type_* empty)


@dataclass
class HealthDelta:
    n_records: int
    n_alive: int
    changed: np.ndarray         # (index << 1) | now_alive


@dataclass
class PciDelta:
    """What changed since the previous scan_pci_delta (include/kvgpu.h kvg_pci_delta)."""
    n_prev: int
    changes: np.ndarray         # PCI_CHANGE, ascending addr
    dev_dirty: np.ndarray       # u32 indices into the result's dev_keys, ascending
    dev_gone: np.ndarray        # u16 device ids absent now, ascending
    grp_dirty: np.ndarray       # u32 indices into the result's grp_keys, ascending
    grp_gone: np.ndarray        # u32 groups absent now, ascending
    by_name: bool = False       # scan_pci_raw_delta: keyed by entry name, each side in its own snapshot's encoding


@dataclass
class MdevDelta:
    """What changed since the previous scan_mdev_delta (include/kvgpu.h kvg_mdev_delta)."""
    n_prev: int
    changes: np.ndarray         # MDEV_CHANGE, ascending UUID
    type_dirty: np.ndarray      # u32 indices into the result's type_keys, ascending
    type_gone: list             # labels (bytes) of the vGpuMap keys absent now, ascending previous canonical id
    par_dirty: np.ndarray       # u32 indices into the result's par_keys, ascending
    par_gone: np.ndarray        # u32 parent handles absent now, ascending
    by_name: bool = False       # scan_mdev_raw_delta: keyed by entry name, each side in its own snapshot's encoding


class _LockedLib:
    """A kvg_ctx is single-threaded (include/kvgpu.h).  gRPC handler threads, the health feed and the
    Allocate re-validation all share one Context (kvgpu/serve.py), so every C call on it is serialised."""

    def __init__(self, lib, lock):
        self._lib, self._lock = lib, lock

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*a):
            with self._lock:
                return fn(*a)
        return call


class Context:
    def __init__(self, device: int = 0):
        self._lock = threading.RLock()
        self._lib = _LockedLib(L.load(), self._lock)
        h = C.c_void_p()
        rc = self._lib.kvg_ctx_create(device, C.byref(h))
        if rc != 0:
            raise L.KvgError(rc, (self._lib.kvg_last_error(None) or b"").decode())
        self._h = h
        self.device = device

    # -- plumbing ---------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self._lib.kvg_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc):
        if rc != 0:
            raise L.KvgError(rc, (self._lib.kvg_last_error(self._h) or b"").decode())

    @property
    def handle(self):
        return self._h

    @property
    def stream(self) -> int:
        return int(self._lib.kvg_stream(self._h) or 0)

    @property
    def launch_count(self) -> int:
        return int(self._lib.kvg_launch_count(self._h))

    # -- pci.ids ----------------------------------------------------------------------------
    def pciids_load(self, text: bytes):
        buf = C.create_string_buffer(text, len(text)) if text else None
        self._ck(self._lib.kvg_pciids_load(self._h, C.cast(buf, C.c_void_p) if buf else None,
                                           len(text)))

    def name_lookup(self, key) -> str:
        """getDeviceName(key) — device_plugin.go:371-422."""
        if isinstance(key, str):
            key = key.encode("latin-1")
        cap = 1 << 17
        out = C.create_string_buffer(cap)
        n = C.c_size_t()
        self._ck(self._lib.kvg_name_lookup(self._h, key, len(key), out, cap, C.byref(n)))
        return out.raw[:n.value].decode("latin-1")

    def name_table(self, first: int = 0, count: int = 65536) -> list:
        off = np.zeros(count + 1, dtype=np.uint32)
        cap = 1 << 22
        out = np.zeros(cap, dtype=np.uint8)
        self._ck(self._lib.kvg_name_table(self._h, first, count, off.ctypes.data, out.ctypes.data,
                                          cap))
        raw = out.tobytes()
        return [raw[off[i]:off[i + 1]].decode("latin-1") for i in range(count)]

    def pciids_info(self) -> dict:
        v = [C.c_uint32() for _ in range(4)]
        self._ck(self._lib.kvg_pciids_info(self._h, *[C.byref(x) for x in v]))
        return dict(zip(("vendor_off", "section_end", "n_entries", "n_lines"),
                        [x.value for x in v]))

    # -- scans ------------------------------------------------------------------------------
    def _take_pci(self, res) -> PciResult:
        r = res.contents
        S, KD, G = int(r.n_survivors), int(r.n_dev_keys), int(r.n_groups)
        dev_off = L._arr(r.dev_off, KD + 1, np.uint32)
        grp_off = L._arr(r.grp_off, G + 1, np.uint32)
        # a sharded scan orders only the keys this rank owns: perms are as long as off[-1]
        out = PciResult(
            n_records=int(r.n_records),
            survivors=L._arr(r.survivors, S, L.PCI_SURV),
            dev_keys=L._arr(r.dev_keys, KD, np.uint16),
            dev_off=dev_off,
            dev_perm=L._arr(r.dev_perm, int(dev_off[-1]), np.uint32),
            dev_name_slot=L._arr(r.dev_name_slot, KD, np.uint32),
            grp_keys=L._arr(r.grp_keys, G, np.uint32),
            grp_off=grp_off,
            grp_perm=L._arr(r.grp_perm, int(grp_off[-1]), np.uint32),
            name_pool=C.string_at(r.name_pool, r.name_pool_len) if r.name_pool_len else b"")
        self._lib.kvg_result_free(res)
        return out

    def scan_pci(self, recs: np.ndarray) -> PciResult:
        """createIommuDeviceMap on a flat snapshot — device_plugin.go:187-247."""
        recs = np.ascontiguousarray(recs, dtype=L.PCI_REC)
        res = C.POINTER(L.PciResultC)()
        self._ck(self._lib.kvg_scan_pci(self._h, recs.ctypes.data, len(recs), C.byref(res)))
        return self._take_pci(res)

    def scan_pci_raw(self, raw):
        """createIommuDeviceMap from the raw reads of its walk (plugin.read_pci_tree_raw): the GPU decodes them into the
        snapshot snapshot_pci_tree packs, then scans it -> (PciResult, PciSnapshot).  Raises plugin.ReferencePanic
        where the Go reference would panic."""
        return self._scan_pci_raw(raw, None)

    def scan_pci_raw_delta(self, raw):
        """scan_pci_raw plus the diff against the previous scan_pci_raw_delta on this context, keyed by entry name and
        exact in every snapshot mode -> (PciResult, PciSnapshot, PciDelta).  Each side of a change is in its own
        snapshot's encoding, so the caller keeps the previous PciSnapshot to name what was removed or has gone."""
        dl = C.POINTER(L.PciDeltaC)()
        res, snap = self._scan_pci_raw(raw, dl)
        delta = self._take_pci_delta(dl)
        delta.by_name = True
        return res, snap, delta

    def scan_pci_raw_delta_reset(self):
        self._ck(self._lib.kvg_scan_pci_raw_delta_reset(self._h))

    def _scan_pci_raw(self, raw, dl):
        """kvg_scan_pci_raw, or kvg_scan_pci_raw_delta into `dl` -> (PciResult, PciSnapshot)"""
        from .plugin import PciSnapshot

        def table(n, off_p, bytes_p):
            return [b.decode("latin-1") for b in self._table(n, off_p, bytes_p)]

        return self._scan_raw(
            "kvg_scan_pci_raw", L.PciRawC, L.PciResultC, L.PciSnapC, self._take_pci, raw, dl,
            lambda sn: PciSnapshot(
                L._arr(sn.recs, int(sn.n_records), L.PCI_REC), list(raw.names), bool(sn.packed_addr),
                None if sn.groups_numeric else table(sn.n_group_names, sn.group_off, sn.group_bytes),
                None if sn.devices_numeric else table(sn.n_device_names, sn.device_off, sn.device_bytes)))

    def _scan_raw(self, entry: str, arg_t, res_t, snap_t, take, raw, dl, snapshot):
        """`entry` (kvg_scan_<kind>_raw), or `entry`_delta into `dl`, on the raw reads `raw` (a PciRaw or MdevRaw,
        passed as an arg_t) -> (take(result), snapshot(decoded snapshot)).  KVG_EPANIC raises plugin.ReferencePanic."""
        from .plugin import ReferencePanic
        off = np.ascontiguousarray(raw.off, dtype=np.uint32)
        state = np.ascontiguousarray(raw.state, dtype=np.uint16)
        blob = np.frombuffer(bytes(raw.bytes) + b"\0", dtype=np.uint8)
        arg = arg_t(len(state), off.ctypes.data, blob.ctypes.data, state.ctypes.data)
        res, snap = C.POINTER(res_t)(), C.POINTER(snap_t)()
        if dl is None:
            rc = getattr(self._lib, entry)(self._h, C.byref(arg), C.byref(res), C.byref(snap))
        else:
            rc = getattr(self._lib, entry + "_delta")(self._h, C.byref(arg), C.byref(res), C.byref(snap), C.byref(dl))
        if rc == L.KVG_EPANIC:
            raise ReferencePanic((self._lib.kvg_last_error(self._h) or b"").decode("latin-1"))
        self._ck(rc)
        out = snapshot(snap.contents)
        self._lib.kvg_result_free(snap)
        return take(res), out

    @staticmethod
    def _table(n, off_p, bytes_p) -> list:
        """The n strings (bytes) of a snapshot string table."""
        o = L._arr(off_p, int(n) + 1, np.uint32)
        b = C.string_at(bytes_p, int(o[-1])) if o[-1] else b""
        return [b[o[k]:o[k + 1]] for k in range(int(n))]

    @staticmethod
    def _type_dict(raw_types):
        off = np.zeros(len(raw_types) + 1, dtype=np.uint32)
        for i, t in enumerate(raw_types):
            off[i + 1] = off[i] + len(t)
        blob = np.frombuffer(b"".join(raw_types) + b"\0", dtype=np.uint8).copy()
        td = L.TypeDict(len(raw_types), off.ctypes.data_as(C.POINTER(C.c_uint32)),
                        blob.ctypes.data_as(C.POINTER(C.c_uint8)))
        return td, (off, blob)

    def _take_mdev(self, res) -> MdevResult:
        r = res.contents
        S, KT, P, nt = int(r.n_survivors), int(r.n_type_keys), int(r.n_parents), int(r.n_types)
        loff = L._arr(r.label_off, nt + 1, np.uint32)
        noff = L._arr(r.type_name_off, nt + 1, np.uint32)
        lbytes = C.string_at(r.label_bytes, int(loff[-1])) if nt and loff[-1] else b""
        nbytes = C.string_at(r.type_name_bytes, int(noff[-1])) if nt and noff[-1] else b""
        out = MdevResult(
            n_records=int(r.n_records),
            survivors=L._arr(r.survivors, S, L.MDEV_SURV),
            type_keys=L._arr(r.type_keys, KT, np.uint16),
            type_off=L._arr(r.type_off, KT + 1, np.uint32),
            type_perm=L._arr(r.type_perm, S, np.uint32),
            labels=[lbytes[loff[i]:loff[i + 1]] for i in range(nt)],
            type_canon=L._arr(r.type_canon, nt, np.uint16),
            type_names=[nbytes[noff[i]:noff[i + 1]].decode("latin-1") for i in range(nt)],
            par_keys=L._arr(r.par_keys, P, np.uint32),
            par_off=L._arr(r.par_off, P + 1, np.uint32),
            par_perm=L._arr(r.par_perm, S, np.uint32))
        self._lib.kvg_result_free(res)
        return out

    def scan_mdev(self, recs: np.ndarray, raw_types: list) -> MdevResult:
        """createVgpuIDMap on a flat snapshot — device_plugin.go:255-291."""
        recs = np.ascontiguousarray(recs, dtype=L.MDEV_REC)
        td, keep = self._type_dict(raw_types)
        res = C.POINTER(L.MdevResultC)()
        self._ck(self._lib.kvg_scan_mdev(self._h, recs.ctypes.data, len(recs), C.byref(td),
                                         C.byref(res)))
        del keep
        return self._take_mdev(res)

    def scan_mdev_raw(self, raw):
        """createVgpuIDMap from the raw reads of its walk (plugin.read_mdev_tree_raw): the GPU decodes them into a
        snapshot and its raw type dictionary, then scans it -> (MdevResult, MdevSnapshot).  Raises plugin.ReferencePanic
        where the Go reference would panic."""
        return self._scan_mdev_raw(raw, None)

    def scan_mdev_raw_delta(self, raw):
        """scan_mdev_raw plus the diff against the previous scan_mdev_raw_delta on this context, keyed by entry name (the
        UUID string) and exact in every snapshot mode -> (MdevResult, MdevSnapshot, MdevDelta).  Parents are in each
        side's own snapshot's encoding, so the caller keeps the previous MdevSnapshot to name gone parents."""
        dl = C.POINTER(L.MdevDeltaC)()
        res, snap = self._scan_mdev_raw(raw, dl)
        delta = self._take_mdev_delta(dl)
        delta.by_name = True
        return res, snap, delta

    def scan_mdev_raw_delta_reset(self):
        self._ck(self._lib.kvg_scan_mdev_raw_delta_reset(self._h))

    def _scan_mdev_raw(self, raw, dl):
        """kvg_scan_mdev_raw, or kvg_scan_mdev_raw_delta into `dl` -> (MdevResult, MdevSnapshot)"""
        from .plugin import MdevSnapshot
        return self._scan_raw(
            "kvg_scan_mdev_raw", L.MdevRawC, L.MdevResultC, L.MdevSnapC, self._take_mdev, raw, dl,
            lambda sn: MdevSnapshot(
                L._arr(sn.recs, int(sn.n_records), L.MDEV_REC), list(raw.names),
                self._table(sn.n_types, sn.type_off, sn.type_bytes),
                None if sn.parents_packed else
                [p.decode("latin-1") for p in self._table(sn.n_parent_names, sn.parent_off, sn.parent_bytes)],
                bool(sn.uuid_ok)))

    def mdev_label_match(self, raw_files: list, name) -> np.ndarray:
        r"""The vGPU plugin's Allocate-time re-check (include/kvgpu.h kvg_mdev_label_match), one launch: element i is
        True iff the label of raw_files[i] (Trim "\n", then every \s+ run -> "_") equals `name`.  A str name is
        encoded as latin-1, the decoding the plugin's labels use."""
        if isinstance(name, str):
            name = name.encode("latin-1")
        td, keep = self._type_dict(raw_files)
        match = np.zeros(max(len(raw_files), 1), dtype=np.uint8)
        self._ck(self._lib.kvg_mdev_label_match(self._h, C.byref(td), name, len(name), match.ctypes.data))
        del keep
        return match[:len(raw_files)].astype(bool)

    def pci_group_check(self, recs: np.ndarray, want) -> int | None:
        """The passthrough plugin's Allocate-time re-check (include/kvgpu.h kvg_pci_group_check), one launch: the
        index of the first record whose iommu_group is not want[i] or whose vendor is not 10de (or whose read of
        either failed), or None when every record passes.  Group handles are interned strings, never numbers."""
        recs = np.ascontiguousarray(recs, dtype=L.PCI_REC)
        want = np.ascontiguousarray(want, dtype=np.uint32)
        if len(want) != len(recs):
            raise ValueError("pci_group_check: %d records but %d wanted groups" % (len(recs), len(want)))
        first = C.c_size_t()
        self._ck(self._lib.kvg_pci_group_check(self._h, recs.ctypes.data, want.ctypes.data, len(recs),
                                               C.byref(first)))
        return None if first.value == len(recs) else first.value

    def pci_allocate_check(self, recs: np.ndarray, want, n_members, ids, n_ids, egm_off, egm_gpu,
                           n_egm_gpus: int) -> tuple:
        """The passthrough plugin's Allocate decisions for every container request of one call, one launch
        (include/kvgpu.h kvg_pci_allocate_check).  recs / want: the members of every request, request after request,
        as for pci_group_check; ids: the requests' DevicesIDs as EGM handles, request after request; n_members, n_ids:
        one count per request; egm_off / egm_gpu: each EGM device's GPU handles (egm_off has one entry more than there
        are devices, or none for no device).  Returns (first_bad, take): first_bad[r] = the first failing position of
        request r, or n_members[r]; take[r, e] = request r holds every GPU of EGM device e."""
        recs = np.ascontiguousarray(recs, dtype=L.PCI_REC)
        want = np.ascontiguousarray(want, dtype=np.uint32)
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        egm_off = np.ascontiguousarray(egm_off, dtype=np.uint32)
        egm_gpu = np.ascontiguousarray(egm_gpu, dtype=np.uint32)
        if len(want) != len(recs) or len(n_members) != len(n_ids):
            raise ValueError("pci_allocate_check: %d records but %d wanted groups, %d / %d per-request counts"
                             % (len(recs), len(want), len(n_members), len(n_ids)))
        reqs = np.zeros(len(n_members), dtype=L.ALLOC_REQ)
        reqs["n_members"], reqs["n_ids"] = n_members, n_ids
        n_egm = max(len(egm_off) - 1, 0)
        first_bad = np.zeros(len(reqs), dtype=np.uint32)
        take = np.zeros((len(reqs), n_egm), dtype=np.uint8)
        self._ck(self._lib.kvg_pci_allocate_check(
            self._h, reqs.ctypes.data, len(reqs), recs.ctypes.data, want.ctypes.data, len(recs), ids.ctypes.data,
            len(ids), egm_off.ctypes.data if len(egm_off) else None, egm_gpu.ctypes.data, n_egm, n_egm_gpus,
            first_bad.ctypes.data, take.ctypes.data))
        return first_bad, take.astype(bool)

    def pci_allocate_raw(self, raw) -> tuple:
        """The passthrough plugin's Allocate decisions for every container request of one call, from the raw reads
        (include/kvgpu.h kvg_pci_allocate_raw; plugin.pack_alloc_raw builds `raw`).  Returns (first_bad, panic, kept,
        take): first_bad[r] = the first failing position of request r, or its member count; panic[r] = that member's
        vendor read is the reference's panic; kept[e] = EGM class entry e is an EGM device; take[r, e] = request r
        mounts entry e.  Raises KvgError for a reached read that was not made (KVG_EINVAL) and for more than
        ALLOC_RAW_MAX_EGM_KEYS distinct EGM keys (KVG_ERANGE)."""
        arr = lambda a, t: np.ascontiguousarray(a, dtype=t)   # noqa: E731
        blob = lambda b: np.frombuffer(bytes(b) + b"\0", dtype=np.uint8)   # noqa: E731
        n_members, n_ids = arr(raw.n_members, np.uint32), arr(raw.n_ids, np.uint32)
        moff, mst, ioff = arr(raw.member_off, np.uint32), arr(raw.member_state, np.uint16), arr(raw.id_off, np.uint32)
        eoff, est = arr(raw.egm_off, np.uint32), arr(raw.egm_state, np.uint16)
        mb, ib, eb = blob(raw.member_bytes), blob(raw.id_bytes), blob(raw.egm_bytes)
        if len(n_members) != len(n_ids):
            raise ValueError("pci_allocate_raw: %d / %d per-request counts" % (len(n_members), len(n_ids)))
        reqs = np.zeros(len(n_members), dtype=L.ALLOC_REQ)
        reqs["n_members"], reqs["n_ids"] = n_members, n_ids
        n_egm = len(est)
        arg = L.AllocRawC(len(mst), moff.ctypes.data, mb.ctypes.data, mst.ctypes.data, max(len(ioff) - 1, 0),
                          ioff.ctypes.data, ib.ctypes.data, n_egm, eoff.ctypes.data, eb.ctypes.data, est.ctypes.data)
        first_bad = np.zeros(len(reqs), dtype=np.uint32)
        panic = np.zeros(len(reqs), dtype=np.uint8)
        kept = np.zeros(n_egm, dtype=np.uint8)
        take = np.zeros((len(reqs), n_egm), dtype=np.uint8)
        self._ck(self._lib.kvg_pci_allocate_raw(self._h, reqs.ctypes.data, len(reqs), C.byref(arg),
                                                first_bad.ctypes.data, panic.ctypes.data, kept.ctypes.data,
                                                take.ctypes.data))
        return first_bad, panic.astype(bool), kept.astype(bool), take.astype(bool)

    def pci_allocate_response(self, raw, resp) -> list:
        """The passthrough plugin's AllocateResponse for every container request of one call, from the raw reads
        (include/kvgpu.h kvg_pci_allocate_response; plugin.pack_alloc_response builds `raw` and `resp`).  Returns per
        request (error, at, paths, env): error = ARESP_*, at = its DevicesID index (ARESP_UNKNOWN_ID) or member
        position; paths = the device specs' host paths (bytes), in order; env = the env value (bytes), or None when
        the key is absent.  Raises KvgError for a refusal (KVG_EINVAL, KVG_ERANGE)."""
        arr = lambda a, t: np.ascontiguousarray(a, dtype=t)   # noqa: E731
        blob = lambda b: np.frombuffer(bytes(b) + b"\0", dtype=np.uint8)   # noqa: E731
        n_members, n_ids = arr(raw.n_members, np.uint32), arr(raw.n_ids, np.uint32)
        moff, mst, ioff = arr(raw.member_off, np.uint32), arr(raw.member_state, np.uint16), arr(raw.id_off, np.uint32)
        eoff, est = arr(raw.egm_off, np.uint32), arr(raw.egm_state, np.uint16)
        mb, ib, eb = blob(raw.member_bytes), blob(raw.id_bytes), blob(raw.egm_bytes)
        if not len(n_members) == len(n_ids) == len(resp.n_visited) == len(resp.lookup_error):
            raise ValueError("pci_allocate_response: %d / %d / %d / %d per-request counts"
                             % (len(n_members), len(n_ids), len(resp.n_visited), len(resp.lookup_error)))
        reqs = np.zeros(len(n_members), dtype=L.ALLOC_REQ)
        reqs["n_members"], reqs["n_ids"] = n_members, n_ids
        arg = L.AllocRawC(len(mst), moff.ctypes.data, mb.ctypes.data, mst.ctypes.data, max(len(ioff) - 1, 0),
                          ioff.ctypes.data, ib.ctypes.data, len(est), eoff.ctypes.data, eb.ctypes.data, est.ctypes.data)
        keep = [arr(resp.n_visited, np.uint32), arr(resp.lookup_error, np.uint8), arr(resp.id_members, np.uint32),
                arr(resp.addr_off, np.uint32), blob(resp.addr_bytes), arr(resp.vfio_first, np.uint32),
                arr(resp.vfio_off, np.uint32), blob(resp.vfio_bytes), arr(resp.vfio_dir, np.uint8),
                arr(resp.vfio_state, np.uint8)]
        rin = L.AllocRespInC(int(resp.iommufd), *[a.ctypes.data for a in keep])
        out = C.POINTER(L.AllocRespC)()
        self._ck(self._lib.kvg_pci_allocate_response(self._h, reqs.ctypes.data, len(reqs), C.byref(arg),
                                                     C.byref(rin), C.byref(out)))
        o = out.contents
        n = len(reqs)
        error, at = L._arr(o.error, n, np.uint8), L._arr(o.error_at, n, np.uint32)
        first, n_specs = L._arr(o.spec_first, n, np.uint32), L._arr(o.n_specs, n, np.uint32)
        env_len, env_key = L._arr(o.env_len, n, np.uint32), L._arr(o.env_key, n, np.uint8)
        res = []
        for r in range(n):
            span = L._arr(o.spec_span + 8 * int(first[r]), 2 * int(n_specs[r]), np.uint32) if n_specs[r] else []
            paths = [C.string_at(o.spec_bytes + int(span[2 * k]), int(span[2 * k + 1])) for k in range(int(n_specs[r]))]
            env = C.string_at(o.env_bytes, int(env_len[r])) if env_key[r] else None
            res.append((int(error[r]), int(at[r]), paths, env))
        self._lib.kvg_result_free(out)
        return res

    def preferred_allocation(self, ids, n_must, n_avail, sizes) -> list:
        """GetPreferredAllocation's NUMA packing for every container request of one call, one launch
        (include/kvgpu.h kvg_preferred_allocation).  ids: PREF_ID entries, request after request, each request's
        must-include entries first; n_must, n_avail, sizes: one value per request.  Returns (n_out, n_must_distinct,
        positions) per request: n_out = -1 when the must-include IDs outnumber the size, else the picks as entry
        positions within the request, in the order the reference appends them."""
        ids = np.ascontiguousarray(ids, dtype=L.PREF_ID)
        n_must, n_avail = np.asarray(n_must, dtype=np.int64), np.asarray(n_avail, dtype=np.int64)
        sizes = np.asarray(sizes, dtype=np.int64)
        if not (len(n_must) == len(n_avail) == len(sizes)):
            raise ValueError("preferred_allocation: %d / %d / %d per-request values"
                             % (len(n_must), len(n_avail), len(sizes)))
        reqs = np.zeros(len(sizes), dtype=L.PREF_REQ)
        reqs["n_must"], reqs["n_avail"], reqs["size"] = n_must, n_avail, sizes
        res = np.zeros(len(reqs), dtype=L.PREF_RES)
        pos = np.zeros(len(ids), dtype=np.uint32)
        self._ck(self._lib.kvg_preferred_allocation(self._h, reqs.ctypes.data, len(reqs), ids.ctypes.data, len(ids),
                                                    res.ctypes.data, pos.ctypes.data))
        out, at = [], 0
        for r in range(len(reqs)):
            n = int(res["n_out"][r])
            out.append((n, int(res["n_must_distinct"][r]), pos[at:at + max(n, 0)].astype(np.int64)))
            at += int(n_must[r] + n_avail[r])
        return out

    def _take_health(self, res) -> HealthDelta:
        r = res.contents
        out = HealthDelta(int(r.n_records), int(r.n_alive),
                          L._arr(r.changed, int(r.n_changed), np.uint32))
        self._lib.kvg_result_free(res)
        return out

    def health_rescan(self, recs: np.ndarray) -> HealthDelta:
        recs = np.ascontiguousarray(recs, dtype=L.PCI_REC)
        res = C.POINTER(L.HealthDeltaC)()
        self._ck(self._lib.kvg_health_rescan(self._h, recs.ctypes.data, len(recs), C.byref(res)))
        return self._take_health(res)

    def health_reset(self):
        self._ck(self._lib.kvg_health_reset(self._h))

    def health_rescan_mdev(self, recs: np.ndarray, n_types: int, xid_parents=()) -> HealthDelta:
        """vGPU health re-scan (include/kvgpu.h kvg_health_rescan_mdev): a record is healthy while it passes
        createVgpuIDMap's keep rule and no XID on its parent marked it since it last appeared.  `xid_parents`: the
        parent handles of the GPUs that reported a critical XID since the previous call (at most 1024)."""
        recs = np.ascontiguousarray(recs, dtype=L.MDEV_REC)
        x = np.ascontiguousarray(np.asarray(xid_parents, dtype=np.uint32).reshape(-1))
        res = C.POINTER(L.HealthDeltaC)()
        self._ck(self._lib.kvg_health_rescan_mdev(self._h, recs.ctypes.data, len(recs), int(n_types),
                                                  x.ctypes.data if len(x) else None, len(x), C.byref(res)))
        return self._take_health(res)

    def health_mdev_reset(self):
        self._ck(self._lib.kvg_health_mdev_reset(self._h))

    def health_rescan_groups(self, recs: np.ndarray, group_nodes=()) -> HealthDelta:
        """Passthrough health re-scan by IOMMU group (include/kvgpu.h kvg_health_rescan_groups): a record is healthy
        while it passes createIommuDeviceMap's filter and the VFIO node of its group exists.  `group_nodes`: the
        handles (kvg_pci_rec.iommu_group encoding) of the groups whose node exists now (at most 4096)."""
        recs = np.ascontiguousarray(recs, dtype=L.PCI_REC)
        g = np.ascontiguousarray(np.asarray(group_nodes, dtype=np.uint32).reshape(-1))
        res = C.POINTER(L.HealthDeltaC)()
        self._ck(self._lib.kvg_health_rescan_groups(self._h, recs.ctypes.data, len(recs),
                                                    g.ctypes.data if len(g) else None, len(g), C.byref(res)))
        return self._take_health(res)

    def health_groups_reset(self):
        self._ck(self._lib.kvg_health_groups_reset(self._h))

    def health_rescan_mdev_keyed(self, recs: np.ndarray, n_types: int, xid_parents=()) -> HealthDelta:
        """health_rescan_mdev with the state kept per UUID (include/kvgpu.h kvg_health_rescan_mdev_keyed): the UUIDs
        of `recs` must ascend strictly (big-endian bytes); a vGPU keeps its XID mark while it stays in the list,
        whatever else is added or removed.  `changed` indexes this call's records.  An empty `recs` resets."""
        recs = np.ascontiguousarray(recs, dtype=L.MDEV_REC)
        x = np.ascontiguousarray(np.asarray(xid_parents, dtype=np.uint32).reshape(-1))
        res = C.POINTER(L.HealthDeltaC)()
        self._ck(self._lib.kvg_health_rescan_mdev_keyed(self._h, recs.ctypes.data, len(recs), int(n_types),
                                                        x.ctypes.data if len(x) else None, len(x), C.byref(res)))
        return self._take_health(res)

    def health_rescan_groups_keyed(self, recs: np.ndarray, group_nodes=()) -> HealthDelta:
        """health_rescan_groups with the state kept per address (include/kvgpu.h kvg_health_rescan_groups_keyed): the
        addresses of `recs` must ascend strictly.  `changed` indexes this call's records.  An empty `recs` resets."""
        recs = np.ascontiguousarray(recs, dtype=L.PCI_REC)
        g = np.ascontiguousarray(np.asarray(group_nodes, dtype=np.uint32).reshape(-1))
        res = C.POINTER(L.HealthDeltaC)()
        self._ck(self._lib.kvg_health_rescan_groups_keyed(self._h, recs.ctypes.data, len(recs),
                                                          g.ctypes.data if len(g) else None, len(g), C.byref(res)))
        return self._take_health(res)

    def health_rescan_groups_raw(self, raw, nodes=()) -> HealthDelta:
        """Passthrough health re-scan by IOMMU group from raw reads (include/kvgpu.h kvg_health_rescan_groups_raw):
        `raw` is a PciRaw of the advertised devices (plugin.read_pci_ids_raw), names ascending byte-wise; `nodes` the
        names (bytes) of one listing of the VFIO directory (plugin.list_nodes_raw).  The state is kept per entry name;
        `changed` indexes this call's entries.  An empty `raw` resets.  Raises plugin.ReferencePanic where the Go
        reference would panic."""
        return self._health_raw("kvg_health_rescan_groups_raw", L.PciRawC, raw, nodes)

    def health_rescan_mdev_raw(self, raw, xid_parents=()) -> HealthDelta:
        """vGPU health re-scan from raw reads (include/kvgpu.h kvg_health_rescan_mdev_raw): `raw` is an MdevRaw of the
        advertised vGPUs (plugin.read_mdev_ids_raw), names ascending byte-wise; `xid_parents` the bus ids (bytes) of
        the GPUs that reported a critical XID since the previous call, matched against the decoded parent strings.
        The state is kept per entry name.  An empty `raw` resets."""
        return self._health_raw("kvg_health_rescan_mdev_raw", L.MdevRawC, raw, xid_parents)

    def _health_raw(self, entry: str, arg_t, raw, strs) -> HealthDelta:
        from .plugin import ReferencePanic
        off = np.ascontiguousarray(raw.off, dtype=np.uint32)
        state = np.ascontiguousarray(raw.state, dtype=np.uint16)
        blob = np.frombuffer(bytes(raw.bytes) + b"\0", dtype=np.uint8)
        arg = arg_t(len(state), off.ctypes.data, blob.ctypes.data, state.ctypes.data)
        td, keep = self._type_dict([os.fsencode(x) if isinstance(x, str) else bytes(x) for x in strs])
        res = C.POINTER(L.HealthDeltaC)()
        rc = getattr(self._lib, entry)(self._h, C.byref(arg), C.byref(td), C.byref(res))
        del keep
        if rc == L.KVG_EPANIC:
            raise ReferencePanic((self._lib.kvg_last_error(self._h) or b"").decode("latin-1"))
        self._ck(rc)
        return self._take_health(res)

    def _take_pci_delta(self, dl) -> PciDelta:
        d = dl.contents
        delta = PciDelta(int(d.n_prev), L._arr(d.changes, int(d.n_changes), L.PCI_CHANGE),
                         L._arr(d.dev_dirty, int(d.n_dev_dirty), np.uint32),
                         L._arr(d.dev_gone, int(d.n_dev_gone), np.uint16),
                         L._arr(d.grp_dirty, int(d.n_grp_dirty), np.uint32),
                         L._arr(d.grp_gone, int(d.n_grp_gone), np.uint32))
        self._lib.kvg_result_free(dl)
        return delta

    def scan_pci_delta(self, recs: np.ndarray):
        """scan_pci plus the keyed diff against the previous scan_pci_delta on this context -> (PciResult, PciDelta).
        Meaningful for numeric (packed-BDF) snapshots; with index-mode handles it is relative to the handles."""
        recs = np.ascontiguousarray(recs, dtype=L.PCI_REC)
        res = C.POINTER(L.PciResultC)()
        dl = C.POINTER(L.PciDeltaC)()
        self._ck(self._lib.kvg_scan_pci_delta(self._h, recs.ctypes.data, len(recs), C.byref(res), C.byref(dl)))
        delta = self._take_pci_delta(dl)
        return self._take_pci(res), delta

    def scan_pci_delta_reset(self):
        self._ck(self._lib.kvg_scan_pci_delta_reset(self._h))

    def scan_mdev_delta(self, recs: np.ndarray, raw_types: list):
        """scan_mdev plus the keyed diff against the previous scan_mdev_delta on this context -> (MdevResult,
        MdevDelta).  Types are compared by label.  Meaningful for canonical UUIDs and packed-BDF parents; with
        index-mode handles it is relative to the handles."""
        recs = np.ascontiguousarray(recs, dtype=L.MDEV_REC)
        td, keep = self._type_dict(raw_types)
        res = C.POINTER(L.MdevResultC)()
        dl = C.POINTER(L.MdevDeltaC)()
        self._ck(self._lib.kvg_scan_mdev_delta(self._h, recs.ctypes.data, len(recs), C.byref(td), C.byref(res),
                                               C.byref(dl)))
        del keep
        delta = self._take_mdev_delta(dl)
        return self._take_mdev(res), delta

    def _take_mdev_delta(self, dl) -> MdevDelta:
        d = dl.contents
        ng = int(d.n_type_gone)
        goff = L._arr(d.type_gone_off, ng + 1, np.uint32)
        gbytes = C.string_at(d.type_gone_bytes, int(goff[-1])) if ng and goff[-1] else b""
        delta = MdevDelta(int(d.n_prev), L._arr(d.changes, int(d.n_changes), L.MDEV_CHANGE),
                          L._arr(d.type_dirty, int(d.n_type_dirty), np.uint32),
                          [gbytes[goff[i]:goff[i + 1]] for i in range(ng)],
                          L._arr(d.par_dirty, int(d.n_par_dirty), np.uint32),
                          L._arr(d.par_gone, int(d.n_par_gone), np.uint32))
        self._lib.kvg_result_free(dl)
        return delta

    def scan_mdev_delta_reset(self):
        self._ck(self._lib.kvg_scan_mdev_delta_reset(self._h))

    # -- device-resident entry points (raw device pointers, e.g. torch tensor.data_ptr()) ----
    def text_pad(self, n: int) -> int:
        return int(self._lib.kvg_text_pad(n))

    def dev_pciids_parse(self, d_text: int, length: int, stride: int, n_files: int = 1):
        self._ck(self._lib.kvg_dev_pciids_parse(self._h, d_text, length, stride, n_files))

    def dev_scan_pci(self, d_recs: int, n: int):
        self._ck(self._lib.kvg_dev_scan_pci(self._h, d_recs, n))

    def dev_scan_pci_fetch(self) -> PciResult:
        res = C.POINTER(L.PciResultC)()
        self._ck(self._lib.kvg_dev_scan_pci_fetch(self._h, C.byref(res)))
        return self._take_pci(res)

    def dev_scan_pci_count(self):
        s, k, g = C.c_uint64(), C.c_uint32(), C.c_uint32()
        self._ck(self._lib.kvg_dev_scan_pci_count(self._h, C.byref(s), C.byref(k), C.byref(g)))
        return s.value, k.value, g.value

    def dev_gen_pci(self, d_recs: int, first: int, n: int, nv_ids: np.ndarray, group_bits: int = 0):
        ids = np.ascontiguousarray(nv_ids, dtype=np.uint16)
        self._ck(self._lib.kvg_dev_gen_pci(self._h, d_recs, first, n, ids.ctypes.data, len(ids),
                                           group_bits))

    def dev_gen_mdev(self, d_recs: int, first: int, n: int):
        self._ck(self._lib.kvg_dev_gen_mdev(self._h, d_recs, first, n))

    def dev_scan_mdev(self, d_recs: int, n: int, raw_types: list):
        td, keep = self._type_dict(raw_types)
        self._ck(self._lib.kvg_dev_scan_mdev(self._h, d_recs, n, C.byref(td)))
        del keep

    def dev_scan_mdev_fetch(self) -> MdevResult:
        res = C.POINTER(L.MdevResultC)()
        self._ck(self._lib.kvg_dev_scan_mdev_fetch(self._h, C.byref(res)))
        return self._take_mdev(res)

    def dev_flush_l2(self):
        self._ck(self._lib.kvg_dev_flush_l2(self._h))

    def set_kernel_timing(self, on: bool):
        self._ck(self._lib.kvg_set_kernel_timing(self._h, 1 if on else 0))

    def kernel_times(self, max_n: int = 4096):
        ms = (C.c_float * max_n)()
        names = C.create_string_buffer(64 * max_n)
        n = self._lib.kvg_kernel_times(self._h, ms, names, len(names), max_n)
        if n < 0:
            self._ck(n)
        parts = names.raw.split(b"\0")
        return [(parts[i].decode(), float(ms[i])) for i in range(n)]

    # -- multi-GPU --------------------------------------------------------------------------
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        rc = self._lib.kvg_comm_unique_id(buf)
        if rc != 0:
            raise L.KvgError(rc, (self._lib.kvg_last_error(None) or b"").decode())
        return buf.raw

    def comm_init(self, rank: int, nranks: int, uid: bytes):
        buf = C.create_string_buffer(uid, 128)
        self._ck(self._lib.kvg_comm_init(self._h, rank, nranks, buf))

    def comm_p2p_export(self, rank: int, nranks: int, cap_local: int) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(self._lib.kvg_comm_p2p_export(self._h, rank, nranks, cap_local, buf))
        return buf.raw

    def comm_p2p_import(self, all_handles: bytes):
        buf = C.create_string_buffer(all_handles, len(all_handles))
        self._ck(self._lib.kvg_comm_p2p_import(self._h, buf))

    def comm_p2p_enable(self, on: bool):
        self._ck(self._lib.kvg_comm_p2p_enable(self._h, 1 if on else 0))

    def comm_destroy(self):
        self._ck(self._lib.kvg_comm_destroy(self._h))

    def dev_scan_pci_sharded(self, d_recs: int, n_local: int):
        self._ck(self._lib.kvg_dev_scan_pci_sharded(self._h, d_recs, n_local))

    def dev_scan_pci_shard_fetch(self) -> PciShardResult:
        res = C.POINTER(L.PciShardResultC)()
        self._ck(self._lib.kvg_dev_scan_pci_shard_fetch(self._h, C.byref(res)))
        return self._take_pci_shard(res)

    def dev_scan_pci_shard_fetch_delta(self):
        """dev_scan_pci_shard_fetch plus this rank's share of the re-scan delta, against the previous successful call
        on this context -> (PciShardResult, PciDelta).  changes are the local shard's (indices into `local`),
        dev_dirty / grp_dirty index the owned keys (res.dev.dev_keys / res.grp.grp_keys), dev_gone / grp_gone are
        owned keys that went.  Not collective; kvgpu.merge_pci_shard_deltas fuses the ranks' parts."""
        res = C.POINTER(L.PciShardResultC)()
        dl = C.POINTER(L.PciDeltaC)()
        self._ck(self._lib.kvg_dev_scan_pci_shard_fetch_delta(self._h, C.byref(res), C.byref(dl)))
        delta = self._take_pci_delta(dl)
        return self._take_pci_shard(res), delta

    def dev_scan_pci_shard_delta_reset(self):
        self._ck(self._lib.kvg_dev_scan_pci_shard_delta_reset(self._h))

    def _take_pci_shard(self, res) -> PciShardResult:
        r = res.contents
        KD, G = int(r.n_dev_keys), int(r.n_groups)
        pool = C.string_at(r.name_pool, r.name_pool_len) if r.name_pool_len else b""
        e32, e16 = np.zeros(0, np.uint32), np.zeros(0, np.uint16)
        z32 = np.zeros(1, np.uint32)
        dev = PciResult(int(r.n_records), L._arr(r.dev_members, int(r.n_dev_members), L.PCI_SURV),
                        L._arr(r.dev_keys, KD, np.uint16), L._arr(r.dev_off, KD + 1, np.uint32),
                        L._arr(r.dev_perm, int(r.n_dev_members), np.uint32), L._arr(r.dev_name_slot, KD, np.uint32),
                        e32, z32, e32, pool)
        grp = PciResult(int(r.n_records), L._arr(r.grp_members, int(r.n_grp_members), L.PCI_SURV),
                        e16, z32, e32, e32, L._arr(r.grp_keys, G, np.uint32), L._arr(r.grp_off, G + 1, np.uint32),
                        L._arr(r.grp_perm, int(r.n_grp_members), np.uint32), pool)
        out = PciShardResult(int(r.n_records), L._arr(r.local, int(r.n_local), L.PCI_SURV), dev, grp)
        self._lib.kvg_result_free(res)
        return out

    def dev_scan_mdev_sharded(self, d_recs: int, n_local: int, raw_types: list):
        td, keep = self._type_dict(raw_types)
        self._ck(self._lib.kvg_dev_scan_mdev_sharded(self._h, d_recs, n_local, C.byref(td)))
        del keep

    def dev_scan_mdev_shard_fetch(self) -> MdevShardResult:
        res = C.POINTER(L.MdevShardResultC)()
        self._ck(self._lib.kvg_dev_scan_mdev_shard_fetch(self._h, C.byref(res)))
        return self._take_mdev_shard(res)

    def dev_scan_mdev_shard_fetch_delta(self):
        """dev_scan_mdev_shard_fetch plus this rank's share of the re-scan delta, against the previous successful call
        on this context -> (MdevShardResult, MdevDelta).  changes are the local shard's (indices into `local`),
        type_dirty / par_dirty index the owned keys (res.by_type.type_keys / res.by_parent.par_keys), type_gone
        (labels) / par_gone are owned keys that went; a label whose owner moved between the scans is gone on its old
        owner and dirty on its new one.  Not collective; kvgpu.merge_mdev_shard_deltas fuses the ranks' parts."""
        res = C.POINTER(L.MdevShardResultC)()
        dl = C.POINTER(L.MdevDeltaC)()
        self._ck(self._lib.kvg_dev_scan_mdev_shard_fetch_delta(self._h, C.byref(res), C.byref(dl)))
        delta = self._take_mdev_delta(dl)
        return self._take_mdev_shard(res), delta

    def dev_scan_mdev_shard_delta_reset(self):
        self._ck(self._lib.kvg_dev_scan_mdev_shard_delta_reset(self._h))

    def _take_mdev_shard(self, res) -> MdevShardResult:
        r = res.contents
        KT, NP, nt = int(r.n_type_keys), int(r.n_parents), int(r.n_types)
        loff = L._arr(r.label_off, nt + 1, np.uint32)
        noff = L._arr(r.type_name_off, nt + 1, np.uint32)
        lbytes = C.string_at(r.label_bytes, int(loff[-1])) if nt and loff[-1] else b""
        nbytes = C.string_at(r.type_name_bytes, int(noff[-1])) if nt and noff[-1] else b""
        labels = [lbytes[loff[i]:loff[i + 1]] for i in range(nt)]
        names = [nbytes[noff[i]:noff[i + 1]].decode("latin-1") for i in range(nt)]
        canon = L._arr(r.type_canon, nt, np.uint16)
        e32, e16, z32 = np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(1, np.uint32)
        by_type = MdevResult(int(r.n_records), L._arr(r.type_members, int(r.n_type_members), L.MDEV_SURV),
                             L._arr(r.type_keys, KT, np.uint16), L._arr(r.type_off, KT + 1, np.uint32),
                             L._arr(r.type_perm, int(r.n_type_members), np.uint32), labels, canon, names, e32, z32, e32)
        by_parent = MdevResult(int(r.n_records), L._arr(r.par_members, int(r.n_par_members), L.MDEV_SURV),
                               e16, z32, e32, labels, canon, names, L._arr(r.par_keys, NP, np.uint32),
                               L._arr(r.par_off, NP + 1, np.uint32), L._arr(r.par_perm, int(r.n_par_members), np.uint32))
        out = MdevShardResult(int(r.n_records), L._arr(r.local, int(r.n_local), L.MDEV_SURV), by_type, by_parent)
        self._lib.kvg_result_free(res)
        return out
