"""Host-side mirror of the reference's plugin interface for the scan path.

Same names, argument meaning and error behaviour as pkg/device_plugin/device_plugin.go, but the
filter / join / bucketing run in libkvgpu.so on the GPU:

    snapshot_pci_tree / snapshot_mdev_tree   the five sysfs readers (:294-357) turned into a flat
                                             record array (syscalls stay on the CPU, nothing is
                                             pre-filtered: read failures travel as flag bits)
    snapshot_mdev_ids                        the same readers over a fixed UUID list (the vGPU
                                             health re-scan)
    DiscoveryScan.create_iommu_device_map    createIommuDeviceMap  (:187-247)
    DiscoveryScan.create_vgpu_id_map         createVgpuIDMap       (:255-291)
    DiscoveryScan.get_device_name            getDeviceName         (:371-422)
    DiscoveryScan.create_device_plugins      the payload half of createDevicePlugins (:99-157):
                                             per key the pluginapi.Device list, resource name,
                                             socket path and env key the Go servers would use
    canonical_dump                           SURVEY.md 8c parity artefact

This module never imports the oracle and has no CPU implementation of the filter/join: without
libkvgpu.so and a CUDA device DiscoveryScan cannot be constructed.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

from . import _lib as L
from .context import Context, MdevResult, PciResult

HEXD = "0123456789abcdef"
DEVICE_NAMESPACE = "nvidia.com"                       # generic_device_plugin.go:51
DEVICE_PLUGIN_PATH = "/var/lib/kubelet/device-plugins/"  # pluginapi.DevicePluginPath
GPU_PREFIX = "PCI_RESOURCE_NVIDIA_COM"                # generic_device_plugin.go:57
VGPU_PREFIX = "MDEV_PCI_RESOURCE_NVIDIA_COM"          # generic_device_plugin.go:58
HEALTHY, UNHEALTHY = "Healthy", "Unhealthy"           # pluginapi constants


class ReferencePanic(RuntimeError):
    """The Go reference would panic on this sysfs content (e.g. data[2:] on a 1-byte file)."""


def format_bdf(p: int) -> str:
    return "%04x:%02x:%02x.%x" % (p >> 16, (p >> 8) & 0xFF, (p >> 3) & 0x1F, p & 7)


def parse_bdf(s: str):
    """'dddd:bb:dd.f' -> packed value, or None if `s` is not exactly that canonical form."""
    if len(s) != 12 or s[4] != ":" or s[7] != ":" or s[10] != ".":
        return None
    hx = s[0:4] + s[5:7] + s[8:10] + s[11]
    if any(c not in HEXD for c in hx):
        return None
    dom, bus, dev, fn = int(s[0:4], 16), int(s[5:7], 16), int(s[8:10], 16), int(s[11], 16)
    if dev > 31 or fn > 7:
        return None
    return (dom << 16) | (bus << 8) | (dev << 3) | fn


def format_uuid(u) -> str:
    h = bytes(u).hex()
    return "%s-%s-%s-%s-%s" % (h[0:8], h[8:12], h[12:16], h[16:20], h[20:32])


# ------------------------------------------------------------------------------------------------
# filepath.Walk + the five readers -> flat snapshot
# ------------------------------------------------------------------------------------------------
def _walk(root: str):
    """filepath.Walk order and Lstat semantics: yields (name, is_dir, err) for every visited
    entry; real directories are descended, symlinks are not followed."""
    try:
        st = os.lstat(root)
    except OSError:
        yield os.path.basename(root), False, True
        return
    import stat as _stat

    def rec(path, name, st):
        if not _stat.S_ISDIR(st.st_mode):
            yield name, False, False
            return
        try:
            names = sorted(os.listdir(path), key=lambda s: s.encode())
            err = False
        except OSError:
            names, err = [], True
        yield name, True, err
        if err:
            return
        for n in names:
            child = os.path.join(path, n)
            try:
                cst = os.lstat(child)
            except OSError:
                yield n, False, True
                return
            yield from rec(child, n, cst)

    yield from rec(root, os.path.basename(root), st)


def _read_raw(path, link: bool = False):
    """The contents of the file `path`, or the target of the link `path` (link=True), as read; None when the read
    fails."""
    try:
        if link:
            return os.readlink(path)
        with open(path, "rb") as f:
            return f.read()
    except OSError:
        return None


def _read_id(base, addr, prop):
    """readIDFromFileFunc :294-302 -> (string, err)"""
    data = _read_raw(os.path.join(base, addr, prop))
    if data is None:
        return "", True
    if len(data) < 2:
        raise ReferencePanic("slice bounds out of range reading %s/%s" % (addr, prop))
    return data[2:].strip(b"\n").decode("latin-1"), False


def _read_link(base, addr, link):
    """readLinkFunc :323-331 -> (basename, err)"""
    try:
        target = os.readlink(os.path.join(base, addr, link))
    except OSError:
        return "", True
    return target.rsplit("/", 1)[-1], False


# unicode.IsSpace (Go): NOT the same set as Python's str.strip() default
_GO_SPACE = "\t\n\v\f\r \u0085\u00a0\u1680\u2028\u2029\u202f\u205f\u3000" + "".join(
    chr(c) for c in range(0x2000, 0x200B))


def _read_numa(base, addr):
    """readNUMANodeFunc :304-320 -> (raw value, err).  The clamp (<0 -> 0) is left to the GPU."""
    data = _read_raw(os.path.join(base, addr, "numa_node"))
    if data is None:
        return 0, True
    try:
        s = data.decode("utf-8")
    except UnicodeDecodeError:
        s = data.decode("latin-1")
    s = s.strip(_GO_SPACE)  # strings.TrimSpace
    body = s[1:] if s[:1] in "+-" else s
    if not body or any(c not in "0123456789" for c in body):
        return 0, True
    v = int(s)
    if v < -(1 << 63) or v > (1 << 63) - 1:
        return 0, True
    return v, False


@dataclass
class PciSnapshot:
    recs: np.ndarray
    names: list            # Walk-order entry names (record i <-> names[i])
    packed_addr: bool      # True: recs.addr is the packed BDF; False: the Walk index
    group_names: list | None   # None: iommu_group is the number itself; else interned strings
    device_names: list | None = None   # None: recs.device is the id itself ("%04x"); else interned `device` strings


def _read_pci_entry(base_path: str, name: str):
    """What the readers of createIommuDeviceMap's walk callback return for one entry -> (vendor, device, group,
    driver, flags, numa); `device` and `group` are the strings read, or 0 / "" when they were not read."""
    flags, vendor, device, group, driver, numa = 0, 0xFFFF, 0, "", L.DRV_NONE, 0
    v, e = _read_id(base_path, name, "vendor")
    if e:
        flags |= L.PF_VENDOR_ERR
    elif len(v) == 4 and all(c in HEXD for c in v):
        vendor = int(v, 16)
    if not e and v == "10de":
        # same short-circuit order as :212-238 — a later file is only touched when the
        # reference would touch it (so a panic can only happen where the reference panics)
        d, e = _read_link(base_path, name, "driver")
        if e:
            flags |= L.PF_DRIVER_ERR
        else:
            driver = {"vfio-pci": L.DRV_VFIO_PCI,
                      "nvgrace_gpu_vfio_pci": L.DRV_NVGRACE}.get(d, L.DRV_OTHER)
        if not e and driver in (L.DRV_VFIO_PCI, L.DRV_NVGRACE):
            group, e = _read_link(base_path, name, "iommu_group")
            if e:
                flags |= L.PF_IOMMU_ERR
            else:
                numa, e = _read_numa(base_path, name)
                if e:
                    flags |= L.PF_NUMA_ERR
                dv, e = _read_id(base_path, name, "device")
                if e:
                    flags |= L.PF_DEVICE_ERR
                else:
                    device = dv   # the reference keeps WHATEVER the file holds as the map key (:240, :294-302)
    return vendor, device, group, driver, flags, numa


def _pci_records(names, rows, ascending: bool, group_of):
    """The records of the entries `names` from what _read_pci_entry returned for each (rows) -> (recs, packed_addr,
    device_names).  addr is the packed BDF when every name parses (and the values ascend, if `ascending`), else the
    index; group_of(group string) -> the group handle.  `device`: "%04x" strings travel as the number; anything else
    switches the column to index mode (interned strings, like the groups): the GPU groups by the interned id, the host
    keeps the strings and asks getDeviceName with the exact bytes."""
    packed = [parse_bdf(n) for n in names]
    packed_ok = all(p is not None for p in packed) and (
        not ascending or all(packed[i] < packed[i + 1] for i in range(len(packed) - 1)))
    devices_numeric = all(len(r[1]) == 4 and all(c in HEXD for c in r[1]) for r in rows if isinstance(r[1], str))
    dintern = {}
    recs = np.zeros(len(rows), dtype=L.PCI_REC)
    for i, (vendor, device, group, driver, flags, numa) in enumerate(rows):
        if isinstance(device, str):
            if devices_numeric:
                device = int(device, 16)
            else:
                device = dintern.setdefault(device, len(dintern))
                if device > 0xFFFF:
                    raise L.KvgError(L.KVG_ERANGE, "more than 65536 distinct non-canonical device strings")
        if not -32768 <= numa <= 32767:
            raise L.KvgError(L.KVG_ERANGE, "numa_node %d of %s does not fit int16" % (numa, names[i]))
        recs[i] = (packed[i] if packed_ok else i, vendor, device, group_of(group), driver, flags, numa)
    return recs, packed_ok, None if devices_numeric else list(dintern)


def snapshot_pci_tree(base_path: str) -> PciSnapshot:
    """Walk `base_path` like createIommuDeviceMap and record what each reader returned."""
    rows, names = [], []
    for name, is_dir, err in _walk(base_path):
        if err:      # :193-196 the walk aborts; entries seen so far stay
            break
        if is_dir:   # :197-200
            continue
        rows.append(_read_pci_entry(base_path, name))
        names.append(name)

    def canon_dec(s):
        return s.isdigit() and s.isascii() and (s == "0" or s[0] != "0") and int(s) < (1 << 32)

    # groups: the number itself when every group read is canonical decimal, else strings interned from 0
    if all(canon_dec(r[2]) for r in rows if r[2] != ""):
        intern, group_of = None, lambda g: int(g) if g else 0
    else:
        intern = {}
        group_of = lambda g: intern.setdefault(g, len(intern)) if g else 0   # noqa: E731
    recs, packed_ok, device_names = _pci_records(names, rows, True, group_of)
    return PciSnapshot(recs, names, packed_ok, None if intern is None else list(intern), device_names)


@dataclass
class PciRaw:
    """What the readers of createIommuDeviceMap's walk callback got, undecoded (include/kvgpu.h kvg_pci_raw): field f of
    entry i is bytes[off[i * RAW_FIELDS + f]:off[i * RAW_FIELDS + f + 1]]; state[i] bit f: read f was made, bit 8 + f:
    it failed.  names: the Walk-order entry names."""
    names: list
    off: np.ndarray     # u32 [n * RAW_FIELDS + 1]
    bytes: bytes
    state: np.ndarray   # u16 [n]


def read_pci_tree_raw(base_path: str) -> PciRaw:
    """The walk of snapshot_pci_tree with all five reads made for every entry and nothing decoded: file contents as
    read, link targets as os.readlink returns them.  Reading what the reference would not reach is allowed: the GPU
    decodes only what it reaches, so no panic is raised here."""
    names = []
    for name, is_dir, err in _walk(base_path):
        if err:
            break
        if not is_dir:
            names.append(name)
    return read_pci_ids_raw(base_path, names)


def _read_pci_entry_raw(bbase: bytes, name: str):
    """The five reads of one entry, raw -> (fields: name, vendor, driver target, iommu_group target, numa_node, device;
    state bits)."""
    bname = os.fsencode(name)
    st, row = 0, [bname]
    for f, prop in ((L.RAW_VENDOR, b"vendor"), (L.RAW_DRIVER, b"driver"), (L.RAW_GROUP, b"iommu_group"),
                    (L.RAW_NUMA, b"numa_node"), (L.RAW_DEVICE, b"device")):
        data = _read_raw(os.path.join(bbase, bname, prop), f in (L.RAW_DRIVER, L.RAW_GROUP))
        st |= 1 << f | (1 << (8 + f) if data is None else 0)
        row.append(data or b"")
    return row, st


def read_pci_ids_raw(base_path: str, names) -> PciRaw:
    """The reads of read_pci_tree_raw for the entries `names` in THAT order (a health re-scan's advertised devices,
    any form of name; an entry that is gone reads as failed reads)."""
    names, fields, state = list(names), [], []
    bbase = os.fsencode(base_path)
    for name in names:
        row, st = _read_pci_entry_raw(bbase, name)
        fields += row
        state.append(st)
    return PciRaw(names, *_pack_raw(fields, state, "the raw reads of %s" % base_path))


def list_nodes_raw(device_path: str) -> list:
    """One listing of the VFIO device directory (/dev/vfio, generic_device_plugin.go:611-690) as the names' bytes, in
    listing order: every name, `vfio` and `devices` included; a missing directory means no node exists."""
    try:
        return os.listdir(os.fsencode(device_path))
    except FileNotFoundError:
        return []


def _pack_raw(fields, state, what: str):
    """Byte fields, entry after entry, and the read bits of each entry (bit f: read f was made, bit 8 + f: it failed)
    -> (u32 offsets, the fields joined, u16 state): field j is bytes[off[j]:off[j + 1]]."""
    off = np.zeros(len(fields) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in fields], out=off[1:])
    if off[-1] > 0xFFFFFFFF:
        raise ValueError("%s exceed 4 GiB" % what)
    return off.astype(np.uint32), b"".join(fields), np.array(state, dtype=np.uint16)


NOT_READ = "not read"   # a read that was not made (pack_alloc_raw); the library refuses one the reference reaches


@dataclass
class AllocRaw:
    """The raw reads of one AllocateRequest (include/kvgpu.h kvg_alloc_raw), undecoded.  n_members / n_ids: one count
    per container request; member_off / member_bytes / member_state: per member the iommu_group link target, the
    vendor contents and the group string the maps hold; id_off / id_bytes: the DevicesIDs; egm_off / egm_bytes /
    egm_state: per EGM class entry its name and gpu_devices contents, and the made / failed bits of both reads and of
    the Stat of its device node."""
    n_members: np.ndarray   # u32 [n_reqs]
    n_ids: np.ndarray       # u32 [n_reqs]
    member_off: np.ndarray  # u32 [n * AMEM_FIELDS + 1]
    member_bytes: bytes
    member_state: np.ndarray  # u16 [n]
    id_off: np.ndarray      # u32 [n_ids + 1]
    id_bytes: bytes
    egm_off: np.ndarray     # u32 [n_egm * AEGM_FIELDS + 1]
    egm_bytes: bytes
    egm_state: np.ndarray   # u16 [n_egm]


def pack_alloc_raw(requests, egm_entries) -> AllocRaw:
    """requests: [(members, ids)] in request order, members = [(link target, vendor contents, group string)] in the
    order the reference visits them, ids = the DevicesIDs; egm_entries: [(name, gpu_devices contents, stat ok)] in
    ReadDir order.  A read is bytes (what it returned), None (it failed) or NOT_READ; a stat is True (it succeeded),
    False (it failed) or NOT_READ.  Strings are encoded with os.fsencode, the bytes Go holds for them."""
    enc = lambda v: os.fsencode(v) if isinstance(v, str) else v   # noqa: E731
    mparts, mstate, iparts, n_members, n_ids = [], [], [], [], []
    for members, ids in requests:
        for link, vendor, group in members:
            st = 0
            for f, v in ((L.AMEM_LINK, link), (L.AMEM_VENDOR, vendor)):
                if v is not NOT_READ:
                    st |= 1 << f
                    if v is None:
                        st |= 1 << (8 + f)
            mparts += [enc(link) if isinstance(link, (bytes, str)) else b"",
                       enc(vendor) if isinstance(vendor, (bytes, str)) else b"", enc(group)]
            mstate.append(st)
        iparts += [enc(b) for b in ids]
        n_members.append(len(members))
        n_ids.append(len(ids))
    eparts, estate = [], []
    for name, gpus, stat in egm_entries:
        st = 0
        if gpus is not NOT_READ:
            st |= 1 << L.AEGM_GPUS | (1 << (8 + L.AEGM_GPUS) if gpus is None else 0)
        if stat is not NOT_READ:
            st |= 1 << L.AEGM_STAT | (0 if stat else 1 << (8 + L.AEGM_STAT))
        eparts += [enc(name), enc(gpus) if isinstance(gpus, (bytes, str)) else b""]
        estate.append(st)
    what = "the raw reads"
    return AllocRaw(np.array(n_members, dtype=np.uint32), np.array(n_ids, dtype=np.uint32),
                    *_pack_raw(mparts, mstate, what), *_pack_raw(iparts, (), what)[:2],
                    *_pack_raw(eparts, estate, what))


@dataclass
class AllocRespIn:
    """The plan and the vfio-dev listings of one AllocateRequest (include/kvgpu.h kvg_alloc_resp_in): iommufd, then
    per request the visited DevicesIDs and the lookup error after them, per visited ID its member count, per member
    dev.addr, its listing's entries (name, IsDir) and the listing's made / failed bits."""
    iommufd: int
    n_visited: np.ndarray   # u32 [n_reqs]
    lookup_error: np.ndarray  # u8 [n_reqs]
    id_members: np.ndarray  # u32 [visited IDs]
    addr_off: np.ndarray    # u32 [n + 1]
    addr_bytes: bytes
    vfio_first: np.ndarray  # u32 [n + 1]
    vfio_off: np.ndarray    # u32 [entries + 1]
    vfio_bytes: bytes
    vfio_dir: np.ndarray    # u8 [entries]
    vfio_state: np.ndarray  # u8 [n]


def pack_alloc_response(requests, egm_entries, iommufd: bool):
    """requests: [(ids, visits, lookup_error)] in request order: ids = the DevicesIDs, visits = per visited ID its
    members in map order, each (addr, link target, vendor contents, group string, listing), lookup_error = the ID after
    the visited ones misses the maps.  A listing is [(name, is_dir)] in any order, None (os.ReadDir failed) or
    NOT_READ; the other reads as pack_alloc_raw takes them.  -> (AllocRaw, AllocRespIn)."""
    enc = lambda v: os.fsencode(v) if isinstance(v, str) else v   # noqa: E731
    raw_reqs, n_visited, lookup, id_members, addrs, first, names, dirs, state = [], [], [], [], [], [0], [], [], []
    for ids, visits, lookup_error in requests:
        members = []
        for visit in visits:
            id_members.append(len(visit))
            for addr, link, vendor, group, listing in visit:
                members.append((link, vendor, group))
                addrs.append(enc(addr))
                if listing is NOT_READ:
                    state.append(0)
                elif listing is None:
                    state.append(L.AVFIO_MADE | L.AVFIO_FAILED)
                else:
                    state.append(L.AVFIO_MADE)
                    for name, is_dir in listing:
                        names.append(enc(name))
                        dirs.append(1 if is_dir else 0)
                first.append(len(names))
        raw_reqs.append((members, list(ids)))
        n_visited.append(len(visits))
        lookup.append(1 if lookup_error else 0)
    what = "the raw reads"
    aoff, ab, _ = _pack_raw(addrs, (), what)
    voff, vb, _ = _pack_raw(names, (), what)
    return pack_alloc_raw(raw_reqs, egm_entries), AllocRespIn(
        1 if iommufd else 0, np.array(n_visited, dtype=np.uint32), np.array(lookup, dtype=np.uint8),
        np.array(id_members, dtype=np.uint32), aoff, ab, np.array(first, dtype=np.uint32), voff, vb,
        np.array(dirs, dtype=np.uint8), np.array(state, dtype=np.uint8))


def snapshot_pci_ids(base_path: str, bdfs, intern: dict) -> PciSnapshot:
    """Snapshot the PCI devices `bdfs` in THAT order (the health re-scan's fixed record order; a Walk would re-index
    when one vanishes), with the readers and flag rules of snapshot_pci_tree.  An address whose entry is gone reads as
    a vendor error, so its record fails the filter.

    Group strings become handles through `intern`, a dict the caller keeps across snapshots (handles from 1; 0 = no
    group), so a group keeps its handle and a VFIO node name resolves through the same dict (group_nodes).  names =
    bdfs; group_names[h] = the string of handle h; addr is the packed BDF when every address parses, else the index.
    The `device` column follows snapshot_pci_tree: "%04x" strings as the number, otherwise interned strings."""
    names = list(bdfs)
    rows = [_read_pci_entry(base_path, name) for name in names]
    recs, packed_ok, device_names = _pci_records(names, rows, False,
                                                 lambda g: intern.setdefault(g, len(intern) + 1) if g else 0)
    return PciSnapshot(recs, names, packed_ok, [""] + sorted(intern, key=intern.get), device_names)


def group_nodes(device_path: str, intern: dict) -> np.ndarray:
    """The handles (from `intern`, as snapshot_pci_ids assigns them) of the IOMMU groups whose VFIO node exists under
    `device_path` (/dev/vfio/<group>, generic_device_plugin.go:611-690), ascending.  Other names (`vfio`, `devices`,
    groups no snapshot has seen) can match no record and are left out; a missing directory means no node exists."""
    try:
        entries = os.listdir(device_path)
    except FileNotFoundError:
        entries = []
    return np.array(sorted(intern[e] for e in entries if e in intern), dtype=np.uint32)


def _read_vgpu_raw(base, addr, prop):
    data = _read_raw(os.path.join(base, addr, prop))
    return (None, True) if data is None else (data, False)


def _read_gpu_id_for_vgpu(base, addr):
    """readGpuIDForVgpuFunc :347-357"""
    try:
        target = os.readlink(os.path.join(base, addr))
    except OSError:
        return "", True
    parts = target.split("/")
    if len(parts) < 2:
        raise ReferencePanic("index out of range splitting link target %r" % target)
    return parts[-2].strip("\n"), False


def _uuid_bytes(s: str):
    """The 16 bytes of `s` when it is a UUID in canonical form (lower-case 8-4-4-4-12 hex), else None."""
    h = s.replace("-", "")
    if len(s) == 36 and len(h) == 32 and all(c in HEXD for c in h) and format_uuid(bytes.fromhex(h)) == s:
        return bytes.fromhex(h)
    return None


def _read_mdev_entry(vgpu_base: str, pci_base: str, name: str, type_ids: dict):
    """What the readers of createVgpuIDMap's walk callback return for one entry -> (type index, parent, flags, numa):
    the type file, then the parent link only when the type read succeeded (:275), then the parent's numa_node only when
    the link read succeeded.  A type file content not in `type_ids` (content -> index) gets the next index."""
    flags, tidx, parent, numa = 0, 0, "", 0
    raw, e = _read_vgpu_raw(vgpu_base, name, "mdev_type/name")
    if e:
        flags |= L.MF_TYPE_ERR
    else:
        tidx = type_ids.setdefault(raw, len(type_ids))
        parent, e = _read_gpu_id_for_vgpu(vgpu_base, name)
        if e:
            flags |= L.MF_PARENT_ERR
        else:
            numa, e = _read_numa(pci_base, parent)
            if e:
                flags |= L.MF_NUMA_ERR
    return tidx, parent, flags, numa


@dataclass
class MdevSnapshot:
    recs: np.ndarray
    names: list
    raw_types: list            # raw mdev_type/name contents (bytes), dictionary order
    parent_names: list | None  # None: parent is a packed BDF; else interned strings
    uuid_ok: bool


def snapshot_mdev_tree(vgpu_base: str, pci_base: str) -> MdevSnapshot:
    rows, names, type_ids = [], [], {}
    for name, is_dir, err in _walk(vgpu_base):
        if err:
            break
        if is_dir:
            continue
        rows.append(_read_mdev_entry(vgpu_base, pci_base, name, type_ids))
        names.append(name)
    ppacked = [parse_bdf(r[1]) for r in rows if r[1] != ""]
    parents_packed = all(p is not None for p in ppacked)
    parent_names, intern = (None, None) if parents_packed else ([], {})
    ub = [_uuid_bytes(n) for n in names]
    uuid_ok = all(u is not None for u in ub) and all(ub[i] < ub[i + 1] for i in range(len(ub) - 1))
    recs = np.zeros(len(rows), dtype=L.MDEV_REC)
    for i, (tidx, parent, flags, numa) in enumerate(rows):
        if parent == "":
            p = 0
        elif parents_packed:
            p = parse_bdf(parent)
        else:
            p = intern.setdefault(parent, len(intern))
            if p == len(parent_names):
                parent_names.append(parent)
        if uuid_ok:
            recs[i]["uuid"] = np.frombuffer(ub[i], dtype=np.uint8)
        else:
            recs[i]["uuid"][:4] = np.frombuffer(int(i).to_bytes(4, "big"), dtype=np.uint8)
        recs[i]["parent"], recs[i]["type_idx"], recs[i]["flags"] = p, tidx, flags
        recs[i]["parent_numa"] = numa
    return MdevSnapshot(recs, names, list(type_ids), parent_names, uuid_ok)


@dataclass
class MdevRaw:
    """What the readers of createVgpuIDMap's walk callback got, undecoded (include/kvgpu.h kvg_mdev_raw): field f of
    entry i is bytes[off[i * MRAW_FIELDS + f]:off[i * MRAW_FIELDS + f + 1]] (name, mdev_type/name contents, the entry's
    link target, the parent's numa_node contents); state[i] bit f: read f was made, bit 8 + f: it failed.
    names: the Walk-order entry names."""
    names: list
    off: np.ndarray     # u32 [n * MRAW_FIELDS + 1]
    bytes: bytes
    state: np.ndarray   # u16 [n]


def mdev_numa_parent(target: bytes):
    """The parent component readGpuIDForVgpuFunc (:347-357) takes from a link target -- strings.Split(target, "/")
    [len-2] with Trim "\n" -- which names the numa_node file to read; None where the reference panics (no '/')."""
    parts = target.split(b"/")
    return None if len(parts) < 2 else parts[-2].strip(b"\n")


def read_mdev_tree_raw(vgpu_base: str, pci_base: str) -> MdevRaw:
    """The walk of snapshot_mdev_tree with every read it can make and nothing decoded: the type file as read, the link
    target as os.readlink returns it, and <pci_base>/<parent>/numa_node for the parent of that target (not made when
    the link is unreadable or has no '/').  The GPU decodes only what the reference reaches."""
    names = []
    for name, is_dir, err in _walk(vgpu_base):
        if err:
            break
        if not is_dir:
            names.append(name)
    return read_mdev_ids_raw(vgpu_base, pci_base, names)


def _read_mdev_entry_raw(vbase: bytes, pbase: bytes, name: str):
    """The reads of one mdev entry, raw -> (fields: name, mdev_type/name, link target, parent numa_node; state bits)."""
    bname = os.fsencode(name)
    st, row = 0, [bname, b"", b"", b""]

    def take(f, path, link=False):
        nonlocal st
        data = _read_raw(path, link)
        st |= 1 << f | (1 << (8 + f) if data is None else 0)
        row[f] = data or b""

    take(L.MRAW_TYPE, os.path.join(vbase, bname, b"mdev_type", b"name"))
    take(L.MRAW_LINK, os.path.join(vbase, bname), link=True)
    parent = mdev_numa_parent(row[L.MRAW_LINK]) if not (st >> (8 + L.MRAW_LINK)) & 1 else None
    if parent is not None:
        take(L.MRAW_NUMA, os.path.join(pbase, parent, b"numa_node"))
    return row, st


def read_mdev_ids_raw(vgpu_base: str, pci_base: str, names) -> MdevRaw:
    """The reads of read_mdev_tree_raw for the entries `names` in THAT order (a health re-scan's advertised vGPUs, any
    form of name; an entry that is gone reads as a failed type read)."""
    names, fields, state = list(names), [], []
    vbase, pbase = os.fsencode(vgpu_base), os.fsencode(pci_base)
    for name in names:
        row, st = _read_mdev_entry_raw(vbase, pbase, name)
        fields += row
        state.append(st)
    return MdevRaw(names, *_pack_raw(fields, state, "the raw reads of %s" % vgpu_base))


def snapshot_mdev_ids(vgpu_base: str, pci_base: str, uuids, intern: dict) -> MdevSnapshot:
    """Snapshot the mdevs `uuids` in THAT order (the health re-scan's fixed record order; a Walk would re-index when
    one vanishes, which is the very event health has to see), with the readers and flag rules of snapshot_mdev_tree.
    A UUID whose entry is gone reads as a type error, so its record is absent.

    Parent strings become handles through `intern`, a dict the caller keeps across snapshots (handles from 1; 0 = no
    parent), so a GPU keeps its handle and an NVML bus id resolves through the same dict.  names = uuids,
    parent_names[h] = the string of handle h."""
    uuids = list(uuids)
    recs = np.zeros(len(uuids), dtype=L.MDEV_REC)
    type_ids, uuid_ok = {}, True
    for i, name in enumerate(uuids):
        tidx, parent, flags, numa = _read_mdev_entry(vgpu_base, pci_base, name, type_ids)
        if not -32768 <= numa <= 32767:
            raise L.KvgError(L.KVG_ERANGE, "numa_node %d of %s does not fit int16" % (numa, parent))
        h = intern.setdefault(parent, len(intern) + 1) if parent else 0
        u = _uuid_bytes(name)
        if u is not None:
            recs[i]["uuid"] = np.frombuffer(u, dtype=np.uint8)
        else:
            uuid_ok = False
            recs[i]["uuid"][:4] = np.frombuffer(int(i).to_bytes(4, "big"), dtype=np.uint8)
        recs[i]["parent"], recs[i]["type_idx"], recs[i]["flags"], recs[i]["parent_numa"] = h, tidx, flags, numa
    return MdevSnapshot(recs, uuids, list(type_ids), [""] + sorted(intern, key=intern.get), uuid_ok)


# ------------------------------------------------------------------------------------------------
# the five maps rebuilt from flat GPU results
# ------------------------------------------------------------------------------------------------
@dataclass
class NvidiaGpuDevice:      # device_plugin.go:50-53
    addr: str
    numaNode: int


@dataclass
class Maps:
    iommuMap: dict = field(default_factory=dict)       # :56
    deviceMap: dict = field(default_factory=dict)      # :59
    bdfToIommuMap: dict = field(default_factory=dict)  # :62
    vGpuMap: dict = field(default_factory=dict)        # :65
    gpuVgpuMap: dict = field(default_factory=dict)     # :68
    deviceNames: dict = field(default_factory=dict)    # key -> getDeviceName(key) ("" = miss)


def pci_maps_from_result(res: PciResult, snap: PciSnapshot | None = None, maps: Maps | None = None,
                         name_of=None) -> Maps:
    """name_of(key) -> getDeviceName(key): needed (and only used) when the snapshot carries the `device`
    strings in index mode — the GPU's per-survivor join is keyed by the numeric id and does not apply."""
    return _pci_maps(maps or Maps(), res, res, res.survivors, snap, name_of)


def _pci_maps(m: Maps, dev: PciResult, grp: PciResult, local: np.ndarray, snap: PciSnapshot | None = None,
              name_of=None) -> Maps:
    """New deviceMap, iommuMap and bdfToIommuMap dicts in `m`: every key of `dev` and of `grp` (_put_pci_keys), and
    the survivors `local` in their order."""
    m.iommuMap, m.deviceMap, m.bdfToIommuMap = {}, {}, {}  # :188-190
    _put_pci_keys(m, dev, grp, range(len(dev.dev_keys)), range(len(grp.grp_keys)), snap, name_of)
    addr_of, _, grp_of = _pci_names(snap)
    for a, g in zip(local["addr"], local["iommu_group"]):
        m.bdfToIommuMap[addr_of(int(a))] = grp_of(g)
    return m


@dataclass
class PciMapsTouched:
    """The deviceMap / iommuMap keys apply_pci_delta rewrote (dirty: present now, new ones included) or removed."""
    dev_dirty: list
    dev_gone: list
    grp_dirty: list
    grp_gone: list


def _fully_numeric(snap: PciSnapshot | None) -> bool:
    return snap is None or (snap.packed_addr and snap.group_names is None and snap.device_names is None)


def _rebuild_into(maps: Maps, build) -> PciMapsTouched:
    """build(maps) rebuilds the PCI maps in `maps`; reports every key of the new maps and every key that went."""
    before_dev, before_grp = set(maps.deviceMap), set(maps.iommuMap)
    build(maps)
    return PciMapsTouched(list(maps.deviceMap), sorted(before_dev - set(maps.deviceMap)),
                          list(maps.iommuMap), sorted(before_grp - set(maps.iommuMap)))


def _rebuild_pci_maps(maps: Maps, res: PciResult, snap, name_of) -> PciMapsTouched:
    """pci_maps_from_result into `maps`, reporting every key of the new maps and every key that went."""
    return _rebuild_into(maps, lambda m: pci_maps_from_result(res, snap, m, name_of=name_of))


def _pci_names(snap: PciSnapshot | None):
    """The strings behind a snapshot's handles: (address, device key, group) of a handle; None is fully numeric."""
    addr = format_bdf if snap is None or snap.packed_addr else (lambda a: snap.names[int(a)])
    dev = (lambda d: "%04x" % int(d)) if snap is None or snap.device_names is None else \
        (lambda d: snap.device_names[int(d)])
    grp = (lambda g: str(int(g))) if snap is None or snap.group_names is None else (lambda g: snap.group_names[int(g)])
    return addr, dev, grp


def _put_pci_keys(maps: Maps, dev: PciResult, grp: PciResult, dev_ks, grp_ks, snap: PciSnapshot | None = None,
                  name_of=None) -> tuple:
    """Set the deviceMap key dev.dev_keys[k] and its deviceNames entry for every k of dev_ks, and the iommuMap key
    grp.grp_keys[k] for every k of grp_ks (each result's permutation indexes its own survivors), named through `snap`
    (None is fully numeric) -> (the device keys, the group keys) set, in that order."""
    addr_of, dev_of, grp_of = _pci_names(snap)
    dev_index = snap is not None and snap.device_names is not None
    if dev_index and name_of is None:
        raise ValueError("snapshot carries device strings in index mode: pass name_of (Context.name_lookup)")

    def members(res, perm, off, k):
        s = res.survivors[perm[off[k]:off[k + 1]]]
        return [NvidiaGpuDevice(addr_of(a), n) for a, n in zip(s["addr"].tolist(), s["numa"].tolist())]

    dev_keys, grp_keys = [], []
    for k in dev_ks:
        key = dev_of(dev.dev_keys[k])
        maps.deviceMap[key] = members(dev, dev.dev_perm, dev.dev_off, k)
        maps.deviceNames[key] = name_of(key) if dev_index else dev.name_at(int(dev.dev_name_slot[k]))
        dev_keys.append(key)
    for k in grp_ks:
        key = grp_of(grp.grp_keys[k])
        maps.iommuMap[key] = members(grp, grp.grp_perm, grp.grp_off, k)
        grp_keys.append(key)
    return dev_keys, grp_keys


def _patch_pci_maps(maps: Maps, dev: PciResult, grp: PciResult, delta, snap: PciSnapshot | None = None,
                    prev_snap: PciSnapshot | None = None, name_of=None) -> PciMapsTouched:
    """The patch of apply_pci_delta: deviceMap keys from `dev`, iommuMap keys from `grp` (_put_pci_keys),
    bdfToIommuMap from the changes.  Handles of the new side are named through `snap`, those of the previous side
    (removed addresses, gone keys) through `prev_snap`; None is a numeric snapshot."""
    addr_of, _, grp_of = _pci_names(snap)
    prev_addr_of, prev_dev_of, prev_grp_of = _pci_names(prev_snap)
    dev_dirty, grp_dirty = _put_pci_keys(maps, dev, grp, delta.dev_dirty, delta.grp_dirty, snap, name_of)
    t = PciMapsTouched(dev_dirty, [prev_dev_of(d) for d in delta.dev_gone], grp_dirty,
                       [prev_grp_of(g) for g in delta.grp_gone])
    for key in t.dev_gone:
        maps.deviceMap.pop(key, None)
        maps.deviceNames.pop(key, None)
    for key in t.grp_gone:
        maps.iommuMap.pop(key, None)
    for c in delta.changes:
        if c["what"] & L.CH_REMOVED:
            maps.bdfToIommuMap.pop(prev_addr_of(int(c["addr"])), None)
        else:
            maps.bdfToIommuMap[addr_of(int(c["addr"]))] = grp_of(c["now_group"])
    return t


def apply_pci_delta(maps: Maps, res: PciResult, delta, snap: PciSnapshot | None = None,
                    prev_snap: PciSnapshot | None = None, name_of=None) -> PciMapsTouched:
    """Patch deviceMap, iommuMap and bdfToIommuMap of `maps` (built from the previous delta scan's result) into
    what pci_maps_from_result(res) builds, touching only dirty or gone keys and changed addresses.  A delta keyed by
    entry name (Context.scan_pci_raw_delta) is patched in every snapshot mode, naming each side's handles through
    its own snapshot.  Otherwise a snapshot that is not fully numeric (index-mode addresses, groups or device strings)
    has no stable handles: the maps are then rebuilt and every key is reported."""
    if getattr(delta, "by_name", False):
        return _patch_pci_maps(maps, res, res, delta, snap, prev_snap, name_of)
    if not (_fully_numeric(snap) and _fully_numeric(prev_snap)):
        return _rebuild_pci_maps(maps, res, snap, name_of)
    return _patch_pci_maps(maps, res, res, delta)


def mdev_maps_from_result(res: MdevResult, snap: MdevSnapshot | None = None, maps: Maps | None = None) -> Maps:
    return _mdev_maps(maps or Maps(), res, res, snap)


def _mdev_maps(m: Maps, by_type: MdevResult, by_par: MdevResult, snap: MdevSnapshot | None = None) -> Maps:
    """New vGpuMap and gpuVgpuMap dicts in `m`: every key of `by_type` and of `by_par` (_put_mdev_keys)."""
    m.vGpuMap, m.gpuVgpuMap = {}, {}  # :256-257
    _put_mdev_keys(m, by_type, by_par, range(len(by_type.type_keys)), range(len(by_par.par_keys)), snap)
    return m


@dataclass
class MdevMapsTouched:
    """The vGpuMap / gpuVgpuMap keys apply_mdev_delta rewrote (dirty: present now, new ones included) or removed."""
    type_dirty: list
    type_gone: list
    par_dirty: list
    par_gone: list


def _numeric_mdev(snap: MdevSnapshot | None) -> bool:
    return snap is None or (snap.uuid_ok and snap.parent_names is None)


def _rebuild_mdev_maps(maps: Maps, by_type: MdevResult, by_par: MdevResult, snap) -> MdevMapsTouched:
    """_mdev_maps into the dicts `maps` already holds (they are shared), reporting every key of the new maps and
    every key that went."""
    fresh = _mdev_maps(Maps(), by_type, by_par, snap)
    type_gone = sorted(set(maps.vGpuMap) - set(fresh.vGpuMap))
    par_gone = sorted(set(maps.gpuVgpuMap) - set(fresh.gpuVgpuMap))
    for label in type_gone:
        if label not in maps.deviceMap:
            maps.deviceNames.pop(label, None)
    maps.vGpuMap.clear()
    maps.vGpuMap.update(fresh.vGpuMap)
    maps.gpuVgpuMap.clear()
    maps.gpuVgpuMap.update(fresh.gpuVgpuMap)
    maps.deviceNames.update(fresh.deviceNames)
    return MdevMapsTouched(list(fresh.vGpuMap), type_gone, list(fresh.gpuVgpuMap), par_gone)


def apply_mdev_delta(maps: Maps, res: MdevResult, delta, snap: MdevSnapshot | None = None,
                     prev_snap: MdevSnapshot | None = None) -> MdevMapsTouched:
    """Patch vGpuMap, gpuVgpuMap and the label entries of deviceNames of `maps` (built from the previous delta scan's
    result) IN PLACE into what mdev_maps_from_result(res) builds, touching only dirty or gone keys: whoever holds
    maps.gpuVgpuMap (XidEventRouter) sees the new vGPUs.  A snapshot whose UUIDs are not canonical or whose parents are
    not packed BDFs has no stable handles: the maps are then rebuilt (in place as well) and every key is reported.  A
    delta keyed by entry name (Context.scan_mdev_raw_delta) is patched in every snapshot mode, naming each side's
    UUIDs and parents through its own snapshot."""
    if getattr(delta, "by_name", False):
        return _patch_mdev_maps(maps, res, res, delta, snap, prev_snap)
    if not (_numeric_mdev(snap) and _numeric_mdev(prev_snap)):
        return _rebuild_mdev_maps(maps, res, res, snap)
    return _patch_mdev_maps(maps, res, res, delta)


def _mdev_names(snap: MdevSnapshot | None):
    """(UUIDs of the survivors s, parent key of a handle) of a snapshot; None is fully numeric"""
    uids = (lambda s: [format_uuid(u) for u in s["uuid"]]) if snap is None or snap.uuid_ok else \
        (lambda s: [snap.names[i] for i in s["src"].tolist()])
    par = (lambda p: format_bdf(int(p))) if snap is None or snap.parent_names is None else \
        (lambda p: snap.parent_names[int(p)])
    return uids, par


def _put_mdev_keys(maps: Maps, by_type: MdevResult, by_par: MdevResult, type_ks, par_ks,
                   snap: MdevSnapshot | None = None) -> tuple:
    """Set the vGpuMap key of by_type.type_keys[k] and its deviceNames entry for every k of type_ks, and the gpuVgpuMap
    key by_par.par_keys[k] for every k of par_ks (each result's permutation indexes its own survivors), named through
    `snap` (None is fully numeric) -> (the labels, the parent keys) set, in that order."""
    uids_of, par_of = _mdev_names(snap)
    labels, parents = [], []
    for k in type_ks:
        c = int(by_type.type_keys[k])
        label = by_type.labels[c].decode("latin-1")
        s = by_type.survivors[by_type.type_perm[by_type.type_off[k]:by_type.type_off[k + 1]]]
        maps.vGpuMap[label] = [NvidiaGpuDevice(u, n) for u, n in zip(uids_of(s), s["numa"].tolist())]
        maps.deviceNames[label] = by_type.type_names[c]
        labels.append(label)
    for k in par_ks:
        key = par_of(by_par.par_keys[k])
        maps.gpuVgpuMap[key] = uids_of(by_par.survivors[by_par.par_perm[by_par.par_off[k]:by_par.par_off[k + 1]]])
        parents.append(key)
    return labels, parents


def _patch_mdev_maps(maps: Maps, by_type: MdevResult, by_par: MdevResult, delta, snap: MdevSnapshot | None = None,
                     prev_snap: MdevSnapshot | None = None) -> MdevMapsTouched:
    """The patch of apply_mdev_delta: vGpuMap keys from `by_type`, gpuVgpuMap keys from `by_par` (_put_mdev_keys).
    The new side is named through `snap`, gone parents through `prev_snap`; None is a numeric snapshot."""
    _, prev_par_of = _mdev_names(prev_snap)
    type_dirty, par_dirty = _put_mdev_keys(maps, by_type, by_par, delta.type_dirty, delta.par_dirty, snap)
    t = MdevMapsTouched(type_dirty, [g.decode("latin-1") for g in delta.type_gone], par_dirty,
                        [prev_par_of(p) for p in delta.par_gone])
    for label in t.type_gone:
        maps.vGpuMap.pop(label, None)
        if label not in maps.deviceMap:
            maps.deviceNames.pop(label, None)
    for key in t.par_gone:
        maps.gpuVgpuMap.pop(key, None)
    return t


def canonical_dump(m: Maps) -> bytes:
    """Byte-identical to oracle kvo_dump for the same maps (SURVEY.md 8c)."""
    out = []
    bkey = lambda s: s.encode("latin-1")

    def dev_section(tag, mp):
        for key in sorted(mp, key=bkey):
            name = m.deviceNames.get(key, "")
            out.append("%s %s %s nvidia.com/%s %d\n" % (tag, key, name or "-", name or key,
                                                        len(mp[key])))
            out.extend("  %s %d\n" % (d.addr, d.numaNode) for d in mp[key])

    dev_section("D", m.deviceMap)
    for key in sorted(m.iommuMap, key=bkey):
        out.append("I %s %d\n" % (key, len(m.iommuMap[key])))
        out.extend("  %s %d\n" % (d.addr, d.numaNode) for d in m.iommuMap[key])
    for key in sorted(m.bdfToIommuMap, key=bkey):
        out.append("B %s %s\n" % (key, m.bdfToIommuMap[key]))
    dev_section("V", m.vGpuMap)
    for key in sorted(m.gpuVgpuMap, key=bkey):
        out.append("G %s %d\n" % (key, len(m.gpuVgpuMap[key])))
        out.extend("  %s\n" % u for u in m.gpuVgpuMap[key])
    return "".join(out).encode("latin-1")


# ------------------------------------------------------------------------------------------------
# the controller half the Go host keeps (payload only — the gRPC servers stay in Go)
# ------------------------------------------------------------------------------------------------
@dataclass
class PluginSpec:
    """What NewGenericDevicePlugin / NewGenericVGpuDevicePlugin + Register would be given."""
    key: str
    device_name: str          # getDeviceName(key) or the key itself (:125-128, :153-155)
    resource_name: str        # "nvidia.com/<name>"   generic_device_plugin.go:299
    socket_path: str          # generic_device_plugin.go:87 / generic_vgpu_device_plugin.go:69
    env_key: str              # generic_device_plugin.go:420 / generic_vgpu_device_plugin.go:223
    devs: list                # [{ID, Health, Topology:{Nodes:[{ID}]}}]  (:111-123, :141-150)
    vgpu: bool = False


class DiscoveryScan:
    """InitiateDevicePlugin's scan half (device_plugin.go:89-96) on the GPU."""

    def __init__(self, pci_ids_path: str = "/usr/pci.ids", base_path: str = "/sys/bus/pci/devices",
                 vgpu_base_path: str = "/sys/bus/mdev/devices", device: int = 0):
        self.pciIdsFilePath, self.basePath, self.vGpuBasePath = pci_ids_path, base_path, vgpu_base_path
        self.ctx = Context(device)
        self.maps = Maps()
        self._loaded_path = None
        self._prev_pci_snap = None   # snapshot of the last rescan_iommu_device_map
        self._prev_pci_raw_snap = None   # ... and of the last rescan_iommu_device_map(raw=True)
        self._prev_mdev_raw_snap = None  # ... and of the last rescan_vgpu_id_map(raw=True)
        self._prev_mdev_snap = None  # snapshot of the last rescan_vgpu_id_map

    def close(self):
        self.ctx.close()

    def _ensure_table(self):
        if self._loaded_path == self.pciIdsFilePath:
            return
        data = _read_raw(self.pciIdsFilePath)
        # unreadable file -> getDeviceName returns "" for every key (:373-377): an empty table
        self.ctx.pciids_load(data if data is not None else b"")
        self._loaded_path = self.pciIdsFilePath

    def get_device_name(self, device_id: str) -> str:
        self._ensure_table()
        return self.ctx.name_lookup(device_id)

    def create_iommu_device_map(self, raw: bool = False) -> Maps:
        """raw=True: the walk reads everything and the GPU decodes the reads (Context.scan_pci_raw); the Maps are the
        same."""
        self._ensure_table()
        if raw:
            res, snap = self.ctx.scan_pci_raw(read_pci_tree_raw(self.basePath))
            return pci_maps_from_result(res, snap, self.maps, name_of=self.ctx.name_lookup)
        try:
            snap = snapshot_pci_tree(self.basePath)
        except ReferencePanic:
            raise
        res = self.ctx.scan_pci(snap.recs)
        return pci_maps_from_result(res, snap, self.maps, name_of=self.ctx.name_lookup)

    def rescan_iommu_device_map(self, raw: bool = False) -> PciMapsTouched:
        """Re-walk the tree and bring deviceMap / iommuMap / bdfToIommuMap up to date through the re-scan delta.
        The first call has no previous delta scan to diff against: it rebuilds the maps and reports every key.
        raw=True: the walk reads everything, the GPU decodes the reads and diffs by entry name
        (Context.scan_pci_raw_delta), so the maps are patched, not rebuilt, in every snapshot mode."""
        self._ensure_table()
        if raw:
            res, snap, delta = self.ctx.scan_pci_raw_delta(read_pci_tree_raw(self.basePath))
            prev, self._prev_pci_raw_snap = self._prev_pci_raw_snap, snap
            if prev is None:
                return _rebuild_pci_maps(self.maps, res, snap, self.ctx.name_lookup)
            return apply_pci_delta(self.maps, res, delta, snap, prev, name_of=self.ctx.name_lookup)
        snap = snapshot_pci_tree(self.basePath)
        res, delta = self.ctx.scan_pci_delta(snap.recs)
        prev, self._prev_pci_snap = self._prev_pci_snap, snap
        if prev is None:
            return _rebuild_pci_maps(self.maps, res, snap, self.ctx.name_lookup)
        return apply_pci_delta(self.maps, res, delta, snap, prev, name_of=self.ctx.name_lookup)

    def create_vgpu_id_map(self, raw: bool = False) -> Maps:
        """raw=True: the walk reads everything and the GPU decodes the reads (Context.scan_mdev_raw).  The Maps are the
        same, except that a vGPU whose parent component is empty is listed under gpuVgpuMap[""] as in the reference
        (the default path lists it under "0000:00:00.0")."""
        self._ensure_table()
        if raw:
            res, snap = self.ctx.scan_mdev_raw(read_mdev_tree_raw(self.vGpuBasePath, self.basePath))
            return mdev_maps_from_result(res, snap, self.maps)
        snap = snapshot_mdev_tree(self.vGpuBasePath, self.basePath)
        res = self.ctx.scan_mdev(snap.recs, snap.raw_types)
        return mdev_maps_from_result(res, snap, self.maps)

    def rescan_vgpu_id_map(self, raw: bool = False) -> MdevMapsTouched:
        """Re-walk the mdev tree and bring vGpuMap / gpuVgpuMap up to date through the re-scan delta.  The first call
        has no previous delta scan to diff against: it rebuilds the maps and reports every key.  raw=True: the walk
        reads everything, the GPU decodes the reads and diffs by entry name (Context.scan_mdev_raw_delta), so the maps
        are patched, not rebuilt, in every snapshot mode."""
        self._ensure_table()
        if raw:
            res, snap, delta = self.ctx.scan_mdev_raw_delta(read_mdev_tree_raw(self.vGpuBasePath, self.basePath))
            prev, self._prev_mdev_raw_snap = self._prev_mdev_raw_snap, snap
            if prev is None:
                return _rebuild_mdev_maps(self.maps, res, res, snap)
            return apply_mdev_delta(self.maps, res, delta, snap, prev)
        snap = snapshot_mdev_tree(self.vGpuBasePath, self.basePath)
        res, delta = self.ctx.scan_mdev_delta(snap.recs, snap.raw_types)
        prev, self._prev_mdev_snap = self._prev_mdev_snap, snap
        if prev is None:
            return _rebuild_mdev_maps(self.maps, res, res, snap)
        return apply_mdev_delta(self.maps, res, delta, snap, prev)

    def create_device_plugins(self) -> list:
        return plugin_specs_from_maps(self.maps)


def plugin_specs_from_maps(maps: Maps) -> list:
    """createDevicePlugins' payload half (device_plugin.go:99-157): one PluginSpec per deviceMap key,
    then one per vGpuMap key; name falls back to the key when getDeviceName returned ""."""
    specs = []
    for devices, prefix, vgpu in ((maps.deviceMap, GPU_PREFIX, False), (maps.vGpuMap, VGPU_PREFIX, True)):
        for key, devs in devices.items():
            name = maps.deviceNames.get(key, "") or key
            specs.append(PluginSpec(
                key, name, "%s/%s" % (DEVICE_NAMESPACE, name),
                "%skubevirt-%s.sock" % (DEVICE_PLUGIN_PATH, name),
                "%s_%s" % (prefix, name.upper()),
                [{"ID": d.addr, "Health": HEALTHY, "Topology": {"Nodes": [{"ID": d.numaNode}]}}
                 for d in devs], vgpu=vgpu))
    return specs
