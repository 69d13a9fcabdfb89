"""The consumer side of the scan: the kubelet-facing DevicePlugin servers fed by the GPU results.

SURVEY.md 8(f): (1) host glue + a mock kubelet to replay Register -> ListAndWatch -> Allocate,
(2) Allocate-time re-validation as ONE batched re-scan, (3) a health feed driven by the K6 delta
kernel, (4) GetPreferredAllocation NUMA packing (on the GPU through NumaPacker) and EGM path
selection (EGM discovery on the host, the all-GPUs match on the GPU through AllocateCheck), both pinned by the reference's own tests.  Function by function this mirrors

    pkg/device_plugin/generic_device_plugin.go       (passthrough plugin)
    pkg/device_plugin/generic_vgpu_device_plugin.go  (vGPU plugin)

with the same names, argument meaning and error strings, so tests/test_serve.py reads like the
reference's generic_device_plugin_test.go.  In a deployment these servers stay in Go
(INTEGRATION.md); this Python mirror exists so that "drops in behind Register / ListAndWatch /
Allocate" is testable end to end in an image without a Go toolchain.

Nothing here computes on the CPU what the scan computes on the GPU: the maps come from
plugin.DiscoveryScan (libkvgpu.so); the passthrough re-validation's group and vendor rule goes through
Context.pci_allocate_check together with the EGM match, one call per AllocateRequest (AllocateCheck; GroupCheck
through Context.pci_group_check with the CPU EGM rule, and BatchRevalidator, the same check through
Context.scan_pci (K3), are the references it is tested against), the vGPU plugin's label check through Context.mdev_label_match (MdevLabelCheck;
a vGPU plugin built without a check keeps the reference's CPU rule, the path the GPU check is tested
against), the passthrough plugin's GetPreferredAllocation through Context.preferred_allocation (NumaPacker;
preferred_allocation below stays the reference it is tested against); the health feeds through Context.health_rescan, Context.health_rescan_mdev and
Context.health_rescan_groups and their keyed forms (K6); the
hot-plug feeds through Context.scan_pci_delta and Context.scan_mdev_delta (K7).
"""
from __future__ import annotations

import os
import queue
import threading
import time
from concurrent import futures
from dataclasses import dataclass, field

import numpy as np

from . import _lib as L
from . import dpapi
from .plugin import (DEVICE_NAMESPACE, GPU_PREFIX, NOT_READ, VGPU_PREFIX, Maps, PluginSpec, ReferencePanic, _read_id,
                     _read_link, _read_raw, _read_vgpu_raw, _rebuild_mdev_maps, _rebuild_pci_maps, apply_mdev_delta,
                     apply_pci_delta, format_uuid, pack_alloc_raw, pack_alloc_response, parse_bdf,
                     plugin_specs_from_maps)

VFIO_DEVICE_PATH = "/dev/vfio"      # generic_device_plugin.go:54
IOMMU_DEVICE_PATH = "/dev/iommu"    # :55
EGM_CLASS_PATH = "/sys/class/egm"   # :56
DEVICE_DIR = "/dev"
NVIDIA_VENDOR_ID = "10de"           # device_plugin.go:46
CONNECTION_TIMEOUT = 5.0            # generic_device_plugin.go:53


class AllocateError(Exception):
    """An error return of Allocate / GetPreferredAllocation (the text is the reference's)."""


# ------------------------------------------------------------------------------------------------
# host logic, pinned by the reference's tests (tests/golden/plugin_vectors.json)
# ------------------------------------------------------------------------------------------------
def preferred_allocation(devs, available, must_include, allocation_size) -> list:
    """GetPreferredAllocation for ONE container request (generic_device_plugin.go:470-608).

    devs: iterable of (device id, numa node or None).  Must-include devices first (request order),
    then try to complete from a single NUMA node — nodes of the must-include devices first, then
    nodes in order of first appearance in `available` — else fall back to kubelet order."""
    device_to_numa = {d: n for d, n in devs if n is not None}

    def numa_of(dev_id):
        return device_to_numa.get(dev_id, -1)

    numa_to_devices, node_order = {}, []
    for dev_id in available:
        node = numa_of(dev_id)
        if node not in numa_to_devices:
            numa_to_devices[node] = []
            node_order.append(node)
        numa_to_devices[node].append(dev_id)

    preferred, chosen, selected_per_node = [], set(), {}

    def add(dev_id):
        if dev_id in chosen:
            return
        chosen.add(dev_id)
        node = numa_of(dev_id)
        selected_per_node[node] = selected_per_node.get(node, 0) + 1
        preferred.append(dev_id)

    selected_node_order = []
    for dev_id in must_include:
        if dev_id in chosen:
            continue
        add(dev_id)
        node = numa_of(dev_id)
        if node not in selected_node_order:
            selected_node_order.append(node)
    if len(preferred) > allocation_size:
        raise AllocateError("number of MustIncludeDeviceIDs (%d) exceeds allocation size (%d)"
                            % (len(preferred), allocation_size))
    if len(preferred) < allocation_size:
        target = None
        candidates = selected_node_order + [n for n in node_order if n not in selected_node_order]
        for node in candidates:
            free = sum(1 for d in numa_to_devices.get(node, []) if d not in chosen)
            if selected_per_node.get(node, 0) + free >= allocation_size:
                target = node
                break
        # the reference encodes "no node" as -1, which is also the id of devices without topology:
        # such a pseudo-node is never used as a target (:552-575)
        if target is not None and target != -1:
            for dev_id in numa_to_devices.get(target, []):
                if len(preferred) >= allocation_size:
                    break
                add(dev_id)
    if len(preferred) < allocation_size:
        for dev_id in available:
            if len(preferred) >= allocation_size:
                break
            add(dev_id)
    return preferred


@dataclass
class EGMDeviceInfo:      # generic_device_plugin.go:62-65
    dev_path: str
    gpu_bdfs: list


def discover_egm_devices(root_path: str = "/") -> list:
    """discoverEGMDevicesFunc :120-157 (a missing class directory is not an error)."""
    class_dir = os.path.join(root_path, EGM_CLASS_PATH.lstrip("/"))
    try:
        entries = sorted(os.listdir(class_dir))
    except FileNotFoundError:
        return []
    out = []
    for name in entries:
        if not name.startswith("egm"):
            continue
        try:
            with open(os.path.join(class_dir, name, "gpu_devices"), "rb") as f:
                raw = f.read().decode("utf-8", "replace")
        except OSError:
            continue
        bdfs = raw.split()
        if not bdfs:
            continue
        dev_path = os.path.join(DEVICE_DIR, name)
        if not os.path.exists(os.path.join(root_path, dev_path.lstrip("/"))):
            continue
        out.append(EGMDeviceInfo(dev_path, bdfs))
    out.sort(key=lambda e: e.dev_path)
    return out


def egm_key(bdf: str) -> str:
    """The string egmPathsForAllocatedGPUs compares (:167, :173): strings.ToLower(strings.TrimSpace(bdf)).  Python's
    strip() and lower() agree with Go's on ASCII; exotic Unicode input may differ."""
    return bdf.strip().lower()


def egm_paths_for_allocated_gpus(allocated_bdfs, egm_devices) -> list:
    """egmPathsForAllocatedGPUs :159-184: an EGM node is injected only when ALL its GPUs are allocated."""
    allocated = {egm_key(b) for b in allocated_bdfs}
    return sorted(e.dev_path for e in (egm_devices or [])
                  if all(egm_key(g) in allocated for g in e.gpu_bdfs))


@dataclass
class EGMEntryRaw:
    """One entry of the EGM class directory as discoverEGMDevicesFunc's reads returned it (:120-157), undecoded:
    gpu_devices is the file's bytes, None when the read failed, or plugin.NOT_READ; stat is whether os.Stat of
    /dev/<name> succeeded, or plugin.NOT_READ."""
    name: bytes
    gpu_devices: object
    stat: object


def discover_egm_raw(root_path: str = "/") -> list:
    """The reads of discoverEGMDevicesFunc :120-157, decoding nothing: every entry of the EGM class directory in
    ReadDir order (sorted by name bytes), its gpu_devices contents and the Stat of its device node, each made for every
    entry (the GPU decides which the reference reaches).  A missing class directory is no entry (:124-126); any other
    listing error raises, so that Allocate continues without EGM mounts (:366-370)."""
    class_dir = os.fsencode(os.path.join(root_path, EGM_CLASS_PATH.lstrip("/")))
    try:
        names = sorted(os.listdir(class_dir))
    except FileNotFoundError:
        return []
    out = []
    for name in names:
        try:
            with open(os.path.join(class_dir, name, b"gpu_devices"), "rb") as f:
                gpus = f.read()
        except OSError:
            gpus = None
        try:
            os.stat(os.path.join(os.fsencode(root_path), DEVICE_DIR.lstrip("/").encode(), name))
            stat = True
        except OSError:
            stat = False
        out.append(EGMEntryRaw(name, gpus, stat))
    return out


def supports_iommufd(root_path: str = "/") -> bool:
    """supportsIOMMUFD :692-701"""
    try:
        os.stat(os.path.join(root_path, IOMMU_DEVICE_PATH.lstrip("/")))
        return True
    except FileNotFoundError:
        return False
    except OSError as e:
        raise AllocateError("could not determine iommufd support: %s" % e)


def read_vfio_dev(base_path: str, addr: str) -> str:
    """readVFIODev :702-716: the first vfio* directory under <addr>/vfio-dev."""
    d = os.path.join(base_path, addr, "vfio-dev")
    for name in sorted(os.listdir(d)):          # os.ReadDir sorts by filename
        if os.path.isdir(os.path.join(d, name)) and name.startswith("vfio"):
            return name
    raise OSError("no iommufd device found")


def read_vfio_dev_raw(base_path: str, addr: str):
    """The listing readVFIODev makes (:702-716), deciding nothing: ([(name bytes, IsDir)], None) in listing order,
    IsDir not following links as DirEntry.IsDir() does, or (None, the error text) when the listing fails."""
    d = os.path.join(os.fsencode(base_path), os.fsencode(addr), b"vfio-dev")
    try:
        with os.scandir(d) as it:
            return [(e.name, e.is_dir(follow_symlinks=False)) for e in it], None
    except OSError as e:     # the text read_vfio_dev's os.listdir raises for the same path
        return None, str(OSError(e.errno, e.strerror, os.fsdecode(d)))


# ------------------------------------------------------------------------------------------------
# Allocate-time re-validation as one batched re-scan (SURVEY.md 8(f) rank 2)
# ------------------------------------------------------------------------------------------------
class BatchRevalidator:
    """Re-check every device of every requested IOMMU group in ONE pass of the classification
    kernel instead of one readLink + one readIDFromFile round per device
    (generic_device_plugin.go:387-399).

    The sysfs reads use the reference's own readers, in the reference's order; what they returned
    becomes ordinary scan records (index mode: addr = position in the batch, iommu_group = interned
    group string).  The record's driver is pinned to vfio-pci and its device id to a constant,
    because Allocate re-checks ONLY the group link and the vendor — with that, K3's predicate
    (vendor == 10de, no vendor / iommu read error) is exactly the reference's acceptance test and
    the survivor's group id says whether the link still points at the expected group."""

    def __init__(self, scan_pci, base_path: str = "/sys/bus/pci/devices",
                 read_link=_read_link, read_id=_read_id):
        self.scan_pci, self.base_path = scan_pci, base_path
        self.read_link, self.read_id = read_link, read_id

    def __call__(self, pairs):
        """pairs: [(addr, expected iommu group)] in the order the reference would visit them.
        Returns the index of the first device the reference would reject, or None.  A reader panic
        (short vendor file) is re-raised only if the reference would have reached that read."""
        n = len(pairs)
        if n == 0:
            return None
        recs = np.zeros(n, dtype=L.PCI_REC)
        intern, panics = {}, {}
        for i, (addr, expect) in enumerate(pairs):
            want = intern.setdefault(expect, len(intern))
            flags, vendor, group = 0, 0xFFFF, want
            got, err = self.read_link(self.base_path, addr, "iommu_group")
            if err:
                flags |= L.PF_IOMMU_ERR
            else:
                group = intern.setdefault(got, len(intern))
            try:
                v, err = self.read_id(self.base_path, addr, "vendor")
            except ReferencePanic as e:
                panics[i] = e
                v, err = "", True
            if err:
                flags |= L.PF_VENDOR_ERR
            elif v == NVIDIA_VENDOR_ID:
                vendor = 0x10de
            recs[i] = (i, vendor, 0, group, L.DRV_VFIO_PCI, flags, 0)
        res = self.scan_pci(recs)
        ok_group = {int(s["addr"]): int(s["iommu_group"]) for s in res.survivors}
        for i, (addr, expect) in enumerate(pairs):
            link_ok = not (int(recs[i]["flags"]) & L.PF_IOMMU_ERR) and int(recs[i]["iommu_group"]) == intern[expect]
            if link_ok and i in panics:   # the reference reads the vendor only after the link check passed
                raise panics[i]
            if ok_group.get(i) != intern[expect]:
                return i
        return None


class GroupCheck:
    """The passthrough plugin's Allocate-time re-check (generic_device_plugin.go:387-399) as its own rule in one
    launch: a drop-in `revalidate` for GenericDevicePlugin with BatchRevalidator's contract, which stays as the
    reference this check is tested against.

    Every device's iommu_group link and vendor are read with the reference's readers, in the reference's order.  What
    they returned goes to ONE `group_check` call (Context.pci_group_check): per device a record with the read errors,
    the link's group and the vendor (0x10de iff it read "10de"), and the group the maps hold for it.  The group
    strings are interned per call, so equal handles mean equal strings ("042" is not "42").  Nothing in the record
    but those reads matters to the rule, so no driver or device id is pinned."""

    def __init__(self, group_check, base_path: str = "/sys/bus/pci/devices", read_link=_read_link, read_id=_read_id):
        self.group_check, self.base_path = group_check, base_path
        self.read_link, self.read_id = read_link, read_id

    def __call__(self, pairs):
        """pairs: [(addr, expected iommu group)] in the order the reference would visit them.
        Returns the index of the first device the reference would reject, or None.  A reader panic
        (short vendor file) is re-raised only if the reference would have reached that read."""
        n = len(pairs)
        if n == 0:
            return None
        recs, want = np.zeros(n, dtype=L.PCI_REC), np.zeros(n, dtype=np.uint32)
        intern, link_ok, panics = {}, [False] * n, {}
        for i, (addr, expect) in enumerate(pairs):
            want[i] = intern.setdefault(expect, len(intern))
            flags, vendor, group = 0, 0xFFFF, 0
            got, err = self.read_link(self.base_path, addr, "iommu_group")
            if err:
                flags |= L.PF_IOMMU_ERR
            else:
                group = intern.setdefault(got, len(intern))
                link_ok[i] = got == expect
            try:
                v, err = self.read_id(self.base_path, addr, "vendor")
            except ReferencePanic as e:
                panics[i] = e
                v, err = "", True
            if err:
                flags |= L.PF_VENDOR_ERR
            elif v == NVIDIA_VENDOR_ID:
                vendor = 0x10de
            recs[i] = (i, vendor, 0, group, 0, flags, 0)
        bad = self.group_check(recs, want)
        # a panicking read fails its record, so the only one the reference can reach is the first rejected device,
        # and only when its link check passed (the vendor is read after it)
        if bad is not None and bad in panics and link_ok[bad]:
            raise panics[bad]
        return bad


class AllocateCheck:
    """The passthrough plugin's Allocate decisions (generic_device_plugin.go:352-444) for every container request of
    one AllocateRequest in ONE launch: the group re-check of GroupCheck and the EGM match of
    egm_paths_for_allocated_gpus.  A drop-in `allocate_check` for GenericDevicePlugin; GroupCheck with the CPU EGM
    rule stays as the reference it is tested against.

    Every member's iommu_group link and vendor are read with the reference's readers, in the reference's order
    (request by request, BDF by BDF, member by member); a reader panic is caught per member.  The group strings are
    interned in one table per call, as GroupCheck does.  The EGM devices' GPU strings are interned by egm_key first,
    and each DevicesID goes as the handle of its key, or as n_egm_gpus when no EGM device lists that key.  `call` is
    Context.pci_allocate_check; what it returns is mapped back, and nothing is decided here."""

    def __init__(self, call, base_path: str = "/sys/bus/pci/devices", read_link=_read_link, read_id=_read_id):
        self.call, self.base_path = call, base_path
        self.read_link, self.read_id = read_link, read_id

    def __call__(self, requests, egm_devices) -> list:
        """requests: [(pairs, devices_ids)] in request order, where pairs = [(addr, expected iommu group)] in the
        order the reference would visit them; egm_devices: the discovered EGM devices (None or [] for none).
        Returns per request (bad, panic, egm_paths): the position of the first member the reference would reject
        (None: none), the ReferencePanic its vendor read raised if the reference reaches that read (None: no panic),
        and the dev paths of the EGM devices to mount, sorted."""
        egm_devices = list(egm_devices or [])
        egm_handle, egm_off, egm_gpu = {}, [0] if egm_devices else [], []
        for e in egm_devices:
            egm_gpu.extend(egm_handle.setdefault(egm_key(g), len(egm_handle)) for g in e.gpu_bdfs)
            egm_off.append(len(egm_gpu))
        n_egm_gpus = len(egm_handle)
        n_pairs = sum(len(pairs) for pairs, _ in requests)
        recs, want = np.zeros(n_pairs, dtype=L.PCI_REC), np.zeros(n_pairs, dtype=np.uint32)
        intern, link_ok, panics, ids, n_members, n_ids = {}, [False] * n_pairs, {}, [], [], []
        i = 0
        for pairs, devices_ids in requests:
            for addr, expect in pairs:
                want[i] = intern.setdefault(expect, len(intern))
                flags, vendor, group = 0, 0xFFFF, 0
                got, err = self.read_link(self.base_path, addr, "iommu_group")
                if err:
                    flags |= L.PF_IOMMU_ERR
                else:
                    group = intern.setdefault(got, len(intern))
                    link_ok[i] = got == expect
                try:
                    v, err = self.read_id(self.base_path, addr, "vendor")
                except ReferencePanic as e:
                    panics[i] = e
                    v, err = "", True
                if err:
                    flags |= L.PF_VENDOR_ERR
                elif v == NVIDIA_VENDOR_ID:
                    vendor = 0x10de
                recs[i] = (i, vendor, 0, group, 0, flags, 0)
                i += 1
            ids.extend(egm_handle.get(egm_key(b), n_egm_gpus) for b in devices_ids)
            n_members.append(len(pairs))
            n_ids.append(len(devices_ids))
        first_bad, take = self.call(recs, want, n_members, ids, n_ids, egm_off, egm_gpu, n_egm_gpus)
        out, at = [], 0
        for r, n in enumerate(n_members):
            bad = None if int(first_bad[r]) == n else int(first_bad[r])
            # a panicking read fails its record; the reference reaches it only as the first rejected member, and only
            # when its link check passed (the vendor is read after it)
            panic = panics.get(at + bad) if bad is not None and link_ok[at + bad] else None
            out.append((bad, panic, sorted(e.dev_path for e, t in zip(egm_devices, take[r]) if t)))
            at += n
        return out


class AllocateRawCheck:
    """The passthrough plugin's Allocate decisions (generic_device_plugin.go:352-444) for every container request of
    one AllocateRequest, decided on the GPU from the raw reads: a drop-in `allocate_check` for GenericDevicePlugin with
    AllocateCheck's contract, whose `discover_egm` is discover_egm_raw.  AllocateCheck stays as the reference it is
    tested against.

    Every member's iommu_group link target and vendor contents are read raw, in the reference's order; with the group
    string the maps hold for the member, the DevicesIDs and the EGM class entries they go to ONE `call`
    (Context.pci_allocate_raw), which decodes, compares and matches them all.  Nothing is decoded or interned here:
    what the call returns is mapped back to (bad, panic, egm_paths) per request."""

    def __init__(self, call, base_path: str = "/sys/bus/pci/devices"):
        self.call, self.base_path = call, base_path

    def _read(self, addr, prop, link):
        return _read_raw(os.path.join(os.fsencode(self.base_path), os.fsencode(addr), prop), link)

    def __call__(self, requests, egm_entries) -> list:
        """requests: [(pairs, devices_ids)] as for AllocateCheck; egm_entries: discover_egm_raw's entries (None or []
        for none).  Returns per request (bad, panic, egm_paths) as AllocateCheck does."""
        egm = list(egm_entries or [])
        raw = pack_alloc_raw(
            [([(self._read(addr, b"iommu_group", True), self._read(addr, b"vendor", False), group)
               for addr, group in pairs], list(devices_ids)) for pairs, devices_ids in requests],
            [(e.name, e.gpu_devices, e.stat) for e in egm])
        first_bad, panic, kept, take = self.call(raw)
        out = []
        for r, (pairs, _) in enumerate(requests):
            bad = None if int(first_bad[r]) == len(pairs) else int(first_bad[r])
            p = (ReferencePanic("slice bounds out of range reading %s/vendor" % pairs[bad][0]) if panic[r] else None)
            names = sorted(e.name for e, k, t in zip(egm, kept, take[r]) if k and t)
            out.append((bad, p, [os.path.join(DEVICE_DIR, os.fsdecode(n)) for n in names]))
        return out


class AllocateResponder:
    """The passthrough plugin's whole Allocate (generic_device_plugin.go:352-444) after the plan, in ONE call
    (Context.pci_allocate_response): a drop-in `allocate_response` for GenericDevicePlugin, whose `discover_egm` is
    discover_egm_raw.  GenericDevicePlugin.Allocate's replay with AllocateRawCheck stays as the reference it is tested
    against.

    Every planned member's iommu_group link, vendor and (with iommufd) vfio-dev listing are read raw; with the plan,
    the DevicesIDs and the EGM class entries they go to the call, which returns per request the reference's first
    error or the device specs and the env value.  Here the error texts are formatted and the response is built;
    nothing is decided."""

    def __init__(self, call, base_path: str = "/sys/bus/pci/devices"):
        self.call, self.base_path = call, base_path

    def _read(self, addr, prop, link):
        return _read_raw(os.path.join(os.fsencode(self.base_path), os.fsencode(addr), prop), link)

    def __call__(self, device_name, requests, iommufd, egm_entries):
        """requests: [(devices_ids, plan, lookup_error_at)] with GenericDevicePlugin._plan's plan; iommufd:
        supports_iommufd; egm_entries: discover_egm_raw's entries (None or [] for none).  Returns the
        AllocateResponse, or raises AllocateError / ReferencePanic with the reference's text."""
        errors, packed = {}, []
        for r, (ids, plan, lookup_error_at) in enumerate(requests):
            visits = []
            for _, group, members in plan:
                visit = []
                for dev in members:
                    listing = NOT_READ
                    if iommufd:
                        listing, text = read_vfio_dev_raw(self.base_path, dev.addr)
                        if text is not None:
                            errors[(r, dev.addr)] = text
                    visit.append((dev.addr, self._read(dev.addr, b"iommu_group", True),
                                  self._read(dev.addr, b"vendor", False), group, listing))
                visits.append(visit)
            packed.append((ids, visits, lookup_error_at is not None))
        egm = [(e.name, e.gpu_devices, e.stat) for e in (egm_entries or [])]
        decided = self.call(*pack_alloc_response(packed, egm, iommufd))
        responses = dpapi.AllocateResponse()
        key = "%s_%s" % (GPU_PREFIX, device_name.upper())
        for r, (error, at, paths, env) in enumerate(decided):
            ids, plan, _ = requests[r]
            addr = lambda p: [d.addr for _, _, members in plan for d in members][p]   # noqa: E731
            if error == L.ARESP_UNKNOWN_ID:
                raise AllocateError("invalid allocation request: unknown device: %s" % ids[at])
            if error == L.ARESP_UNKNOWN_MEMBER:
                raise AllocateError("invalid allocation request: unknown device: %s" % addr(at))
            if error == L.ARESP_PANIC:
                raise ReferencePanic("slice bounds out of range reading %s/vendor" % addr(at))
            if error in (L.ARESP_VFIO_READ, L.ARESP_VFIO_NONE):
                why = errors[(r, addr(at))] if error == L.ARESP_VFIO_READ else "no iommufd device found"
                raise AllocateError("could not determine iommufd device for device %s: %s" % (addr(at), why))
            specs = [dpapi.DeviceSpec(host_path=os.fsdecode(p), container_path=os.fsdecode(p), permissions="mrw")
                     for p in paths]
            envs = {key: os.fsdecode(env)} if env is not None else {}
            responses.container_responses.append(dpapi.ContainerAllocateResponse(envs=envs, devices=specs))
        return responses


# ------------------------------------------------------------------------------------------------
# the plugins
# ------------------------------------------------------------------------------------------------
def devices_from_spec(spec: PluginSpec) -> list:
    """PluginSpec.devs -> []*pluginapi.Device (device_plugin.go:111-123, :141-150)."""
    return [dpapi.Device(ID=d["ID"], health=d["Health"],
                         topology=dpapi.TopologyInfo(nodes=[dpapi.NUMANode(ID=n["ID"]) for n in d["Topology"]["Nodes"]]))
            for d in spec.devs]


class _PluginBase:
    """Start / Stop / Register / ListAndWatch shared by both plugins
    (generic_device_plugin.go:216-349, generic_vgpu_device_plugin.go:75-205)."""
    vgpu = False

    def __init__(self, device_name: str, devs: list, socket_dir: str = dpapi.DEVICE_PLUGIN_PATH,
                 kubelet_socket: str | None = None):
        self.device_name = device_name
        self.devs = list(devs)
        self.socket_path = os.path.join(socket_dir, "kubevirt-%s.sock" % device_name)
        self.kubelet_socket = kubelet_socket or os.path.join(socket_dir, "kubelet.sock")
        self.server = None
        self._events = queue.Queue()     # ("healthy" | "unhealthy", device id): the two Go channels;
                                         # ("devices", None): the device list changed (a re-scan feed)
        self._stop = threading.Event()
        self._term = threading.Event()
        self._lock = threading.Lock()

    # -- the two channels of the reference (dpi.healthy / dpi.unhealthy)
    def healthy(self, dev_id: str):
        self._events.put(("healthy", dev_id))

    def unhealthy(self, dev_id: str):
        self._events.put(("unhealthy", dev_id))

    def set_devices(self, devs: list):
        """A new device list (a re-scan changed this key): devices that stay keep their current health, and
        ListAndWatch re-sends the whole list."""
        with self._lock:
            health = {d.ID: d.health for d in self.devs}
            for d in devs:
                d.health = health.get(d.ID, d.health)
            self.devs = list(devs)
        self._events.put(("devices", None))

    def resource_name(self) -> str:
        return "%s/%s" % (DEVICE_NAMESPACE, self.device_name)

    # -- gRPC methods
    def GetDevicePluginOptions(self, request, context):
        # passthrough: preferred allocation available (:451-457); vGPU: not (:252-257)
        return dpapi.DevicePluginOptions(pre_start_required=False,
                                         get_preferred_allocation_available=not self.vgpu)

    def PreStartContainer(self, request, context):
        return dpapi.PreStartContainerResponse()

    def ListAndWatch(self, request, context):
        """:312-349 — send the list once, then the whole list again after every health flip and after every
        set_devices."""
        yield dpapi.ListAndWatchResponse(devices=self.devs)
        while not (self._stop.is_set() or self._term.is_set()):
            if context is not None and not context.is_active():
                return
            try:
                kind, dev_id = self._events.get(timeout=0.02)
            except queue.Empty:
                continue
            with self._lock:
                for dev in self.devs:
                    if kind != "devices" and dev.ID == dev_id:
                        dev.health = dpapi.HEALTHY if kind == "healthy" else dpapi.UNHEALTHY
                devs = list(self.devs)
            yield dpapi.ListAndWatchResponse(devices=devs)

    # -- lifecycle
    def _handlers(self):
        import grpc
        table = {}
        for mname, (req, resp, stream) in dpapi.SERVICES["DevicePlugin"].items():
            fn = self._wrap(getattr(self, mname))
            make = grpc.unary_stream_rpc_method_handler if stream else grpc.unary_unary_rpc_method_handler
            table[mname] = make(fn, request_deserializer=dpapi.MESSAGES[req].FromString,
                                response_serializer=dpapi.MESSAGES[resp].SerializeToString)
        return grpc.method_handlers_generic_handler(dpapi.service_name("DevicePlugin"), table)

    @staticmethod
    def _wrap(fn):
        import grpc
        import inspect
        if inspect.isgeneratorfunction(fn):
            return fn

        def call(request, context):
            try:
                return fn(request, context)
            except AllocateError as e:    # a Go `return nil, err` -> status UNKNOWN with the text
                context.abort(grpc.StatusCode.UNKNOWN, str(e))
        return call

    def start(self):
        """Start :216-257: serve on the plugin socket, then Register with the kubelet."""
        import grpc
        if self.server is not None:
            raise RuntimeError("gRPC server already started")
        self._stop.clear()
        self._term.clear()
        self.cleanup()
        self.server = grpc.server(futures.ThreadPoolExecutor(max_workers=8))
        self.server.add_generic_rpc_handlers((self._handlers(),))
        self.server.add_insecure_port("unix://" + self.socket_path)
        self.server.start()
        self.register()

    def stop(self):
        """Stop :260-273"""
        if self.server is None:
            return
        self._term.set()
        self.server.stop(0.2).wait(2.0)
        self.server = None
        self.cleanup()

    def restart(self):
        """restart :276-287 (kubelet restarted: the plugin socket was removed under us)."""
        if self.server is None:
            raise RuntimeError("grpc server instance not found for %s" % self.device_name)
        self.stop()
        self.start()

    def cleanup(self):
        try:
            os.remove(self.socket_path)
        except FileNotFoundError:
            pass

    def register(self):
        """Register :289-309"""
        import grpc
        with grpc.insecure_channel("unix://" + self.kubelet_socket) as ch:
            grpc.channel_ready_future(ch).result(timeout=CONNECTION_TIMEOUT)
            call = ch.unary_unary(dpapi.method_path("Registration", "Register"),
                                  request_serializer=dpapi.RegisterRequest.SerializeToString,
                                  response_deserializer=dpapi.Empty.FromString)
            call(dpapi.RegisterRequest(version=dpapi.VERSION, endpoint=os.path.basename(self.socket_path),
                                       resource_name=self.resource_name()), timeout=CONNECTION_TIMEOUT)


class GenericDevicePlugin(_PluginBase):
    """The passthrough plugin (generic_device_plugin.go).  `maps` supplies what returnIommuMap /
    returnBdfToIommuMap supply in the reference; `revalidate` is the Allocate-time re-check
    (GroupCheck, or BatchRevalidator over a scan function); `allocate_check` (AllocateCheck), when set, takes every
    Allocate decision of an AllocateRequest in one GPU call instead: the re-check and the EGM match of every container
    request; `allocate_response` (AllocateResponder), when set, builds the whole AllocateResponse of an AllocateRequest
    in one GPU call after the plan; `prefer` answers GetPreferredAllocation
    (NumaPacker: every container request in one GPU call; None: preferred_allocation per request on the CPU)."""

    def __init__(self, device_name, device_path, devs, maps: Maps, *, revalidate=None,
                 base_path="/sys/bus/pci/devices", root_path="/", discover_egm=None, prefer=None, allocate_check=None,
                 allocate_response=None, **kw):
        super().__init__(device_name, devs, **kw)
        self.device_path, self.maps = device_path, maps
        self.base_path, self.root_path = base_path, root_path
        self.revalidate, self.prefer, self.allocate_check = revalidate, prefer, allocate_check
        self.allocate_response = allocate_response
        self.discover_egm = discover_egm or (lambda: discover_egm_devices(self.root_path))

    def GetPreferredAllocation(self, request, context):
        resp = dpapi.PreferredAllocationResponse()
        devs = [(d.ID, d.topology.nodes[0].ID if len(d.topology.nodes) else None) for d in self.devs]
        if self.prefer is not None:
            reqs = [(list(r.available_deviceIDs), list(r.must_include_deviceIDs), int(r.allocation_size))
                    for r in request.container_requests]
            for ids in self.prefer(devs, reqs):
                resp.container_responses.append(dpapi.ContainerPreferredAllocationResponse(deviceIDs=ids))
            return resp
        for req in request.container_requests:
            ids = preferred_allocation(devs, list(req.available_deviceIDs), list(req.must_include_deviceIDs),
                                       int(req.allocation_size))
            resp.container_responses.append(dpapi.ContainerPreferredAllocationResponse(deviceIDs=ids))
        return resp

    def _plan(self, req):
        """Map lookups only: the (bdf, group, members) the reference would visit, in order, and the (position, bdf)
        of a lookup error that stops the request, or None."""
        iommu_map, bdf_to_iommu = self.maps.iommuMap, self.maps.bdfToIommuMap
        plan = []
        for k, bdf in enumerate(req.devices_ids):
            group = bdf_to_iommu.get(bdf)
            members = iommu_map.get(group, []) if group is not None else []
            if group is None or not members:
                return plan, (k, bdf)
            plan.append((bdf, group, members))
        return plan, None

    def Allocate(self, request, context):
        """:352-447.  The sequence of checks, device specs and env values is the reference's.  With
        `allocate_check`, every container request is planned first and ONE call decides the re-check and the EGM match
        of them all; each request is then replayed in the reference's order, so the first error of the first failing
        request wins.  Otherwise the per-device re-validation of each request is handed to `self.revalidate` as one
        batch, and the EGM match is the CPU rule."""
        if self.revalidate is None and self.allocate_check is None and self.allocate_response is None:
            raise AllocateError("no re-validation function configured (the scan context is required)")
        responses = dpapi.AllocateResponse()
        env_list = {}                       # declared OUTSIDE the request loop in the reference (:361)
        iommufd = supports_iommufd(self.root_path)
        try:
            egm_devices = self.discover_egm()
        except Exception:                   # :366-370 a discovery failure only disables EGM mounts
            egm_devices = None
        reqs = list(request.container_requests)
        if self.allocate_response is not None:
            return self.allocate_response(self.device_name,
                                          [(list(req.devices_ids),) + self._plan(req) for req in reqs], iommufd,
                                          egm_devices)
        plans = decided = None
        if self.allocate_check is not None:
            plans = [self._plan(req) for req in reqs]
            decided = iter(self.allocate_check(
                [([(d.addr, group) for _, group, members in plan for d in members], list(req.devices_ids))
                 for req, (plan, _) in zip(reqs, plans)], egm_devices))
        for r, req in enumerate(reqs):
            specs, seen = [], set()

            def append_spec(host_path):
                if host_path not in seen:   # appendDeviceSpec :108-118
                    seen.add(host_path)
                    specs.append(dpapi.DeviceSpec(host_path=host_path, container_path=host_path, permissions="mrw"))

            # plan: which devices would be visited, in order, and where a lookup error would stop
            plan, lookup_error_at = plans[r] if plans is not None else self._plan(req)
            if decided is not None:
                bad, panic, egm_paths = next(decided)
            else:
                pairs = [(d.addr, group) for _, group, members in plan for d in members]
                bad, panic = self.revalidate(pairs), None    # ONE batch for the whole container request
                egm_paths = None
            pos = 0
            for bdf, group, members in plan:   # replay in the reference's order: the FIRST error wins
                addrs, found = [], False
                for dev in members:
                    if bad is not None and pos == bad:
                        if panic is not None:   # the reference's vendor read of this member panics
                            raise panic
                        raise AllocateError("invalid allocation request: unknown device: %s" % dev.addr)
                    pos += 1
                    addrs.append(dev.addr)
                    found = found or dev.addr == bdf
                    if iommufd:
                        try:
                            vfiodev = read_vfio_dev(self.base_path, dev.addr)
                        except OSError as e:
                            raise AllocateError("could not determine iommufd device for device %s: %s"
                                                % (dev.addr, e))
                        append_spec(os.path.join(VFIO_DEVICE_PATH, "devices", vfiodev))
                if not found:
                    raise AllocateError("invalid allocation request: unknown device: %s" % bdf)
                append_spec(os.path.join(VFIO_DEVICE_PATH, "vfio"))
                append_spec(os.path.join(VFIO_DEVICE_PATH, group))
                if iommufd:
                    append_spec(IOMMU_DEVICE_PATH)
                env_list.setdefault("%s_%s" % (GPU_PREFIX, self.device_name.upper()), []).extend(addrs)
            if lookup_error_at is not None:
                raise AllocateError("invalid allocation request: unknown device: %s" % lookup_error_at[1])
            if egm_paths is None:
                egm_paths = egm_paths_for_allocated_gpus(list(req.devices_ids), egm_devices)
            for path in egm_paths:
                append_spec(path)
            responses.container_responses.append(dpapi.ContainerAllocateResponse(
                envs={k: ",".join(v) for k, v in env_list.items()}, devices=specs))   # buildEnv :100-106
        return responses


class GenericVGpuDevicePlugin(_PluginBase):
    """The vGPU plugin (generic_vgpu_device_plugin.go).  `check` is the Allocate-time re-check of the type labels
    (MdevLabelCheck: one GPU call per AllocateRequest); without it each ID is read and its label built on the CPU."""
    vgpu = True

    def __init__(self, device_name, device_path, devs, *, vgpu_base_path="/sys/bus/mdev/devices",
                 read_vgpu_id=None, check=None, **kw):
        super().__init__(device_name, devs, **kw)
        self.device_path, self.vgpu_base_path = device_path, vgpu_base_path
        self.read_vgpu_id = read_vgpu_id or _read_vgpu_label
        self.check = check

    def GetPreferredAllocation(self, request, context):
        # "has not been implemented" in the reference: returns (nil, nil) (:262-271) -> empty message
        return dpapi.PreferredAllocationResponse()

    def Allocate(self, request, context):
        """:208-245 — ids whose type label no longer equals the plugin's name are skipped, not errors.  With a check,
        the IDs of all container requests go to it in one call, in request order."""
        reqs = list(request.container_requests)
        if self.check is not None:
            ok = iter(self.check(self.device_name, [dev_id for req in reqs for dev_id in req.devices_ids]))

            def keep(dev_id):
                return bool(next(ok))
        else:
            def keep(dev_id):
                label, err = self.read_vgpu_id(self.vgpu_base_path, dev_id, "mdev_type/name")
                return not err and label == self.device_name
        responses = dpapi.AllocateResponse()
        for req in reqs:
            env_list = {}
            for dev_id in req.devices_ids:
                if not keep(dev_id):
                    continue
                env_list.setdefault("%s_%s" % (VGPU_PREFIX, self.device_name.upper()), []).append(dev_id)
            spec = dpapi.DeviceSpec(host_path=VFIO_DEVICE_PATH, container_path=VFIO_DEVICE_PATH, permissions="mrw")
            responses.container_responses.append(dpapi.ContainerAllocateResponse(
                envs={k: ",".join(v) for k, v in env_list.items()}, devices=[spec]))
        return responses


class MdevLabelCheck:
    """The vGPU plugin's Allocate-time re-check (generic_vgpu_device_plugin.go:216-228) with the label rule on the
    GPU.  Every ID's mdev_type/name is read with the reference's raw reader, in request order; the files that were
    read go to ONE `label_match` call (Context.mdev_label_match), which builds each label and compares it with the
    plugin's name.  An ID whose read failed never reaches the rule and is not kept."""

    def __init__(self, label_match, vgpu_base_path: str = "/sys/bus/mdev/devices", read_raw=_read_vgpu_raw):
        self.label_match, self.vgpu_base_path, self.read_raw = label_match, vgpu_base_path, read_raw

    def __call__(self, device_name, ids) -> list:
        """One bool per ID: its label equals device_name."""
        out, files, at = [False] * len(ids), [], []
        for i, dev_id in enumerate(ids):
            raw, err = self.read_raw(self.vgpu_base_path, dev_id, "mdev_type/name")
            if not err:
                files.append(raw)
                at.append(i)
        if files:
            for i, m in zip(at, self.label_match(files, device_name)):
                out[i] = bool(m)
        return out


class NumaPacker:
    """GetPreferredAllocation's NUMA packing (generic_device_plugin.go:470-608) on the GPU: a drop-in `prefer` for
    GenericDevicePlugin, with preferred_allocation, which stays, as the reference it is tested against.

    `call` is Context.preferred_allocation.  From the plugin's devices it builds ID -> NUMA node, where the last entry
    with topology wins; a node of -1, a device without topology and an ID the plugin does not know all become
    PREF_NODE_NONE, the reference's -1.  Per container request the ID strings (must-include first, then available)
    are interned into handles and the node values into dense indices.  ONE call covers every container request of a
    PreferredAllocationRequest; the positions it returns map back to the ID strings.  Which device is preferred is
    decided by the kernel alone."""

    def __init__(self, call):
        self.call = call

    def __call__(self, devs, requests) -> list:
        """devs: [(device id, numa node or None)]; requests: [(available, must_include, size)] in request order.
        Returns the preferred IDs per request, or raises AllocateError with the reference's text for the first
        request that fails."""
        node_of = {d: n for d, n in devs if n is not None}
        ids, n_must, n_avail, sizes, entries = [], [], [], [], []
        for available, must, size in requests:
            handles, nodes, ent = {}, {}, list(must) + list(available)
            for dev_id in ent:
                node = node_of.get(dev_id, -1)
                ids.append((handles.setdefault(dev_id, len(handles)),
                            L.PREF_NODE_NONE if node == -1 else nodes.setdefault(node, len(nodes))))
            n_must.append(len(must))
            n_avail.append(len(available))
            sizes.append(size)
            entries.append(ent)
        out = self.call(np.array(ids, dtype=L.PREF_ID), n_must, n_avail, sizes)
        for (n, p, _), size in zip(out, sizes):
            if n < 0:
                raise AllocateError("number of MustIncludeDeviceIDs (%d) exceeds allocation size (%d)" % (p, size))
        return [[ent[k] for k in pos] for ent, (_, _, pos) in zip(entries, out)]


def _read_vgpu_label(base, addr, prop):
    """readVgpuIDFromFileFunc :334-344 for ONE id at Allocate time: trim '\\n', \\s+ -> '_'."""
    import re
    raw, err = _read_vgpu_raw(base, addr, prop)
    if err:
        return "", True
    return re.sub(rb"[\t\n\f\r ]+", b"_", raw.strip(b"\n")).decode("latin-1"), False


def plugins_from_specs(specs, maps: Maps, revalidate, vgpu_check=None, prefer=None, allocate_check=None, **kw) -> list:
    """createDevicePlugins' server half (device_plugin.go:99-157): one plugin object per spec.  `revalidate` is the
    passthrough plugins' Allocate-time re-check, `allocate_check` their Allocate decisions in one call per
    AllocateRequest (AllocateCheck; None: `revalidate` and the CPU EGM rule), `vgpu_check` the vGPU plugins' re-check
    (None: the CPU rule), `prefer` the passthrough plugins' GetPreferredAllocation (None: the CPU rule)."""
    out = []
    for spec in specs:
        devs = devices_from_spec(spec)
        if spec.vgpu:
            out.append(GenericVGpuDevicePlugin(spec.device_name, "vgpu", devs, check=vgpu_check,
                                               **{k: v for k, v in kw.items() if k in ("socket_dir", "kubelet_socket",
                                                                                          "vgpu_base_path")}))
        else:
            out.append(GenericDevicePlugin(spec.device_name, VFIO_DEVICE_PATH, devs, maps, revalidate=revalidate,
                                           prefer=prefer, allocate_check=allocate_check,
                                           **{k: v for k, v in kw.items() if k != "vgpu_base_path"}))
    return out


# ------------------------------------------------------------------------------------------------
# health feed driven by the K6 delta kernel (SURVEY.md 8(f) rank 3)
# ------------------------------------------------------------------------------------------------
class _PollFeed:
    """A feed polled on a daemon thread: start() calls self.tick() every period_s seconds until stop()."""

    def __init__(self, period_s: float):
        self.period_s = period_s
        self._stop = threading.Event()
        self._thread = None

    def start(self):
        def loop():
            while not self._stop.is_set():
                self.tick()
                time.sleep(self.period_s)
        self._thread = threading.Thread(target=loop, daemon=True)
        self._thread.start()

    def stop(self):
        self._stop.set()
        if self._thread:
            self._thread.join(2.0)


class HealthRescanFeed(_PollFeed):
    """Periodic re-snapshot -> Context.health_rescan (K6) -> healthy / unhealthy events.

    `snapshot()` returns (records, ids): the PCI snapshot in a FIXED device order and the device id
    of every record.  Each transition the kernel reports ((index << 1) | alive) is routed to the
    plugin that advertises that id.  The first tick only establishes the alive set."""

    def __init__(self, health_rescan, snapshot, plugins, period_s: float = 0.001):
        super().__init__(period_s)
        self.health_rescan, self.snapshot = health_rescan, snapshot
        self.owner = {d.ID: p for p in plugins for d in p.devs}
        self._primed = False

    def tick(self) -> int:
        recs, ids = self.snapshot()
        delta = self.health_rescan(recs)
        sent = 0
        if self._primed:
            for word in delta.changed:
                idx, alive = int(word) >> 1, int(word) & 1
                plugin = self.owner.get(ids[idx])
                if plugin is not None:
                    (plugin.healthy if alive else plugin.unhealthy)(ids[idx])
                    sent += 1
        self._primed = True
        return sent


# ------------------------------------------------------------------------------------------------
# hot-plug feeds driven by the K7 re-scan deltas
# ------------------------------------------------------------------------------------------------
class _RescanFeed(_PollFeed):
    """The plugin lifecycle both re-scan feeds share; a subclass supplies tick()."""

    def __init__(self, scan_delta, snapshot, maps: Maps, plugins: dict, make_plugin, period_s: float):
        super().__init__(period_s)
        self.scan_delta, self.snapshot, self.maps = scan_delta, snapshot, maps
        self.plugins, self.make_plugin = plugins, make_plugin
        self._prev_snap = None

    def _follow(self, dirty: Maps, gone: list):
        """The plugins of the dirty keys (`dirty` holds their maps) get their new device list, or are started and
        registered when the key is new; the plugins of the keys that went are stopped."""
        for spec in plugin_specs_from_maps(dirty):
            plugin = self.plugins.get(spec.key)
            if plugin is None:
                plugin = self.make_plugin(spec)
                plugin.start()
                self.plugins[spec.key] = plugin
            else:
                plugin.set_devices(devices_from_spec(spec))
        for key in gone:
            plugin = self.plugins.pop(key, None)
            if plugin is not None:
                plugin.stop()


class PciRescanFeed(_RescanFeed):
    """Periodic re-snapshot -> Context.scan_pci_delta (K7) -> the shared maps and the set of passthrough plugins.

    `snapshot()` returns a PciSnapshot, `scan_delta(recs)` is Context.scan_pci_delta, `plugins` maps deviceMap keys
    to running plugins and `make_plugin(spec)` builds one for a new key.  Each tick patches `maps` in place (Allocate
    reads iommuMap / bdfToIommuMap from it, so it sees a moved device at once), gives every plugin whose key is
    dirty its new device list, starts and registers a plugin for every new key, and stops the plugin of every key
    that went.  The first tick has no previous snapshot: it rebuilds the maps and treats every key as dirty.

    raw=True runs the feed from raw reads: `snapshot()` returns a PciRaw (plugin.read_pci_tree_raw) and
    `scan_delta(raw)` is Context.scan_pci_raw_delta, whose delta is keyed by entry name, so a tick patches the maps
    and re-sends only the dirty keys in every snapshot mode.  name_of (Context.name_lookup) names device keys when
    the snapshot carries device strings in index mode."""

    def __init__(self, scan_delta, snapshot, maps: Maps, plugins: dict, make_plugin, period_s: float = 0.01,
                 raw: bool = False, name_of=None):
        super().__init__(scan_delta, snapshot, maps, plugins, make_plugin, period_s)
        self.raw, self.name_of = raw, name_of

    def tick(self):
        if self.raw:
            res, snap, delta = self.scan_delta(self.snapshot())
        else:
            snap = self.snapshot()
            res, delta = self.scan_delta(snap.recs)
        if self._prev_snap is None:
            touched = _rebuild_pci_maps(self.maps, res, snap, self.name_of)
        else:
            touched = apply_pci_delta(self.maps, res, delta, snap, self._prev_snap, name_of=self.name_of)
        self._prev_snap = snap
        self._follow(Maps(deviceMap={k: self.maps.deviceMap[k] for k in touched.dev_dirty},
                          deviceNames=self.maps.deviceNames), touched.dev_gone)
        return touched


class MdevRescanFeed(_RescanFeed):
    """Periodic re-snapshot -> Context.scan_mdev_delta (K7) -> the shared maps and the set of vGPU plugins.

    `snapshot()` returns an MdevSnapshot, `scan_delta(recs, raw_types)` is Context.scan_mdev_delta, `plugins` maps
    vGpuMap keys (labels) to running plugins and `make_plugin(spec)` builds a GenericVGpuDevicePlugin for a new label.
    Each tick patches vGpuMap / gpuVgpuMap of `maps` in place (an XidEventRouter holding maps.gpuVgpuMap sees a new
    vGPU at once), re-sends the device list of every plugin whose label is dirty (a NUMA move re-sends topology),
    starts and registers a plugin for every new label, and stops the plugin of every label that went.  The first
    tick has no previous snapshot: it rebuilds the maps and treats every key as dirty.

    raw=True runs the feed from raw reads: `snapshot()` returns an MdevRaw (plugin.read_mdev_tree_raw) and
    `scan_delta(raw)` is Context.scan_mdev_raw_delta, whose delta is keyed by entry name, so a tick patches the maps
    and re-sends only the dirty labels in every snapshot mode."""

    def __init__(self, scan_delta, snapshot, maps: Maps, plugins: dict, make_plugin, period_s: float = 0.01,
                 raw: bool = False):
        super().__init__(scan_delta, snapshot, maps, plugins, make_plugin, period_s)
        self.raw = raw

    def tick(self):
        if self.raw:
            res, snap, delta = self.scan_delta(self.snapshot())
        else:
            snap = self.snapshot()
            res, delta = self.scan_delta(snap.recs, snap.raw_types)
        if self._prev_snap is None:
            touched = _rebuild_mdev_maps(self.maps, res, res, snap)
        else:
            touched = apply_mdev_delta(self.maps, res, delta, snap, self._prev_snap)
        self._prev_snap = snap
        self._follow(Maps(vGpuMap={k: self.maps.vGpuMap[k] for k in touched.type_dirty},
                          deviceNames=self.maps.deviceNames), touched.type_gone)
        return touched


# ------------------------------------------------------------------------------------------------
# NVML XID events -> vGPU health (generic_vgpu_device_plugin.go:330-339 and watchXIDsFunc :387-433)
# ------------------------------------------------------------------------------------------------
XID_APPLICATION_ERRORS = (31, 43, 45)   # :413-417 "Application errors: the GPU should still be healthy"


class XidEventRouter:
    """The decision logic between an NVML XidCriticalError event and the `unhealthy` channel of a vGPU plugin,
    without NVML itself (the binding stays in the Go host; out of scope here):

      on_event(xid, uuid)    XIDs 31 / 43 / 45 are ignored (:415); an event without a device UUID marks EVERY GPU
                             (:419-424); otherwise the GPU with that UUID (:427-431)
      on_unsupported(uuid)   registration failed with "Not Supported": that GPU is marked at once (:392-397)
      a marked GPU           -> every vGPU of returnGpuVgpuMap()[gpu.PCI.BusID] goes to plugin.unhealthy (:333-338)

    `gpus`: list of (uuid, bus_id) in NVML enumeration order; `gpu_vgpu_map`: the scan's gpuVgpuMap
    (parent BDF -> [mdev uuid]); `plugins`: the vGPU plugins (an id is routed to the plugin that advertises it;
    the reference sends it down ITS OWN channel whether or not the id is its own — ListAndWatch then finds no
    such device and changes nothing, :186-199)."""

    def __init__(self, gpus, gpu_vgpu_map, plugins):
        self.gpus, self.gpu_vgpu_map = list(gpus), gpu_vgpu_map
        self.owner = {d.ID: p for p in plugins for d in p.devs}

    def _mark(self, bus_id) -> int:
        sent = 0
        for vgpu in self.gpu_vgpu_map.get(bus_id, []):
            plugin = self.owner.get(vgpu)
            if plugin is not None:
                plugin.unhealthy(vgpu)
                sent += 1
        return sent

    def on_unsupported(self, uuid) -> int:
        return sum(self._mark(bus) for u, bus in self.gpus if u == uuid)

    def on_event(self, xid: int, uuid=None) -> int:
        if xid in XID_APPLICATION_ERRORS:
            return 0
        if not uuid:
            return sum(self._mark(bus) for _, bus in self.gpus)
        return sum(self._mark(bus) for u, bus in self.gpus if u == uuid)


class VgpuHealthFeed(_PollFeed):
    """The vGPU health check of generic_vgpu_device_plugin.go:280-385 on the GPU: periodic re-snapshot plus the XID
    events since the last tick -> Context.health_rescan_mdev (K6) -> healthy / unhealthy events.

      device path   an mdev whose entry vanishes (or stops passing createVgpuIDMap's keep rule) goes unhealthy, and
                    healthy again when it returns (Create / Remove / Rename, :340-351)
      XID           on_event / on_unsupported queue the bus ids of the GPUs to mark, with XidEventRouter's filters
                    (31 / 43 / 45 ignored, no UUID = every GPU, :392-424); each vGPU on such a GPU goes unhealthy and
                    stays so until its path is created again (:330-339)

    `health_rescan_mdev(recs, n_types, xid_parents)` is Context.health_rescan_mdev; `snapshot(uuids, intern)` returns
    an MdevSnapshot of `uuids` in that order with parent handles from `intern` (plugin.snapshot_mdev_ids over the
    sysfs paths); `plugins` are the vGPU plugins, whose devices are the advertised UUIDs; `gpus` is [(nvml_uuid,
    bus_id)] as in XidEventRouter.  A bus id resolves through the same intern dict as the sysfs parent strings, so
    a bus id string that differs from the parent's sysfs name marks nothing, as the reference's map lookup misses.

    tick(): snapshot, take the queued bus ids, one kernel call, then each transition to the plugin advertising that
    UUID.  An arming tick (the first, or one whose UUID list differs from the previous tick's) resets the state and
    sends each vGPU whose health differs from what its plugin advertises, so a vGPU already absent, or on a GPU marked
    before the first tick, goes unhealthy at once.  Deliberate difference: only transitions are sent, where the
    reference re-sends `unhealthy` for a vGPU already unhealthy on every repeated XID (ListAndWatch then re-sends an
    unchanged list)."""

    def __init__(self, health_rescan_mdev, snapshot, plugins, gpus, period_s: float = 0.001):
        super().__init__(period_s)
        self.health_rescan_mdev, self.snapshot = health_rescan_mdev, snapshot
        self.plugins, self.gpus = list(plugins), list(gpus)
        self.intern = {}
        self._uuids = None
        self._queued = []
        self._lock = threading.Lock()

    def _queue(self, buses) -> int:
        with self._lock:
            self._queued.extend(buses)
        return len(buses)

    def on_unsupported(self, uuid) -> int:
        return self._queue([bus for u, bus in self.gpus if u == uuid])

    def on_event(self, xid: int, uuid=None) -> int:
        if xid in XID_APPLICATION_ERRORS:
            return 0
        return self._queue([bus for u, bus in self.gpus if not uuid or u == uuid])

    def tick(self) -> int:
        devs = [(d, p) for p in self.plugins for d in p.devs]
        uuids = [d.ID for d, _ in devs]
        snap = self.snapshot(uuids, self.intern)
        with self._lock:
            buses, self._queued = self._queued, []
        xids = [self.intern[b] for b in buses if b in self.intern]
        arming = uuids != self._uuids
        if arming:
            self.health_rescan_mdev(snap.recs[:0], len(snap.raw_types))    # a different n re-arms the state
            self._uuids = uuids
        delta = self.health_rescan_mdev(snap.recs, len(snap.raw_types), xids)
        return _send_health(devs, delta, arming)


def _send_health(devs, delta, arming: bool) -> int:
    """Route a health delta over [(device, plugin)] (record k = devs[k]) to the plugins' channels.  On an arming tick
    (the state was just re-armed, so every healthy record is listed) send each device whose health differs from what
    its plugin advertises; otherwise send each transition.  Returns the number of events sent."""
    sent = 0
    if arming:
        healthy = np.zeros(len(devs), dtype=bool)
        ch = np.asarray(delta.changed, dtype=np.int64)
        healthy[ch[(ch & 1) == 1] >> 1] = True
        for k, (d, plugin) in enumerate(devs):
            if (d.health == dpapi.HEALTHY) != healthy[k]:
                (plugin.healthy if healthy[k] else plugin.unhealthy)(d.ID)
                sent += 1
        return sent
    for word in delta.changed:
        k, ok = int(word) >> 1, int(word) & 1
        d, plugin = devs[k]
        (plugin.healthy if ok else plugin.unhealthy)(d.ID)
        sent += 1
    return sent


class GroupHealthFeed(_PollFeed):
    """The passthrough health check of generic_device_plugin.go:611-690 on the GPU: periodic re-snapshot plus one
    listing of the VFIO device directory -> Context.health_rescan_groups (K6) -> healthy / unhealthy events.

      device node   every device of an IOMMU group goes unhealthy when /dev/vfio/<group> vanishes (Remove / Rename)
                    and healthy when it returns (Create), :659-668
      sysfs         a device whose record stops passing createIommuDeviceMap's filter goes unhealthy, as with
                    HealthRescanFeed, and healthy again when it passes and its node exists

    `health_rescan_groups(recs, group_nodes)` is Context.health_rescan_groups; `snapshot(bdfs, intern)` returns a
    PciSnapshot of `bdfs` in that order with group handles from `intern` (plugin.snapshot_pci_ids over the sysfs
    tree); `list_nodes(intern)` returns the handles of the groups whose node exists (plugin.group_nodes over the device
    directory), resolved through the same dict, so a node no advertised device's group has is ignored; `plugins` are
    the passthrough plugins, whose devices are the advertised BDFs.

    tick(): snapshot, list the nodes, one kernel call, then each transition to the plugin advertising that BDF.  An
    arming tick (the first, or one whose BDF list differs from the previous tick's) resets the state and sends each
    device whose health differs from what its plugin advertises, so a device whose node is already absent goes
    unhealthy at once.  Deliberate difference: only transitions are sent, where the reference re-sends `healthy` for
    every device of a group on a repeated Create of its node (ListAndWatch then re-sends an unchanged list)."""

    def __init__(self, health_rescan_groups, snapshot, list_nodes, plugins, period_s: float = 0.001):
        super().__init__(period_s)
        self.health_rescan_groups, self.snapshot, self.list_nodes = health_rescan_groups, snapshot, list_nodes
        self.plugins = list(plugins)
        self.intern = {}
        self._bdfs = None

    def tick(self) -> int:
        devs = [(d, p) for p in self.plugins for d in p.devs]
        bdfs = [d.ID for d, _ in devs]
        snap = self.snapshot(bdfs, self.intern)
        nodes = self.list_nodes(self.intern)
        arming = bdfs != self._bdfs
        if arming:
            self.health_rescan_groups(snap.recs[:0])      # a different n re-arms the state
            self._bdfs = bdfs
        delta = self.health_rescan_groups(snap.recs, nodes)
        return _send_health(devs, delta, arming)


def _uuid_key(s: str) -> bytes:
    """The UUID bytes of a canonical (lower-case, hyphenated) UUID string; ValueError naming anything else."""
    h = s.replace("-", "") if isinstance(s, str) else ""
    if len(s) == 36 and len(h) == 32 and all(c in "0123456789abcdef" for c in h) and format_uuid(bytes.fromhex(h)) == s:
        return bytes.fromhex(h)
    raise ValueError("not a canonical vGPU UUID, so it has no stable key: %r" % (s,))


def _bdf_key(s: str) -> int:
    """The packed address of a canonical BDF string; ValueError naming anything else."""
    p = parse_bdf(s) if isinstance(s, str) else None
    if p is None:
        raise ValueError("not a canonical PCI address, so it has no stable key: %r" % (s,))
    return p


def _by_key(plugins, key):
    """[(device, plugin)] of every advertised device, ascending by key(device ID): the record order of a keyed call."""
    devs = [(d, p) for p in plugins for d in p.devs]
    keys = [key(d.ID) for d, _ in devs]
    return [devs[k] for k in sorted(range(len(devs)), key=keys.__getitem__)]


def _send_keyed_health(devs, delta, prev_ids) -> int:
    """Route a keyed health delta over [(device, plugin)] (record k = devs[k]).  A device whose ID was in the previous
    tick's list gets each transition; a new one (prior state "nothing", so it is listed iff it is healthy now) is sent
    only when that differs from what its plugin advertises.  A tick whose list did not change walks the listed
    records only.  Returns the number of events sent."""
    sent = 0
    listed_new = set()
    for w in delta.changed:
        k, ok = int(w) >> 1, int(w) & 1
        d, plugin = devs[k]
        if d.ID not in prev_ids:
            listed_new.add(k)
            if d.health == dpapi.HEALTHY:
                continue
        (plugin.healthy if ok else plugin.unhealthy)(d.ID)
        sent += 1
    ids = [d.ID for d, _ in devs]
    if len(ids) != len(prev_ids) or not prev_ids.issuperset(ids):
        for k, i in enumerate(ids):   # new and not listed: unhealthy now
            if i not in prev_ids and k not in listed_new and devs[k][0].health == dpapi.HEALTHY:
                devs[k][1].unhealthy(i)
                sent += 1
    return sent


class KeyedVgpuHealthFeed(VgpuHealthFeed):
    """VgpuHealthFeed on Context.health_rescan_mdev_keyed: the state is kept per UUID, so it survives changes of the
    advertised list (MdevRescanFeed's set_devices).  A vGPU marked by an XID stays unhealthy while it stays advertised,
    whatever other vGPUs are created or destroyed; only its own path being created again clears the mark.

    Construct it as VgpuHealthFeed, with `health_rescan_mdev` = Context.health_rescan_mdev_keyed.  tick(): order the
    advertised vGPUs by UUID bytes, snapshot them in that order, one keyed call (never an arming call), then each
    transition of a UUID that was advertised on the previous tick; a new UUID is sent only when the kernel's health
    differs from what its plugin advertises.  Every advertised ID must be a canonical UUID (ValueError names the first
    that is not): a Walk-index handle is not a stable identity, so names that are not UUIDs need VgpuHealthFeed, whose
    state follows the record index.

    raw=True runs the feed from raw reads, with no intern dict: `health_rescan_mdev(raw, xid_parents)` is
    Context.health_rescan_mdev_raw, `snapshot(names)` returns an MdevRaw of `names` in that order
    (plugin.read_mdev_ids_raw over the sysfs paths).  The advertised IDs are ordered by os.fsencode(ID) and may take
    any form; the state is kept per name.  The queued bus ids go to the call as strings, matched byte for byte against
    the parents the GPU decodes from the link targets, as the reference's gpuVgpuMap[busID] lookup matches them."""

    def __init__(self, health_rescan_mdev, snapshot, plugins, gpus, period_s: float = 0.001, raw: bool = False):
        super().__init__(health_rescan_mdev, snapshot, plugins, gpus, period_s)
        self.raw = raw

    def tick(self) -> int:
        if self.raw:
            devs = _by_key(self.plugins, os.fsencode)
            names = [d.ID for d, _ in devs]
            raw = self.snapshot(names)
            with self._lock:
                buses, self._queued = self._queued, []
            delta = self.health_rescan_mdev(raw, buses)
            prev, self._uuids = self._uuids or frozenset(), frozenset(names)
            return _send_keyed_health(devs, delta, prev)
        devs = _by_key(self.plugins, _uuid_key)
        uuids = [d.ID for d, _ in devs]
        snap = self.snapshot(uuids, self.intern)
        with self._lock:
            buses, self._queued = self._queued, []
        xids = [self.intern[b] for b in buses if b in self.intern]
        delta = self.health_rescan_mdev(snap.recs, len(snap.raw_types), xids)
        prev, self._uuids = self._uuids or frozenset(), frozenset(uuids)
        return _send_keyed_health(devs, delta, prev)


class KeyedGroupHealthFeed(GroupHealthFeed):
    """GroupHealthFeed on Context.health_rescan_groups_keyed: the state is kept per address, so a change of the
    advertised list costs no arming call and no sweep over every device.

    Construct it as GroupHealthFeed, with `health_rescan_groups` = Context.health_rescan_groups_keyed.  tick(): order
    the advertised devices by packed BDF, snapshot them in that order, list the nodes, one keyed call, then each
    transition of an address advertised on the previous tick; a new address is sent only when the kernel's health
    differs from what its plugin advertises.  Every advertised ID must be a canonical BDF (ValueError names the first
    that is not); other names need GroupHealthFeed.

    raw=True runs the feed from raw reads, with no intern dict: `health_rescan_groups(raw, nodes)` is
    Context.health_rescan_groups_raw, `snapshot(names)` returns a PciRaw of `names` in that order
    (plugin.read_pci_ids_raw over the sysfs tree) and `list_nodes()` the raw names of one listing of the VFIO directory
    (plugin.list_nodes_raw).  The advertised IDs are ordered by os.fsencode(ID) and may take any form; the state is
    kept per name, and a group's node is matched by its name's bytes, as the reference joins the directory with the
    group string (generic_device_plugin.go:639-676)."""

    def __init__(self, health_rescan_groups, snapshot, list_nodes, plugins, period_s: float = 0.001,
                 raw: bool = False):
        super().__init__(health_rescan_groups, snapshot, list_nodes, plugins, period_s)
        self.raw = raw

    def tick(self) -> int:
        if self.raw:
            devs = _by_key(self.plugins, os.fsencode)
            names = [d.ID for d, _ in devs]
            delta = self.health_rescan_groups(self.snapshot(names), self.list_nodes())
            prev, self._bdfs = self._bdfs or frozenset(), frozenset(names)
            return _send_keyed_health(devs, delta, prev)
        devs = _by_key(self.plugins, _bdf_key)
        bdfs = [d.ID for d, _ in devs]
        snap = self.snapshot(bdfs, self.intern)
        nodes = self.list_nodes(self.intern)
        delta = self.health_rescan_groups(snap.recs, nodes)
        prev, self._bdfs = self._bdfs or frozenset(), frozenset(bdfs)
        return _send_keyed_health(devs, delta, prev)


# ------------------------------------------------------------------------------------------------
# a mock kubelet: Registration server + DevicePlugin client (SURVEY.md 8(f) rank 1)
# ------------------------------------------------------------------------------------------------
@dataclass
class Registration:
    version: str
    endpoint: str
    resource_name: str
    options: object = None


class PluginClient:
    """What the kubelet's device manager does with a registered endpoint."""

    def __init__(self, socket_path: str):
        import grpc
        self.channel = grpc.insecure_channel("unix://" + socket_path)
        grpc.channel_ready_future(self.channel).result(timeout=CONNECTION_TIMEOUT)
        self._calls = {}
        for mname, (req, resp, stream) in dpapi.SERVICES["DevicePlugin"].items():
            make = self.channel.unary_stream if stream else self.channel.unary_unary
            self._calls[mname] = make(dpapi.method_path("DevicePlugin", mname),
                                      request_serializer=dpapi.MESSAGES[req].SerializeToString,
                                      response_deserializer=dpapi.MESSAGES[resp].FromString)

    def options(self):
        return self._calls["GetDevicePluginOptions"](dpapi.Empty(), timeout=CONNECTION_TIMEOUT)

    def list_and_watch(self):
        return self._calls["ListAndWatch"](dpapi.Empty())

    def allocate(self, *container_device_ids):
        req = dpapi.AllocateRequest(container_requests=[dpapi.ContainerAllocateRequest(devices_ids=list(ids))
                                                        for ids in container_device_ids])
        return self._calls["Allocate"](req, timeout=CONNECTION_TIMEOUT)

    def preferred_allocation(self, available, must_include, size):
        req = dpapi.PreferredAllocationRequest(container_requests=[dpapi.ContainerPreferredAllocationRequest(
            available_deviceIDs=list(available), must_include_deviceIDs=list(must_include), allocation_size=size)])
        return self._calls["GetPreferredAllocation"](req, timeout=CONNECTION_TIMEOUT)

    def close(self):
        self.channel.close()


@dataclass
class MockKubelet:
    """Serves v1beta1.Registration on <socket_dir>/kubelet.sock and remembers who registered."""
    socket_dir: str
    registrations: list = field(default_factory=list)

    def __post_init__(self):
        self.socket_path = os.path.join(self.socket_dir, "kubelet.sock")
        self._cv = threading.Condition()
        self.server = None

    def _register(self, request, context):
        with self._cv:
            self.registrations.append(Registration(request.version, request.endpoint, request.resource_name,
                                                   request.options))
            self._cv.notify_all()
        return dpapi.Empty()

    def start(self):
        import grpc
        try:
            os.remove(self.socket_path)
        except FileNotFoundError:
            pass
        self.server = grpc.server(futures.ThreadPoolExecutor(max_workers=4))
        handler = grpc.unary_unary_rpc_method_handler(
            self._register, request_deserializer=dpapi.RegisterRequest.FromString,
            response_serializer=dpapi.Empty.SerializeToString)
        self.server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler(
            dpapi.service_name("Registration"), {"Register": handler}),))
        self.server.add_insecure_port("unix://" + self.socket_path)
        self.server.start()
        return self

    def wait_for(self, n: int, timeout: float = CONNECTION_TIMEOUT) -> list:
        with self._cv:
            self._cv.wait_for(lambda: len(self.registrations) >= n, timeout)
            return list(self.registrations)

    def connect(self, registration: Registration) -> PluginClient:
        return PluginClient(os.path.join(self.socket_dir, registration.endpoint))

    def stop(self):
        if self.server is not None:
            self.server.stop(0.2).wait(2.0)
            self.server = None
        try:
            os.remove(self.socket_path)
        except FileNotFoundError:
            pass


# ------------------------------------------------------------------------------------------------
# healthCheck(): the reference's own health source (generic_device_plugin.go:611-690) — inotify on the
# device nodes and on the plugin socket.  (HealthRescanFeed above is the GPU-side alternative.)
# ------------------------------------------------------------------------------------------------
class DeviceNodeWatcher:
    """Watches <device_path>/<iommu group> for every advertised device and the plugin's own socket:

      node created            -> healthy(id)   for every device of that group   (:659-662)
      node removed / renamed  -> unhealthy(id)                                   (:663-668)
      plugin socket removed   -> kubelet restarted: restart() = Stop + Start + Register (:669-679).  The
                                 reference's Start() spawns a fresh healthCheck goroutine and the old one
                                 returns; here the SAME watcher keeps running (its inotify watches are on the
                                 parent directories and survive), so every later restart is handled too.

    For a vGPU plugin the watched nodes are <vgpu_base_path>/<uuid> (generic_vgpu_device_plugin.go:319-351).

    fsnotify watches the PARENT directories; so does this (inotify through libc, no extra package)."""
    IN_CREATE, IN_DELETE, IN_MOVED_FROM, IN_DELETE_SELF, IN_MOVE_SELF = 0x100, 0x200, 0x40, 0x400, 0x800

    def __init__(self, plugin: GenericDevicePlugin, bdf_to_iommu=None):
        import ctypes
        self.plugin = plugin
        self._libc = ctypes.CDLL("libc.so.6", use_errno=True)
        self._fd = self._libc.inotify_init1(0o4000)          # IN_NONBLOCK
        if self._fd < 0:
            raise OSError(ctypes.get_errno(), "inotify_init1")
        self.path_devices = {}                               # node path -> [device ids]
        if getattr(plugin, "vgpu", False):
            for dev in plugin.devs:                          # one node per mediated device
                self.path_devices.setdefault(os.path.join(plugin.vgpu_base_path, dev.ID), []).append(dev.ID)
        else:
            bdf_to_iommu = bdf_to_iommu if bdf_to_iommu is not None else plugin.maps.bdfToIommuMap
            for dev in plugin.devs:
                group = bdf_to_iommu.get(dev.ID)
                if group is None:                            # :634-637 logged and skipped
                    continue
                self.path_devices.setdefault(os.path.join(plugin.device_path, group), []).append(dev.ID)
        self._wd_dir = {}
        dirs = {os.path.dirname(p) for p in self.path_devices} | {os.path.dirname(plugin.socket_path)}
        mask = self.IN_CREATE | self.IN_DELETE | self.IN_MOVED_FROM
        for d in sorted(dirs):
            wd = self._libc.inotify_add_watch(self._fd, d.encode(), mask)
            if wd < 0:
                err = ctypes.get_errno()
                os.close(self._fd)
                raise OSError(err, "inotify_add_watch(%s)" % d)
            self._wd_dir[wd] = d
        self._stop = threading.Event()
        self._thread = None
        self.restarted = threading.Event()
        self.restarts = 0

    def poll_once(self) -> int:
        """Drain pending inotify events; returns how many health / restart actions were taken."""
        import struct
        try:
            buf = os.read(self._fd, 65536)
        except BlockingIOError:
            return 0
        acted, off = 0, 0
        while off + 16 <= len(buf):
            wd, mask, _cookie, ln = struct.unpack_from("iIII", buf, off)
            name = buf[off + 16:off + 16 + ln].split(b"\0", 1)[0].decode()
            off += 16 + ln
            path = os.path.join(self._wd_dir.get(wd, ""), name)
            ids = self.path_devices.get(path)
            if ids is not None:
                if mask & self.IN_CREATE:
                    for i in ids:
                        self.plugin.healthy(i)
                    acted += len(ids)
                elif mask & (self.IN_DELETE | self.IN_MOVED_FROM):
                    for i in ids:
                        self.plugin.unhealthy(i)
                    acted += len(ids)
            elif path == self.plugin.socket_path and mask & self.IN_DELETE:
                self.plugin.restart()
                self.restarts += 1
                self.restarted.set()
                acted += 1
        return acted

    def start(self, period_s: float = 0.01):
        def loop():
            while not self._stop.is_set():
                self.poll_once()
                time.sleep(period_s)
        self._thread = threading.Thread(target=loop, daemon=True)
        self._thread.start()

    def stop(self):
        self._stop.set()
        if self._thread:
            self._thread.join(2.0)
        try:
            os.close(self._fd)
        except OSError:
            pass
