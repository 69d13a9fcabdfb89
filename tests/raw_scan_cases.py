"""Raw walk reads for kvg_scan_pci_raw and a Go-exact restatement of what createIommuDeviceMap's readers make of them
(device_plugin.go:202-238, :294-331): numa_node through the oracle's strings.TrimSpace (kvo_trim_space) and a plain
strconv.ParseInt(s, 10, 64).  snapshot_pci_tree and kvg_host.cpp differ from Go on some numa_node bytes; this file is
the reference for those."""
import numpy as np

import kvgpu
from kvgpu import _lib as L
from oracle import oracle as O

MISSING = object()   # the read was not made
FIELDS = ("vendor", "driver", "iommu_group", "numa_node", "device")


class RawError(Exception):
    def __init__(self, kind, entry, field):
        super().__init__("%s at entry %d field %d" % (kind, entry, field))
        self.kind, self.entry, self.field = kind, entry, field


def raw_of(entries) -> kvgpu.PciRaw:
    """entries: [(name bytes, {field: bytes | None (failed) | MISSING})]; a field left out reads as b"" """
    names, parts, state = [], [], []
    for name, e in entries:
        st, row = 0, [name]
        for f, key in enumerate(FIELDS, start=1):
            v = e.get(key, b"")
            if v is MISSING:
                v = b""
            else:
                st |= 1 << f
                if v is None:
                    st |= 1 << (8 + f)
                    v = b""
            row.append(v)
        names.append(name.decode("latin-1"))
        parts.append(row)
        state.append(st)
    lens = [len(x) for row in parts for x in row]
    off = np.zeros(len(lens) + 1, dtype=np.uint32)
    off[1:] = np.cumsum(lens, dtype=np.uint64)
    return kvgpu.PciRaw(names, off, b"".join(x for row in parts for x in row), np.array(state, dtype=np.uint16))


def parse_int64(s: bytes):
    if not s:
        return None
    neg, body = s[:1] == b"-", s[1:] if s[:1] in (b"+", b"-") else s
    if not body or any(c < 0x30 or c > 0x39 for c in body):
        return None
    v = -int(body) if neg else int(body)
    return v if -(1 << 63) <= v < (1 << 63) else None


def _hex4(s: bytes):
    return int(s, 16) if len(s) == 4 and all(c in b"0123456789abcdef" for c in s) else None


def go_snapshot(raw: kvgpu.PciRaw):
    """-> (recs, packed_addr, group_names | None, device_names | None); raises RawError('miss' | 'panic' | 'range')."""
    n = len(raw.state)
    get = lambda i, f: raw.bytes[raw.off[i * 6 + f]:raw.off[i * 6 + f + 1]]
    rows, miss, panic, rng = [], [], [], []
    for i in range(n):
        st = int(raw.state[i])

        def reach(f):
            if not (st >> f) & 1:
                miss.append((i, f))
                return None
            return None if (st >> (8 + f)) & 1 else get(i, f)

        vendor, device, group, driver, flags, numa = 0xFFFF, None, b"", L.DRV_NONE, 0, 0
        go = False
        v = reach(L.RAW_VENDOR)
        if v is None:
            flags |= L.PF_VENDOR_ERR if (st >> L.RAW_VENDOR) & 1 else 0
        elif len(v) < 2:
            panic.append((i, L.RAW_VENDOR))
        else:
            s = v[2:].strip(b"\n")
            vendor = _hex4(s) if _hex4(s) is not None else 0xFFFF
            go = s == b"10de"
        if go:
            d = reach(L.RAW_DRIVER)
            if d is None:
                flags |= L.PF_DRIVER_ERR if (st >> L.RAW_DRIVER) & 1 else 0
                go = False
            else:
                driver = {b"vfio-pci": L.DRV_VFIO_PCI, b"nvgrace_gpu_vfio_pci": L.DRV_NVGRACE}.get(
                    d.rsplit(b"/", 1)[-1], L.DRV_OTHER)
                go = driver != L.DRV_OTHER
        if go:
            g = reach(L.RAW_GROUP)
            if g is None:
                flags |= L.PF_IOMMU_ERR if (st >> L.RAW_GROUP) & 1 else 0
                go = False
            else:
                group = g.rsplit(b"/", 1)[-1]
        if go:
            m = reach(L.RAW_NUMA)
            if m is None:
                flags |= L.PF_NUMA_ERR if (st >> L.RAW_NUMA) & 1 else 0
            else:
                val = parse_int64(O.trim_space(m))
                if val is None:
                    flags |= L.PF_NUMA_ERR
                else:
                    numa = val
                    if not -32768 <= val <= 32767:
                        rng.append((i, L.RAW_NUMA))
            dv = reach(L.RAW_DEVICE)
            if dv is None:
                flags |= L.PF_DEVICE_ERR if (st >> L.RAW_DEVICE) & 1 else 0
            elif len(dv) < 2:
                panic.append((i, L.RAW_DEVICE))
            else:
                device = dv[2:].strip(b"\n")
        rows.append((vendor, device, group, driver, flags, numa))
    if miss:
        raise RawError("miss", *miss[0])
    if panic:
        raise RawError("panic", *panic[0])
    names = [x.encode("latin-1") for x in raw.names]
    packed = [kvgpu.parse_bdf(x.decode("latin-1")) for x in names]
    packed_ok = all(p is not None for p in packed) and all(packed[k] < packed[k + 1] for k in range(n - 1))
    canon = lambda s: s.isdigit() and (s == b"0" or s[:1] != b"0") and int(s) < (1 << 32)
    groups_numeric = all(canon(r[2]) for r in rows if r[2] != b"")
    devices_numeric = all(_hex4(r[1]) is not None for r in rows if r[1] is not None)
    gi, di = {}, {}
    recs = np.zeros(n, dtype=L.PCI_REC)
    for i, (vendor, device, group, driver, flags, numa) in enumerate(rows):
        if device is None:
            dval = 0
        elif devices_numeric:
            dval = _hex4(device)
        else:
            dval = di.setdefault(device, len(di))
            if dval > 0xFFFF:
                rng.append((i, L.RAW_DEVICE))
        if group == b"":
            gval = 0
        elif groups_numeric:
            gval = int(group)
        else:
            gval = gi.setdefault(group, len(gi))
        recs[i] = (packed[i] if packed_ok else i, vendor, dval & 0xFFFF, gval, driver, flags,
                   numa if -32768 <= numa <= 32767 else 0)
    if rng:
        raise RawError("range", *min(rng))
    return (recs, packed_ok, None if groups_numeric else [g.decode("latin-1") for g in gi],
            None if devices_numeric else [d.decode("latin-1") for d in di])


# ---- the edge matrix ---------------------------------------------------------------------------------------------
VENDORS = [b"0x10de\n", b"0x10DE\n", b"0x10de\n\n", b"10de", b"0x10de", b"0x8086\n", b"0xffff\n", b"0x\n"]
DRIVERS = [b"../../../bus/pci/drivers/vfio-pci", b"vfio-pci", b"../nvgrace_gpu_vfio_pci", b"../../drivers/nvidia",
           b"../vfio-pci/", b""]
GROUPS = [b"../../../kernel/iommu_groups/7", b"042", b"0", b"4294967296", b"4294967295", b"../g/", b"12", b"x/13"]
NUMAS = [b"", b"+", b"-0", b"+5", b" 7\n", b"0\n", b"-1\n", b"5\xa0", "5　".encode(), "  3".encode(),
         b"9223372036854775807", b"9223372036854775808", b"-9223372036854775808", b"-9223372036854775809", b"32768",
         b"-32768", b"32767", b"-32769", b"1_0", b"\xe3\x80", b"5\xe3\x80\x80\xe3"]
DEVICES = [b"0x1db6\n", b"0x20b0\n", b"0x2330\n", b"0xABCD\n", b"0x1db6", b"0x\n", b"0x12345\n", b"0xzz\n"]
SHORT = [b"", b"0"]


def gen_entries(rng, n, short=False, names="canonical", modes=None):
    """n random entries.  short: files of fewer than 2 bytes may appear (panics where they are reached).
    names: 'canonical' (ascending BDFs), 'mixed' (some non-canonical or out of order).
    modes: None (any), or (groups_numeric, devices_numeric) to keep those columns numeric where True."""
    out = []
    addrs = np.sort(rng.choice(1 << 20, size=n, replace=False)) if n else []
    for k in range(n):
        a = int(addrs[k])
        name = kvgpu.format_bdf(((a >> 8) << 16) | (a & 0xFF)).encode()
        if names == "mixed" and rng.random() < 0.05:
            name = rng.choice([b"0000:00:00.8", b"ABCD:00:00.0", b"devices", b"0000:00:1f.0", name + b" "])
        e = {}
        for key, pool in (("vendor", VENDORS), ("driver", DRIVERS), ("iommu_group", GROUPS), ("numa_node", NUMAS),
                          ("device", DEVICES)):
            if key in ("vendor", "device") and short and rng.random() < 0.02:
                e[key] = SHORT[rng.integers(2)]
            elif rng.random() < 0.05:
                e[key] = None
            else:
                e[key] = pool[rng.integers(len(pool))] if rng.random() < 0.5 else pool[0]
        if modes is not None:
            if modes[0] and e["iommu_group"] is not None:
                e["iommu_group"] = b"../g/%d" % rng.integers(0, 64)
            if modes[1] and e["device"] is not None:
                e["device"] = DEVICES[rng.integers(3)]
        out.append((name, e))
    return out


def render_records(recs) -> kvgpu.PciRaw:
    """sysfs text for synthetic records (oracle gen_pci): every read made; a flag makes that read fail."""
    drv = {L.DRV_VFIO_PCI: b"../vfio-pci", L.DRV_NVGRACE: b"../nvgrace_gpu_vfio_pci", L.DRV_OTHER: b"../nvidia",
           L.DRV_NONE: b"../none"}
    entries = []
    for r in recs:
        fl = int(r["flags"])
        e = {"vendor": None if fl & L.PF_VENDOR_ERR else b"0x%04x\n" % int(r["vendor"]),
             "driver": None if fl & L.PF_DRIVER_ERR else drv.get(int(r["driver"]), b"../other"),
             "iommu_group": None if fl & L.PF_IOMMU_ERR else b"../%d" % int(r["iommu_group"]),
             "numa_node": None if fl & L.PF_NUMA_ERR else b"%d\n" % int(r["numa"]),
             "device": None if fl & L.PF_DEVICE_ERR else b"0x%04x\n" % int(r["device"])}
        entries.append((kvgpu.format_bdf(int(r["addr"])).encode(), e))
    return raw_of(entries)
