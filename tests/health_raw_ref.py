"""String-level reference of the health re-scans from raw reads (kvg_health_rescan_groups_raw /
kvg_health_rescan_mdev_raw): the readers' decode in the reference's short-circuit order (device_plugin.go:202-238,
:269-284) with the oracle's numa_node rule (strings.TrimSpace, then strconv.ParseInt), then the two state machines
over entry names, group strings, node names and bus-id strings.  Nothing is interned: every identity is bytes."""
from dataclasses import dataclass

from kvgpu import _lib as L
from oracle import oracle as O
from raw_scan_cases import RawError, parse_int64


@dataclass
class Delta:
    n_records: int
    n_alive: int
    changed: list


def _reader(raw, fields):
    def get(i, f):
        return raw.bytes[int(raw.off[i * fields + f]):int(raw.off[i * fields + f + 1])]
    return get


def _numa(m, i, field, rng):
    """a reached numa_node that parses but does not fit int16 is the range error (a parse error is only a flag)"""
    val = parse_int64(O.trim_space(m))
    if val is not None and not -32768 <= val <= 32767:
        rng.append((i, field))


def _verdicts(miss, panic, rng, names):
    if miss:
        raise RawError("miss", *miss[0])
    if panic:
        raise RawError("panic", *panic[0])
    if rng:
        raise RawError("range", *min(rng))
    for i in range(1, len(names)):
        if names[i - 1] >= names[i]:
            raise RawError("order", i, 0)


def pci_entries(raw):
    """-> [(name, alive, iommu_group basename or None)]; raises RawError('miss' | 'panic' | 'range' | 'order')."""
    n, get = len(raw.state), _reader(raw, L.RAW_FIELDS)
    out, miss, panic, rng = [], [], [], []
    for i in range(n):
        st = int(raw.state[i])

        def reach(f):
            if not (st >> f) & 1:
                miss.append((i, f))
                return None
            return None if (st >> (8 + f)) & 1 else get(i, f)

        alive, group = False, None
        v = reach(L.RAW_VENDOR)
        if v is not None and len(v) < 2:
            panic.append((i, L.RAW_VENDOR))
        elif v is not None and v[2:].strip(b"\n") == b"10de":
            d = reach(L.RAW_DRIVER)
            if d is not None and d.rsplit(b"/", 1)[-1] in (b"vfio-pci", b"nvgrace_gpu_vfio_pci"):
                g = reach(L.RAW_GROUP)
                if g is not None:
                    group = g.rsplit(b"/", 1)[-1]
                    m = reach(L.RAW_NUMA)
                    if m is not None:
                        _numa(m, i, L.RAW_NUMA, rng)
                    dv = reach(L.RAW_DEVICE)
                    if dv is not None and len(dv) < 2:
                        panic.append((i, L.RAW_DEVICE))
                    alive = dv is not None
        out.append((get(i, L.RAW_NAME), alive, group))
    _verdicts(miss, panic, rng, [e[0] for e in out])
    return out


def mdev_entries(raw):
    """-> [(name, present, decoded parent or None)]; raises RawError as pci_entries."""
    n, get = len(raw.state), _reader(raw, L.MRAW_FIELDS)
    out, miss, panic, rng = [], [], [], []
    for i in range(n):
        st = int(raw.state[i])

        def reach(f):
            if not (st >> f) & 1:
                miss.append((i, f))
                return None
            return None if (st >> (8 + f)) & 1 else get(i, f)

        present, parent = False, None
        if reach(L.MRAW_TYPE) is not None:
            link = reach(L.MRAW_LINK)
            if link is not None:
                present = True
                parts = link.split(b"/")
                if len(parts) < 2:
                    panic.append((i, L.MRAW_LINK))
                else:
                    parent = parts[-2].strip(b"\n")
                    m = reach(L.MRAW_NUMA)
                    if m is not None:
                        _numa(m, i, L.MRAW_NUMA, rng)
        out.append((get(i, L.MRAW_NAME), present, parent))
    _verdicts(miss, panic, rng, [e[0] for e in out])
    return out


class RawGroupsRef:
    """h' = alive && the group string is one of the node names; state kept per entry name."""

    def __init__(self):
        self.prev = {}

    def step(self, raw, nodes) -> Delta:
        ents = pci_entries(raw)
        nodes = set(bytes(x) for x in nodes)
        now, changed = {}, []
        for i, (name, alive, group) in enumerate(ents):
            h = int(alive and group is not None and group in nodes)
            if h != (self.prev.get(name, 0) & 1):
                changed.append((i << 1) | h)
            now[name] = h
        self.prev = now
        return Delta(len(ents), sum(now.values()), changed)


class RawMdevRef:
    """p' = present; m' = p' && (non-empty parent in the XID bus ids || (p && m)); healthy = p && !m; state (bit 0
    healthy, bit 1 marked) kept per entry name."""

    def __init__(self):
        self.prev = {}

    def step(self, raw, xids) -> Delta:
        ents = mdev_entries(raw)
        xids = set(bytes(x) for x in xids)
        now, changed, alive = {}, [], 0
        for i, (name, present, parent) in enumerate(ents):
            s = self.prev.get(name, 0)
            if not present:
                t = 0
            else:
                marked = bool(s & 2) or (bool(parent) and parent in xids)
                t = 2 if marked else 1
            if (t & 1) != (s & 1):
                changed.append((i << 1) | (t & 1))
            now[name] = t
            alive += t & 1
        self.prev = now
        return Delta(len(ents), alive, changed)
