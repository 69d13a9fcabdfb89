"""Raw walk reads for kvg_scan_mdev_raw and a Go-exact restatement of what createVgpuIDMap's readers make of them
(device_plugin.go:269-284, readGpuIDForVgpuFunc :347-357, readNUMANodeFunc :304-320): the parent is
strings.Split(target, "/")[len-2] with Trim "\\n", numa_node goes through the oracle's strings.TrimSpace (kvo_trim_space)
and a plain strconv.ParseInt(s, 10, 64).  snapshot_mdev_tree gives an empty parent the packed key 0 and reads numa_node
with its own trimming; this file is the reference for both."""
import os

import numpy as np

import kvgpu
import util
from kvgpu import _lib as L
from oracle import oracle as O
from raw_scan_cases import MISSING, NUMAS, RawError, parse_int64  # noqa: F401  (re-exported for the tests)

FIELDS = ("type", "link", "numa_node")
MAX_TYPES = 65535   # load_type_dict


def raw_of(entries) -> kvgpu.MdevRaw:
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
    return kvgpu.MdevRaw(names, off, b"".join(x for row in parts for x in row), np.array(state, dtype=np.uint16))


def uuid_bytes(name: bytes):
    """the 16 bytes of a canonical lower-case 8-4-4-4-12 UUID, else None"""
    if len(name) != 36 or any(name[k] != 0x2D for k in (8, 13, 18, 23)):
        return None
    h = name.replace(b"-", b"")
    if len(h) != 32 or any(c not in b"0123456789abcdef" for c in h):
        return None
    return bytes.fromhex(h.decode())


def go_mdev_snapshot(raw: kvgpu.MdevRaw):
    """-> (recs, uuid_ok, parents_packed, raw_types, parent_names | None); raises RawError('miss' | 'panic' | 'range')
    with the lowest entry and its field."""
    n = len(raw.state)
    F = L.MRAW_FIELDS
    get = lambda i, f: raw.bytes[int(raw.off[i * F + f]):int(raw.off[i * F + f + 1])]
    rows, miss, panic, rng = [], [], [], []
    for i in range(n):
        st = int(raw.state[i])

        def reach(f):
            if not (st >> f) & 1:
                miss.append((i, f))
                return None
            return None if (st >> (8 + f)) & 1 else get(i, f)

        flags, tbytes, parent, numa = 0, None, None, 0
        t = reach(L.MRAW_TYPE)
        if t is None:
            flags |= L.MF_TYPE_ERR if (st >> L.MRAW_TYPE) & 1 else 0
        else:
            tbytes = t
            link = reach(L.MRAW_LINK)
            if link is None:
                flags |= L.MF_PARENT_ERR if (st >> L.MRAW_LINK) & 1 else 0
            else:
                parts = link.split(b"/")
                if len(parts) < 2:
                    panic.append((i, L.MRAW_LINK))
                else:
                    parent = parts[-2].strip(b"\n")
                    m = reach(L.MRAW_NUMA)
                    if m is None:
                        flags |= L.MF_NUMA_ERR if (st >> L.MRAW_NUMA) & 1 else 0
                    else:
                        val = parse_int64(O.trim_space(m))
                        if val is None:
                            flags |= L.MF_NUMA_ERR
                        else:
                            numa = val
                            if not -32768 <= val <= 32767:
                                rng.append((i, L.MRAW_NUMA))
        rows.append((tbytes, parent, flags, numa))
    if miss:
        raise RawError("miss", *miss[0])
    if panic:
        raise RawError("panic", *panic[0])
    names = [get(i, L.MRAW_NAME) for i in range(n)]
    ub = [uuid_bytes(x) for x in names]
    uuid_ok = all(u is not None for u in ub) and all(ub[k] < ub[k + 1] for k in range(n - 1))
    parents_packed = all(kvgpu.parse_bdf(r[1].decode("latin-1")) is not None for r in rows if r[1] is not None)
    types, pidx = {}, {}
    recs = np.zeros(n, dtype=L.MDEV_REC)
    for i, (tbytes, parent, flags, numa) in enumerate(rows):
        t = 0
        if tbytes is not None:
            t = types.setdefault(tbytes, len(types))
            if t >= MAX_TYPES:
                rng.append((i, L.MRAW_TYPE))
        if parent is None:
            p = 0
        elif parents_packed:
            p = kvgpu.parse_bdf(parent.decode("latin-1"))
        else:
            p = pidx.setdefault(parent, len(pidx))
        if uuid_ok:
            recs[i]["uuid"] = np.frombuffer(ub[i], dtype=np.uint8)
        else:
            recs[i]["uuid"][:4] = np.frombuffer(int(i).to_bytes(4, "big"), dtype=np.uint8)
        recs[i]["parent"], recs[i]["type_idx"], recs[i]["flags"] = p, t & 0xFFFF, flags
        recs[i]["parent_numa"] = numa if -32768 <= numa <= 32767 else 0
    if rng:
        raise RawError("range", *min(rng))
    return (recs, uuid_ok, parents_packed, list(types),
            None if parents_packed else [x.decode("latin-1") for x in pidx])


# ---- the edge matrix ---------------------------------------------------------------------------------------------
TYPES = [b"GRID P40-1Q\n", b"GRID  P40-1Q\n", b"GRID\tP40-1Q", b" GRID P40-1Q \n", b"GRID P40-1Q\n\n", b"", b"\n",
         "GRID P40-Ä1Q\n".encode(), b"\xff\xfeQ", b"NVIDIA A100-4C\r\n"]
PARENT = b"0000:01:00.0"


def link_to(parent: bytes, name: bytes) -> bytes:
    return b"../../devices/pci0000:00/" + parent + b"/" + name


# link targets as a function of the entry name (u); "nolash" panics
LINKS = [lambda u: link_to(PARENT, u), lambda u: b"nolash", lambda u: b"/x", lambda u: b"a//" + u,
         lambda u: b"a/0000:01:00.0\n/" + u, lambda u: b"a/\n/" + u, lambda u: b"0000:02:00.0/" + u,
         lambda u: b"x/0000:01:00.08/" + u, lambda u: b"x/0000:0A:00.0/" + u, lambda u: b"/" + u]
PANIC_LINKS = (1,)
NAMES = {"upper": lambda k: b"%08X-0000-0000-0000-%012X" % (k, k), "ginkgo": lambda k: b"%d" % (k + 1),
         "short": lambda k: b"%08x-0000-0000-0000-%011x" % (k, k)}


def uuid_name(rng_bytes) -> bytes:
    return kvgpu.format_uuid(rng_bytes).encode()


def canonical_names(rng, n):
    hi = np.sort(rng.choice(1 << 40, size=n, replace=False)) if n else []
    return [uuid_name(int(h).to_bytes(5, "big") + rng.bytes(11)) for h in hi]


def gen_entries(rng, n, panic=False, names="canonical", parents="packed"):
    """n random entries.  panic: link targets without '/' may appear.  names: 'canonical' (ascending UUIDs) or
    'mixed' (some upper-case, out of order or Ginkgo's plain numbers).  parents: 'packed' (every decoded parent a
    canonical BDF) or 'mixed' (the LINKS edges, empty and "\\n"-wrapped parents among them)."""
    out = []
    nm = canonical_names(rng, n)
    for k in range(n):
        name = nm[k]
        if names == "mixed" and rng.random() < 0.05:
            r = rng.integers(4)
            name = NAMES[("upper", "ginkgo", "short")[r]](k) if r < 3 else nm[max(k - 1, 0)]
        e = {}
        e["type"] = None if rng.random() < 0.05 else (
            TYPES[rng.integers(len(TYPES))] if rng.random() < 0.5 else b"GRID T4-%dQ\n" % rng.integers(8))
        if rng.random() < 0.05:
            e["link"] = None
        elif panic and rng.random() < 0.02:
            e["link"] = LINKS[PANIC_LINKS[0]](name)
        elif parents == "mixed" and rng.random() < 0.2:
            j = rng.integers(len(LINKS))
            e["link"] = LINKS[j](name) if j not in PANIC_LINKS else LINKS[0](name)
        else:
            e["link"] = link_to(kvgpu.format_bdf(int(rng.integers(64)) << 8).encode(), name)
        e["numa_node"] = None if rng.random() < 0.05 else (
            NUMAS[rng.integers(len(NUMAS))] if rng.random() < 0.3 else b"%d\n" % rng.integers(-1, 4))
        out.append((name, e))
    return out


def render_records(recs, type_names) -> kvgpu.MdevRaw:
    """sysfs text for synthetic records (oracle gen_mdev with its type names): every read made; a flag makes that read
    fail.  Names are the records' UUIDs, links name the parent's packed BDF."""
    entries = []
    for r in recs:
        fl = int(r["flags"])
        name = kvgpu.format_uuid(r["uuid"]).encode()
        e = {"type": None if fl & L.MF_TYPE_ERR else type_names[int(r["type_idx"])],
             "link": None if fl & L.MF_PARENT_ERR else link_to(kvgpu.format_bdf(int(r["parent"])).encode(), name),
             "numa_node": None if fl & L.MF_NUMA_ERR else b"%d\n" % int(r["parent_numa"])}
        entries.append((name, e))
    return raw_of(entries)


# ---- sysfs trees ---------------------------------------------------------------------------------------------
def _link_tree(root, entries):
    """<root>/mdev/<name> -> symlink with the given target text; the type file lives where the target resolves.
    entries: name -> (target relative to <root>/pci, type contents).  <root>/pci/<bdf>/numa_node for canonical parents."""
    mdev, pci = os.path.join(root, "mdev"), os.path.join(root, "pci")
    os.makedirs(mdev)
    os.makedirs(pci)
    for name, (target, typ) in entries.items():
        real = os.path.normpath(pci + "/" + target)
        os.makedirs(os.path.join(real, "mdev_type"), exist_ok=True)
        with open(os.path.join(real, "mdev_type", "name"), "w") as f:
            f.write(typ)
        parent = os.path.dirname(real)
        if parent != pci and not os.path.exists(os.path.join(parent, "numa_node")):
            with open(os.path.join(parent, "numa_node"), "w") as f:
                f.write("1\n")
        os.symlink(pci + "/" + target, os.path.join(mdev, name))
    return mdev, pci


def trees(tmp):
    """The sysfs trees the GPU tests compare with the oracle's tree walk -> [(name, vgpu base, pci base, plain)];
    plain: free of the empty-parent edges, so snapshot_mdev_tree agrees too.  Type contents and parent components stay
    under the 1,024-byte buffers of the oracle's walk."""
    u = [uuid_name(bytes([k]) * 16).decode() for k in range(1, 9)]
    spec = util.ginkgo()["create_vgpu_id_map"]
    out = [("ginkgo",) + util.make_mdev_tree(str(tmp / "g"), {spec["parent_dir"]: spec["parent_numa_content"]},
                                             spec["entries"]) + (True,)]
    out.append(("canonical",) + util.make_mdev_tree(
        str(tmp / "c"), {"0000:01:00.0": "0\n", "0000:02:00.0": "1\n", "0000:03:00.0": None},
        {u[0]: dict(type="GRID P40-1Q\n", parent="0000:01:00.0"),
         u[1]: dict(type="GRID P40-2Q", parent="0000:01:00.0"),
         u[2]: dict(type="GRID  P40-1Q\n", parent="0000:02:00.0"), u[3]: dict(parent="0000:02:00.0"),
         u[4]: dict(type="GRID P40-1Q\n"), u[5]: dict(type="GRID P40-1Q\n", parent="0000:03:00.0")}) + (True,))
    out.append(("empty-parent",) + _link_tree(str(tmp / "e"), {
        u[0]: ("0000:01:00.0/" + u[0], "GRID P40-1Q\n"), u[1]: ("/" + u[1], "GRID P40-1Q\n"),
        u[2]: ("0000:01:00.0/" + u[2], "GRID P40-2Q\n")}) + (False,))
    out.append(("newline-parent",) + _link_tree(str(tmp / "n"), {
        u[0]: ("\n/" + u[0], "GRID P40-1Q\n"), u[1]: ("0000:02:00.0/" + u[1], "GRID P40-1Q\n")}) + (False,))
    return out
