"""kvg_snap.cuh's mdev decode (kvg_scan_mdev_raw) executed on the CPU from its real source under the warp emulator of
tools/emu/, in the library's launch order, against the Go-exact restatement of tests/mdev_raw_cases.py (records, modes,
raw type dictionary, parent strings and the verdict words) from 0 to 5,000 entries, and against snapshot_mdev_tree on
sysfs trees without an empty parent."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import mdev_raw_cases as MC
import util
import kvgpu
from kvgpu import _lib as L

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("snap"))
    lib.emu_scan_mdev_raw.argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 3
    return lib


def run(emu, raw):
    """-> the snapshot tuple of MC.go_mdev_snapshot, or raises MC.RawError"""
    n = len(raw.state)
    off = np.ascontiguousarray(raw.off, dtype=np.uint32)
    state = np.ascontiguousarray(raw.state, dtype=np.uint16)
    blob = np.frombuffer(raw.bytes + b"\0", dtype=np.uint8)
    recs = np.zeros(max(n, 1), dtype=L.MDEV_REC)
    tab = np.zeros((2, max(n, 1), 2), dtype=np.uint32)
    hdr = np.zeros(5, dtype=np.uint64)
    emu.emu_scan_mdev_raw(off.ctypes.data, state.ctypes.data, blob.ctypes.data, n, recs.ctypes.data, tab.ctypes.data,
                          hdr.ctypes.data)
    for kind, w in (("miss", hdr[0]), ("panic", hdr[1]), ("range", hdr[2])):
        if int(w) != (1 << 64) - 1:
            raise MC.RawError(kind, int(w) >> 8, int(w) & 0xFF)
    words = hdr[3:].view(np.uint32)
    broken = int(words[0])
    strings = lambda c: [raw.bytes[int(a):int(b)] for a, b in tab[c, :int(words[1 + c])]]
    return (recs[:n], not broken & 1, not broken & 2, strings(0) if n else [],
            [p.decode("latin-1") for p in strings(1)] if broken & 2 else None)


def check(emu, raw):
    try:
        want = MC.go_mdev_snapshot(raw)
    except MC.RawError as e:
        with pytest.raises(MC.RawError) as got:
            run(emu, raw)
        assert (got.value.kind, got.value.entry, got.value.field) == (e.kind, e.entry, e.field)
        return None
    got = run(emu, raw)
    assert got[1:] == want[1:]
    assert got[0].tobytes() == want[0].tobytes()
    return got


@pytest.mark.parametrize("n", [0, 1, 2, 31, 255, 256, 257, 1023, 1024, 1025, 5000])
@pytest.mark.parametrize("names,parents", [("canonical", "packed"), ("mixed", "mixed"), ("canonical", "mixed"),
                                           ("mixed", "packed")])
def test_random_matrix(emu, n, names, parents):
    rng = np.random.default_rng(n * 7 + len(names) + 3 * len(parents))
    got = check(emu, MC.raw_of(MC.gen_entries(rng, n, names=names, parents=parents)))
    if got is not None and n > 300:
        assert got[1] == (names == "canonical") and got[2] == (parents == "packed")


@pytest.mark.parametrize("seed", range(6))
def test_panics_lowest_entry_wins(emu, seed):
    rng = np.random.default_rng(100 + seed)
    check(emu, MC.raw_of(MC.gen_entries(rng, 2000, panic=True, parents="mixed")))


U = [MC.uuid_name(bytes([k]) * 16) for k in range(1, 4)]


def one(u, **kw):
    e = {"type": b"GRID P40-1Q\n", "link": MC.link_to(MC.PARENT, u), "numa_node": b"0\n"}
    e.update(kw)
    return e


@pytest.mark.parametrize("entry", [
    *[dict(type=t) for t in MC.TYPES],
    *[dict(link=f(U[1])) for f in MC.LINKS],
    *[dict(numa_node=v) for v in MC.NUMAS],
    dict(type=None), dict(link=None), dict(numa_node=None),
    dict(type=MC.MISSING), dict(link=MC.MISSING), dict(numa_node=MC.MISSING),
    dict(type=None, link=MC.MISSING, numa_node=MC.MISSING), dict(link=None, numa_node=MC.MISSING),
    dict(link=b"nolash", numa_node=MC.MISSING), dict(link=b"nolash", numa_node=b"99999"),
    dict(link=b"a/\n/u", numa_node=MC.MISSING), dict(numa_node=b"32768"),
])
def test_edges(emu, entry):
    check(emu, MC.raw_of([(U[0], one(U[0])), (U[1], one(U[1], **entry)), (U[2], one(U[2], type=b"GRID P40-2Q\n"))]))


@pytest.mark.parametrize("names", [[U[1], U[0]], [U[0], U[0]], [MC.uuid_name(b"\x0a" * 16).upper(), U[1]],
                                   [b"1", b"2"], [U[0], U[1][:-1]], [U[0], U[1] + b"\n"]])
def test_names(emu, names):
    got = check(emu, MC.raw_of([(nm, one(nm)) for nm in names]))
    assert got is not None and not got[1]


def test_type_cap(emu):
    # 65,535 distinct type strings fit the dictionary; the 65,536th is the range error of its entry
    names = MC.canonical_names(np.random.default_rng(1), 65536)
    entries = [(u, one(u, type=b"T%d" % k)) for k, u in enumerate(names)]
    got = check(emu, MC.raw_of(entries[:65535]))
    assert len(got[3]) == 65535
    check(emu, MC.raw_of(entries))


def _tree(tmp, k, parents, mdevs):
    return util.make_mdev_tree(str(tmp / str(k)), parents, mdevs)


def trees():
    u = [MC.uuid_name(bytes([k]) * 16).decode() for k in range(1, 9)]
    g = util.ginkgo()
    out = [({"0000:01:00.0": "0\n", "0000:02:00.0": "1\n"},
            {u[0]: dict(type="GRID P40-1Q\n", parent="0000:01:00.0"), u[1]: dict(type="GRID P40-2Q", parent="0000:01:00.0"),
             u[2]: dict(type="GRID  P40-1Q\n", parent="0000:02:00.0"), u[3]: dict(parent="0000:02:00.0"),
             u[4]: dict(type="GRID P40-1Q\n")})]
    spec = g["create_vgpu_id_map"]
    out.append(({spec["parent_dir"]: spec["parent_numa_content"]}, spec["entries"]))
    out.append(({"0000:01:00.0": "0\n", "gpu-a": "1\n", "gpu-b": None},
                {"1": dict(type="A\n", parent="gpu-a"), "2": dict(type="B\n", parent="0000:01:00.0"),
                 u[5]: dict(type="A \n", parent="gpu-b"), "0": dict(type="", parent="gpu-a")}))
    return out


def test_trees_equal_snapshot_mdev_tree(emu, tmp_path):
    """records, dictionary and modes byte for byte equal to snapshot_mdev_tree's on trees without an empty parent"""
    for k, (parents, mdevs) in enumerate(trees()):
        vbase, pbase = _tree(tmp_path, k, parents, mdevs)
        want = kvgpu.snapshot_mdev_tree(vbase, pbase)
        got = run(emu, kvgpu.read_mdev_tree_raw(vbase, pbase))
        assert got[0].tobytes() == want.recs.tobytes()
        assert (got[1], got[3], got[4]) == (want.uuid_ok, want.raw_types, want.parent_names)
