"""kvg_snap.cuh (the raw-read decode of kvg_scan_pci_raw) executed on the CPU from its real source under the warp
emulator of tools/emu/, in the library's launch order, against the Go-exact restatement of tests/raw_scan_cases.py and
against snapshot_pci_tree on sysfs trees, from 0 to 5,000 entries."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import raw_scan_cases as RC
import util
import kvgpu
from kvgpu import _lib as L

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("snap"))
    lib.emu_scan_pci_raw.argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 3
    return lib


def run(emu, raw):
    """-> the snapshot tuple of RC.go_snapshot, or raises RC.RawError"""
    n = len(raw.state)
    off = np.ascontiguousarray(raw.off, dtype=np.uint32)
    state = np.ascontiguousarray(raw.state, dtype=np.uint16)
    blob = np.frombuffer(raw.bytes + b"\0", dtype=np.uint8)
    recs = np.zeros(max(n, 1), dtype=L.PCI_REC)
    tab = np.zeros((2, max(n, 1), 2), dtype=np.uint32)
    hdr = np.zeros(5, dtype=np.uint64)
    emu.emu_scan_pci_raw(off.ctypes.data, state.ctypes.data, blob.ctypes.data, n, recs.ctypes.data, tab.ctypes.data,
                         hdr.ctypes.data)
    for kind, w in (("miss", hdr[0]), ("panic", hdr[1]), ("range", hdr[2])):
        if int(w) != (1 << 64) - 1:
            raise RC.RawError(kind, int(w) >> 8, int(w) & 0xFF)
    words = hdr[3:].view(np.uint32)
    broken = int(words[0])

    def names(c):
        return [raw.bytes[int(a):int(b)].decode("latin-1") for a, b in tab[c, :int(words[1 + c])]]

    return (recs[:n], not broken & 1, names(0) if broken & 2 else None, names(1) if broken & 4 else None)


def check(emu, raw):
    try:
        want = RC.go_snapshot(raw)
    except RC.RawError as e:
        with pytest.raises(RC.RawError) as got:
            run(emu, raw)
        assert (got.value.kind, got.value.entry, got.value.field) == (e.kind, e.entry, e.field)
        return None
    got = run(emu, raw)
    assert got[1:] == want[1:]
    assert got[0].tobytes() == want[0].tobytes()
    return got


@pytest.mark.parametrize("n", [0, 1, 2, 31, 255, 256, 257, 1023, 1024, 1025, 5000])
@pytest.mark.parametrize("names", ["canonical", "mixed"])
def test_random_matrix(emu, n, names):
    rng = np.random.default_rng(n * 7 + len(names))
    check(emu, RC.raw_of(RC.gen_entries(rng, n, names=names)))


@pytest.mark.parametrize("modes", [(True, True), (True, False), (False, True), (False, False)])
def test_mixed_modes(emu, modes):
    rng = np.random.default_rng(11)
    raw = RC.raw_of(RC.gen_entries(rng, 3000, modes=modes))
    got = check(emu, raw)
    if got is not None and modes == (True, True):
        assert got[2] is None and got[3] is None


@pytest.mark.parametrize("seed", range(6))
def test_panics_lowest_entry_wins(emu, seed):
    rng = np.random.default_rng(100 + seed)
    check(emu, RC.raw_of(RC.gen_entries(rng, 2000, short=True)))


NV = {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "iommu_group": b"../7", "numa_node": b"0\n",
      "device": b"0x1db6\n"}


def one(**kw):
    e = dict(NV)
    e.update(kw)
    return e


@pytest.mark.parametrize("entry", [
    one(vendor=b"0x10DE\n"), one(vendor=b"0x10de\n\n"), one(vendor=b"10de"), one(vendor=b"\n\n10de"),
    one(vendor=b"0"), one(vendor=b""), one(vendor=b"0", device=b"0"),
    dict(vendor=b"0x8086\n", device=b"0"), dict(vendor=b"0x8086\n", device=b""),
    one(device=b"0"), one(device=b""), one(device=b"0x"), one(device=b"0x1DB6\n"),
    one(driver=b"vfio-pci"), one(driver=b"../vfio-pci/"), one(driver=b"nvgrace_gpu_vfio_pci"),
    one(iommu_group=b"7"), one(iommu_group=b"../g/"), one(iommu_group=b"042"), one(iommu_group=b"0"),
    one(iommu_group=b"4294967296"), one(iommu_group=b"4294967295"),
    one(numa_node=None), one(device=None), one(iommu_group=None), one(driver=None), one(vendor=None),
    one(driver=b"../nvidia", iommu_group=RC.MISSING, numa_node=RC.MISSING, device=RC.MISSING),
    one(vendor=b"0x8086\n", driver=RC.MISSING, iommu_group=RC.MISSING, numa_node=RC.MISSING, device=RC.MISSING),
    one(vendor=RC.MISSING), one(device=RC.MISSING), one(numa_node=RC.MISSING),
] + [one(numa_node=v) for v in RC.NUMAS])
def test_edges(emu, entry):
    lead = [(b"0000:00:01.0", one())]
    check(emu, RC.raw_of(lead + [(b"0000:00:02.0", entry)] + [(b"0000:00:03.0", one(iommu_group=b"../9"))]))


@pytest.mark.parametrize("names", [[b"0000:00:02.0", b"0000:00:01.0"], [b"0000:00:01.0", b"0000:00:01.0"],
                                   [b"0000:00:01.0", b"0000:00:20.0"], [b"0000:00:01.0", b"0000:00:00.8"],
                                   [b"a", b"b"], [b"0000:00:01.0", b"0000:0:01.0"]])
def test_names(emu, names):
    got = check(emu, RC.raw_of([(nm, one()) for nm in names]))
    assert got is not None and not got[1]


def test_device_handles_at_the_cap(emu):
    # 65,536 distinct device strings fit in index mode; the 65,537th is the range error of its first entry
    entries = [(b"%04x:00:00.0" % k, one(device=b"0xd%x\n" % k)) for k in range(65537)]
    check(emu, RC.raw_of(entries[:65536]))
    check(emu, RC.raw_of(entries))


def test_trees_equal_snapshot_pci_tree(emu, tmp_path):
    """records and tables byte for byte equal to snapshot_pci_tree's on the suite's trees, modes included"""
    trees = [util.c1_tree_entries(), util.ginkgo()["create_iommu_device_map"]["entries"],
             {"0000:00:01.0": dict(vendor="10de", device="1db6", driver="vfio-pci", iommu_group="g1", numa_node="0"),
              "0000:00:02.0": dict(vendor="10de", device="1db6", driver="vfio-pci", numa_node="1"),
              "0000:00:03.0": dict(vendor="10de", device="1db6", driver="vfio-pci", iommu_group="g2",
                                   numa_node="1"),
              "0000:00:04.0": dict(vendor="10de", device="abcd", driver="vfio-pci", iommu_group="g1"),
              "xyz": dict(vendor="10de", device="0x1db6x", driver="vfio-pci", iommu_group="7", numa_node="2")}]
    for k, ent in enumerate(trees):
        base = util.make_pci_tree(str(tmp_path / str(k)), ent)
        want = kvgpu.snapshot_pci_tree(base)
        got = run(emu, kvgpu.read_pci_tree_raw(base))
        assert got[0].tobytes() == want.recs.tobytes()
        assert (got[1], got[2], got[3]) == (want.packed_addr, want.group_names, want.device_names)
