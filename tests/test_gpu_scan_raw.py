"""kvg_scan_pci_raw on the H100: the decoded snapshot against the Go-exact restatement (tests/raw_scan_cases.py) and
snapshot_pci_tree, the result against kvg_scan_pci on the decoded records, the canonical dump against the oracle,
refusals, launch counts and isolation from the delta, health and allocation states."""
import numpy as np
import pytest

import raw_scan_cases as RC
import util
import kvgpu
from kvgpu import _lib as L
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = kvgpu.Context(0)
    c.pciids_load(util.pciids_text())
    yield c
    c.close()


def same_result(a, b):
    for f in ("n_records", "name_pool"):
        assert getattr(a, f) == getattr(b, f), f
    for f in ("survivors", "dev_keys", "dev_off", "dev_perm", "dev_name_slot", "grp_keys", "grp_off", "grp_perm"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def check(ctx, raw):
    try:
        want = RC.go_snapshot(raw)
    except RC.RawError as e:
        exc = kvgpu.ReferencePanic if e.kind == "panic" else L.KvgError
        with pytest.raises(exc) as got:
            ctx.scan_pci_raw(raw)
        if e.kind != "panic":
            assert got.value.rc == (L.KVG_EINVAL if e.kind == "miss" else L.KVG_ERANGE)
        assert ("entry %d " % e.entry) in str(got.value)
        return None
    res, snap = ctx.scan_pci_raw(raw)
    assert snap.recs.tobytes() == want[0].tobytes()
    assert (snap.packed_addr, snap.group_names, snap.device_names) == want[1:]
    assert snap.names == list(raw.names)
    same_result(res, ctx.scan_pci(snap.recs))
    return res, snap


@pytest.mark.parametrize("n", [0, 1, 257, 1025, 5000, 70000])
@pytest.mark.parametrize("names", ["canonical", "mixed"])
def test_random_matrix(ctx, n, names):
    check(ctx, RC.raw_of(RC.gen_entries(np.random.default_rng(n + len(names)), n, names=names)))


@pytest.mark.parametrize("modes", [(True, True), (True, False), (False, True)])
def test_mixed_modes(ctx, modes):
    check(ctx, RC.raw_of(RC.gen_entries(np.random.default_rng(5), 20000, modes=modes)))


@pytest.mark.parametrize("seed", range(4))
def test_panic_precedence(ctx, seed):
    # short files where they are reached: the lowest entry wins, and any panic beats a numa_node range error
    check(ctx, RC.raw_of(RC.gen_entries(np.random.default_rng(200 + seed), 4000, short=True)))


def test_panic_beats_range(ctx):
    nv = {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "iommu_group": b"../7", "device": b"0x1db6\n"}
    raw = RC.raw_of([(b"0000:00:01.0", dict(nv, numa_node=b"40000")), (b"0000:00:02.0", dict(nv, device=b"0"))])
    with pytest.raises(kvgpu.ReferencePanic, match="entry 1 .*device"):
        ctx.scan_pci_raw(raw)


@pytest.mark.parametrize("k", [65536, 65537])
def test_device_index_cap(ctx, k):
    nv = {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "iommu_group": b"../7", "numa_node": b"0"}
    check(ctx, RC.raw_of([(b"0000:%02x:%02x.%x" % (j >> 8, (j >> 3) & 31, j & 7), dict(nv, device=b"0xd%x\n" % j))
                          for j in range(k)]))


def test_trees(ctx, tmp_path):
    trees = [util.c1_tree_entries(), util.ginkgo()["create_iommu_device_map"]["entries"],
             {"0000:00:01.0": dict(vendor="10de", device="1db6", driver="vfio-pci", iommu_group="g1", numa_node="0"),
              "0000:00:02.0": dict(vendor="10de", device="1db6", driver="vfio-pci", numa_node="1"),
              "0000:00:04.0": dict(vendor="10de", device="abcd", driver="vfio-pci", iommu_group="g1"),
              "xyz": dict(vendor="10de", device="0x1db6x", driver="vfio-pci", iommu_group="7", numa_node="2")}]
    text = util.pciids_text()
    for k, ent in enumerate(trees):
        base = util.make_pci_tree(str(tmp_path / str(k)), ent)
        want = kvgpu.snapshot_pci_tree(base)
        res, snap = ctx.scan_pci_raw(kvgpu.read_pci_tree_raw(base))
        assert snap.recs.tobytes() == want.recs.tobytes()
        assert (snap.packed_addr, snap.group_names, snap.device_names) == (
            want.packed_addr, want.group_names, want.device_names)
        same_result(res, ctx.scan_pci(want.recs))
        om = O.Maps()
        om.create_iommu_device_map_tree(base)
        got = kvgpu.canonical_dump(kvgpu.pci_maps_from_result(res, snap, name_of=ctx.name_lookup))
        assert got == om.dump(text)


def test_million_numeric(ctx):
    recs = O.gen_pci(0, 1_000_000, O.nv_ids(util.pciids_text()), 16)
    res, snap = ctx.scan_pci_raw(RC.render_records(recs))
    assert snap.packed_addr and snap.group_names is None and snap.device_names is None
    same_result(res, ctx.scan_pci(recs))


def test_refusals(ctx):
    lib, h = ctx._lib, ctx.handle
    raw = RC.raw_of([(b"0000:00:01.0", {"vendor": b"0x8086\n"})])
    res, snap = C_ptrs()
    base = ctx.launch_count
    assert lib.kvg_scan_pci_raw(None, None, None, None) == L.KVG_EINVAL
    assert lib.kvg_scan_pci_raw(h, None, res, snap) == L.KVG_EINVAL
    arg = raw_arg(raw)
    assert lib.kvg_scan_pci_raw(h, arg[0], None, snap) == L.KVG_EINVAL
    assert lib.kvg_scan_pci_raw(h, arg[0], res, None) == L.KVG_EINVAL
    bad = raw.off.copy()
    bad[2] = 0  # decreasing
    assert lib.kvg_scan_pci_raw(h, raw_arg(kvgpu.PciRaw(raw.names, bad, raw.bytes, raw.state))[0], res,
                                snap) == L.KVG_EINVAL
    bad = raw.off.copy() + 1
    assert lib.kvg_scan_pci_raw(h, raw_arg(kvgpu.PciRaw(raw.names, bad, raw.bytes, raw.state))[0], res,
                                snap) == L.KVG_EINVAL
    import ctypes as C
    nul = L.PciRawC(1, None, None, None)
    assert lib.kvg_scan_pci_raw(h, C.byref(nul), res, snap) == L.KVG_EINVAL
    assert ctx.launch_count == base and not res._obj and not snap._obj
    # before a pci.ids load
    fresh = kvgpu.Context(0)
    try:
        with pytest.raises(L.KvgError) as e:
            fresh.scan_pci_raw(raw)
        assert e.value.rc == L.KVG_ESTATE and fresh.launch_count == 0
    finally:
        fresh.close()


def C_ptrs():
    import ctypes as C
    return C.byref(C.POINTER(L.PciResultC)()), C.byref(C.POINTER(L.PciSnapC)())


def raw_arg(raw):
    import ctypes as C
    off = np.ascontiguousarray(raw.off, dtype=np.uint32)
    state = np.ascontiguousarray(raw.state, dtype=np.uint16)
    blob = np.frombuffer(raw.bytes + b"\0", dtype=np.uint8)
    a = L.PciRawC(len(state), off.ctypes.data, blob.ctypes.data, state.ctypes.data)
    return C.byref(a), (a, off, state, blob)


def test_launch_counts(ctx):
    """decode + the scan's launches when every column is numeric; + probe and compaction per interned column and one
    pack otherwise; none for n = 0"""
    nv = {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "iommu_group": b"../7", "numa_node": b"0",
          "device": b"0x1db6\n"}
    numeric = RC.raw_of([(b"0000:00:%02x.0" % k, nv) for k in range(1, 20)])
    snap_recs = ctx.scan_pci_raw(numeric)[1].recs
    ctx.scan_pci(snap_recs)
    b0 = ctx.launch_count
    ctx.scan_pci(snap_recs)
    scan = ctx.launch_count - b0
    b0 = ctx.launch_count
    ctx.scan_pci_raw(numeric)
    assert ctx.launch_count - b0 == 1 + scan
    both = RC.raw_of([(b"x%02d" % k, dict(nv, iommu_group=b"g%d" % (k % 3), device=b"0xD%d\n" % (k % 2)))
                      for k in range(1, 20)])
    ctx.scan_pci_raw(both)
    b0 = ctx.launch_count
    ctx.scan_pci_raw(both)
    assert ctx.launch_count - b0 == 1 + 2 * 2 + 1 + scan
    addr_only = RC.raw_of([(b"x%02d" % k, nv) for k in range(1, 20)])
    b0 = ctx.launch_count
    ctx.scan_pci_raw(addr_only)
    assert ctx.launch_count - b0 == 1 + 1 + scan
    b0 = ctx.launch_count
    res, snap = ctx.scan_pci_raw(RC.raw_of([]))
    assert ctx.launch_count == b0 and len(res.survivors) == 0 and len(snap.recs) == 0


def test_isolation(ctx):
    """delta, health and allocation state are untouched: the next delta / health call sees only its own history"""
    recs = O.gen_pci(0, 5000, O.nv_ids(util.pciids_text()), 8)
    ctx.scan_pci_delta_reset()
    ctx.health_reset()
    r1, d1 = ctx.scan_pci_delta(recs)
    h1 = ctx.health_rescan(recs)
    nv = {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "numa_node": b"1"}
    check(ctx, RC.raw_of([(b"x%05d" % k, dict(nv, iommu_group=b"g%d" % (k % 7), device=b"0xD%d\n" % (k % 5)))
                          for k in range(3000)]))
    r2, d2 = ctx.scan_pci_delta(recs)
    h2 = ctx.health_rescan(recs)
    assert len(d2.changes) == 0 and d2.n_prev == len(r1.survivors)
    assert len(h2.changed) == 0 and h2.n_alive == h1.n_alive
