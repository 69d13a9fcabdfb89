"""Re-scans from raw reads on sysfs trees (util.make_pci_tree), in numeric and index mode: after each hot-add, removal,
regroup and NUMA move, DiscoveryScan.rescan_iommu_device_map(raw=True) leaves the Maps equal to a fresh
create_iommu_device_map(raw=True) of the same tree, touching exactly the keys whose members changed, and a raw-driven
PciRescanFeed re-sends the device list only for plugins whose key is dirty.  The same for the vGPU half on
util.make_mdev_tree trees (create, destroy, retype, move, parent NUMA move): rescan_vgpu_id_map(raw=True) against
create_vgpu_id_map(raw=True), and a raw-driven MdevRescanFeed."""
import dataclasses
import os
import shutil

import pytest

import util
import kvgpu
from kvgpu import serve

pytestmark = pytest.mark.gpu


def entry(device, group, numa="0\n"):
    return dict(vendor="10de", device=device, driver="vfio-pci", iommu_group=group, numa_node=numa)


def trees(mode):
    """the tree before each step, then after it: hot-add, removal, regroup, NUMA move (and back to the start)"""
    t0 = {"0000:00:01.0": entry("1db6", "1"), "0000:00:02.0": entry("1db6", "2"), "0000:00:03.0": entry("20b0", "2"),
          "0000:00:04.0": entry("2330", "3")}
    if mode == "index":   # a group that is not a canonical decimal, an upper-case device id, a name that is no BDF
        t0["0000:00:02.0"] = entry("1db6", "g2")
        t0["0000:00:04.0"] = entry("0x2330x", "3")
        t0["zz-extra"] = entry("20b0", "9")
    t1 = dict(t0, **{"0000:00:00.1": entry("1db6", "7")})                 # hot-add at the front
    t2 = {k: v for k, v in t1.items() if k != "0000:00:03.0"}             # removal
    t3 = dict(t2, **{"0000:00:01.0": entry("1db6", "2")})                 # regroup
    t4 = dict(t3, **{"0000:00:02.0": dict(t3["0000:00:02.0"], numa_node="1\n")})   # NUMA move
    return [t0, t1, t2, t3, t4, t0]


def write_tree(root, ent):
    for sub in ("devices", "real", "targets"):
        shutil.rmtree(os.path.join(root, sub), ignore_errors=True)
    return util.make_pci_tree(root, ent)


def fresh_maps(ids, base):
    ds = kvgpu.DiscoveryScan(pci_ids_path=ids, base_path=base)
    try:
        return ds.create_iommu_device_map(raw=True)
    finally:
        ds.close()


def changed_keys(before: dict, after: dict):
    return ({k for k, v in after.items() if before.get(k) != v}, {k for k in before if k not in after})


@pytest.mark.parametrize("mode", ["numeric", "index"])
def test_rescan_raw_patches_exactly(tmp_path, mode):
    root = str(tmp_path)
    ids = os.path.join(root, "pci.ids")
    with open(ids, "wb") as f:
        f.write(util.pciids_text())
    steps = trees(mode)
    base = write_tree(root, steps[0])
    ds = kvgpu.DiscoveryScan(pci_ids_path=ids, base_path=base)
    try:
        ds.rescan_iommu_device_map(raw=True)
        assert dataclasses.asdict(ds.maps) == dataclasses.asdict(fresh_maps(ids, base))
        for ent in steps[1:]:
            before = dataclasses.asdict(ds.maps)
            write_tree(root, ent)
            touched = ds.rescan_iommu_device_map(raw=True)
            after = dataclasses.asdict(ds.maps)
            assert after == dataclasses.asdict(fresh_maps(ids, base))
            dirty, gone = changed_keys(before["deviceMap"], after["deviceMap"])
            assert set(touched.dev_dirty) == dirty and set(touched.dev_gone) == gone
            dirty, gone = changed_keys(before["iommuMap"], after["iommuMap"])
            assert set(touched.grp_dirty) == dirty and set(touched.grp_gone) == gone
    finally:
        ds.close()


class Stub:
    """a plugin that counts the device lists it is sent"""

    def __init__(self, spec):
        self.key, self.sent, self.running = spec.key, 0, False

    def start(self):
        self.running = True

    def stop(self):
        self.running = False

    def set_devices(self, devs):
        self.sent += 1


@pytest.mark.parametrize("mode", ["numeric", "index"])
def test_raw_feed_resends_only_dirty_keys(tmp_path, mode):
    root = str(tmp_path)
    steps = trees(mode)
    base = write_tree(root, steps[0])
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(util.pciids_text())
        plugins = {}
        feed = serve.PciRescanFeed(ctx.scan_pci_raw_delta, lambda: kvgpu.read_pci_tree_raw(base), kvgpu.Maps(),
                                   plugins, Stub, raw=True, name_of=ctx.name_lookup)
        feed.tick()
        assert set(plugins) == set(feed.maps.deviceMap)
        for ent in steps[1:]:
            before = {k: list(v) for k, v in feed.maps.deviceMap.items()}
            sent = {k: p.sent for k, p in plugins.items()}
            write_tree(root, ent)
            touched = feed.tick()
            dirty, gone = changed_keys(before, feed.maps.deviceMap)
            assert set(touched.dev_dirty) == dirty and set(touched.dev_gone) == gone
            for k, p in plugins.items():
                resent = p.sent - sent.get(k, 0)
                assert resent == (1 if k in dirty and k in sent else 0), (k, resent)
            assert set(plugins) == set(feed.maps.deviceMap)


U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(1, 8)]


def mdev_trees(mode):
    """the vGPU tree before each step, then after it: create, destroy, retype, move to another parent, NUMA move of
    a parent (and back to the start); index mode adds a parent that is no BDF and a name that is no UUID"""
    parents = {"0000:01:00.0": "0\n", "0000:02:00.0": "1\n"}
    m0 = {U[1]: dict(type="GRID T4-1Q\n", parent="0000:01:00.0"), U[3]: dict(type="GRID T4-1Q\n", parent="0000:02:00.0"),
          U[4]: dict(type="GRID T4-2Q\n", parent="0000:01:00.0")}
    if mode == "index":
        parents["gpu-a"] = "0\n"
        m0[U[5]] = dict(type="GRID T4-2Q\n", parent="gpu-a")
        m0["zz-vgpu"] = dict(type="GRID T4-1Q\n", parent="0000:02:00.0")
    m1 = dict(m0, **{U[0]: dict(type="GRID T4-2Q\n", parent="0000:02:00.0")})   # create, first in the Walk
    m2 = {k: v for k, v in m1.items() if k != U[3]}                             # destroy
    m3 = dict(m2, **{U[4]: dict(type="GRID T4-4Q\n", parent="0000:01:00.0")})   # retype to a new label
    m4 = dict(m3, **{U[1]: dict(type="GRID T4-1Q\n", parent="0000:02:00.0")})   # move
    p5 = dict(parents, **{"0000:02:00.0": "3\n"})                                # NUMA move
    return [(parents, m0), (parents, m1), (parents, m2), (parents, m3), (parents, m4), (p5, m4), (parents, m0)]


def write_mdev_tree(root, parents, mdevs):
    for sub in ("pci", "mdev"):
        shutil.rmtree(os.path.join(root, sub), ignore_errors=True)
    return util.make_mdev_tree(root, parents, mdevs)


@pytest.mark.parametrize("mode", ["numeric", "index"])
def test_rescan_vgpu_raw_patches_exactly(tmp_path, mode):
    root = str(tmp_path)
    ids = os.path.join(root, "pci.ids")
    with open(ids, "wb") as f:
        f.write(util.pciids_text())
    steps = mdev_trees(mode)
    vgpu, pci = write_mdev_tree(root, *steps[0])

    def fresh():
        ds = kvgpu.DiscoveryScan(pci_ids_path=ids, base_path=pci, vgpu_base_path=vgpu)
        try:
            return ds.create_vgpu_id_map(raw=True)
        finally:
            ds.close()

    ds = kvgpu.DiscoveryScan(pci_ids_path=ids, base_path=pci, vgpu_base_path=vgpu)
    try:
        ds.rescan_vgpu_id_map(raw=True)
        assert dataclasses.asdict(ds.maps) == dataclasses.asdict(fresh())
        for parents, mdevs in steps[1:]:
            before = dataclasses.asdict(ds.maps)
            write_mdev_tree(root, parents, mdevs)
            touched = ds.rescan_vgpu_id_map(raw=True)
            after = dataclasses.asdict(ds.maps)
            assert after == dataclasses.asdict(fresh())
            dirty, gone = changed_keys(before["vGpuMap"], after["vGpuMap"])
            assert set(touched.type_dirty) == dirty and set(touched.type_gone) == gone
            dirty, gone = changed_keys(before["gpuVgpuMap"], after["gpuVgpuMap"])
            assert set(touched.par_dirty) == dirty and set(touched.par_gone) == gone
    finally:
        ds.close()


@pytest.mark.parametrize("mode", ["numeric", "index"])
def test_raw_mdev_feed_resends_only_dirty_labels(tmp_path, mode):
    root = str(tmp_path)
    steps = mdev_trees(mode)
    vgpu, pci = write_mdev_tree(root, *steps[0])
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(util.pciids_text())
        plugins = {}
        feed = serve.MdevRescanFeed(ctx.scan_mdev_raw_delta, lambda: kvgpu.read_mdev_tree_raw(vgpu, pci), kvgpu.Maps(),
                                    plugins, Stub, raw=True)
        feed.tick()
        assert set(plugins) == set(feed.maps.vGpuMap)
        for parents, mdevs in steps[1:]:
            before = {k: list(v) for k, v in feed.maps.vGpuMap.items()}
            sent = {k: p.sent for k, p in plugins.items()}
            write_mdev_tree(root, parents, mdevs)
            touched = feed.tick()
            dirty, gone = changed_keys(before, feed.maps.vGpuMap)
            assert set(touched.type_dirty) == dirty and set(touched.type_gone) == gone
            for k, p in plugins.items():
                assert p.sent - sent.get(k, 0) == (1 if k in dirty and k in sent else 0), k
            assert set(plugins) == set(feed.maps.vGpuMap)
