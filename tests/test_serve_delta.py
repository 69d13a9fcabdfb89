"""PciRescanFeed over real gRPC with MockKubelet: a sysfs tree under a temporary directory changes between ticks
and the plugin set follows it.  A hot-added device with a new device id registers a new plugin; removing one member
of a key makes its plugin re-send the shorter list; removing the last device of a key stops its plugin; moving a
device to another IOMMU group changes what Allocate expands to.  The CPU variant computes each scan and delta with
the numpy restatements of tests/util.py and tests/delta_ref.py; the GPU variant runs Context.scan_pci_delta."""
import os
import shutil
import tempfile

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import delta_ref
import util
from kvgpu import _lib as L
from kvgpu import dpapi, serve


def numpy_scan_delta():
    """scan_pci_delta restated in numpy: the result (no names joined) and the delta against the previous call."""
    prev = [np.zeros(0, dtype=L.PCI_SURV)]

    def ordering(keys):
        order = np.argsort(keys, kind="stable")
        uk, first = np.unique(keys[order], return_index=True)
        return uk, np.append(first, len(keys)).astype(np.uint32), order.astype(np.uint32)

    def scan(recs):
        e = util.expect_pci(recs)
        s = np.zeros(len(e["addr"]), dtype=L.PCI_SURV)
        for f in ("addr", "iommu_group", "device", "numa"):
            s[f] = e[f]
        s["name_slot"] = L.KVG_NO_NAME
        dk, doff, dperm = ordering(s["device"])
        gk, goff, gperm = ordering(s["iommu_group"])
        res = kvgpu.PciResult(len(recs), s, dk.astype(np.uint16), doff, dperm,
                              np.full(len(dk), L.KVG_NO_NAME, np.uint32), gk.astype(np.uint32), goff, gperm, b"")
        d = delta_ref.expect_pci_delta(prev[0], s, L.PCI_CHANGE)
        delta = kvgpu.PciDelta(len(prev[0]), d["changes"], d["dev_dirty"], d["dev_gone"], d["grp_dirty"], d["grp_gone"])
        prev[0] = s
        return res, delta
    return scan


def entry(device, group, numa="0\n"):
    return dict(vendor="10de", device=device, driver="vfio-pci", iommu_group=group, numa_node=numa)


def regroup(root, addr, group):
    link = os.path.join(root, "real", addr, "iommu_group")
    tgt = os.path.join(root, "targets", "iommu_groups", group)
    os.makedirs(tgt, exist_ok=True)
    os.remove(link)
    os.symlink(tgt, link)


def run_scenario(scan_delta):
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")     # unix socket paths are limited to 107 bytes
    root = os.path.join(sockdir, "sys")
    base = util.make_pci_tree(root, {"0000:04:00.0": entry("1b38", "40"), "0000:04:00.1": entry("1b38", "40"),
                                     "0000:05:00.0": entry("1b38", "41", "1\n"), "0000:06:00.0": entry("20b0", "42")})
    kubelet = serve.MockKubelet(sockdir).start()
    maps, plugins = kvgpu.Maps(), {}

    def make_plugin(spec):
        return serve.GenericDevicePlugin(spec.device_name, serve.VFIO_DEVICE_PATH, serve.devices_from_spec(spec), maps,
                                         revalidate=lambda pairs: None, base_path=base, root_path=sockdir,
                                         discover_egm=lambda: [], socket_dir=sockdir,
                                         kubelet_socket=kubelet.socket_path)
    feed = serve.PciRescanFeed(scan_delta, lambda: kvgpu.snapshot_pci_tree(base), maps, plugins, make_plugin)
    clients = []
    try:
        feed.tick()
        assert sorted(plugins) == ["1b38", "20b0"] and len(kubelet.wait_for(2)) == 2
        c = kubelet.connect(next(r for r in kubelet.registrations
                                 if r.endpoint == os.path.basename(plugins["1b38"].socket_path)))
        clients.append(c)
        stream = c.list_and_watch()
        assert [d.ID for d in next(stream).devices] == ["0000:04:00.0", "0000:04:00.1", "0000:05:00.0"]
        plugins["1b38"].unhealthy("0000:04:00.1")
        assert [d.health for d in next(stream).devices] == ["Healthy", "Unhealthy", "Healthy"]

        # hot-add with a new device id: a new plugin registers
        util.make_pci_tree(root, {"0000:07:00.0": entry("2330", "43")})
        t = feed.tick()
        assert t.dev_dirty == ["2330"] and t.dev_gone == []
        assert "2330" in plugins and len(kubelet.wait_for(3)) == 3

        # one member of 1b38 goes: the plugin re-sends the shorter list, the survivor keeps its health
        os.remove(os.path.join(base, "0000:05:00.0"))
        t = feed.tick()
        assert t.dev_dirty == ["1b38"] and "41" in t.grp_gone
        got = next(stream).devices
        assert [(d.ID, d.health) for d in got] == [("0000:04:00.0", "Healthy"), ("0000:04:00.1", "Unhealthy")]
        stream.cancel()

        # the last device of 20b0 goes: its plugin stops
        p20 = plugins["20b0"]
        os.remove(os.path.join(base, "0000:06:00.0"))
        t = feed.tick()
        assert t.dev_gone == ["20b0"] and "20b0" not in plugins and p20.server is None
        assert "20b0" not in maps.deviceMap and "0000:06:00.0" not in maps.bdfToIommuMap

        # a device moves to another group: Allocate expands to the new group
        c2 = kubelet.connect(next(r for r in kubelet.registrations
                                  if r.endpoint == os.path.basename(plugins["2330"].socket_path)))
        clients.append(c2)
        r = c2.allocate(["0000:07:00.0"]).container_responses[0]
        assert [d.host_path for d in r.devices] == ["/dev/vfio/vfio", "/dev/vfio/43"]
        regroup(root, "0000:07:00.0", "44")
        t = feed.tick()
        assert t.dev_dirty == [] and t.grp_dirty == ["44"] and t.grp_gone == ["43"]
        r = c2.allocate(["0000:07:00.0"]).container_responses[0]
        assert [d.host_path for d in r.devices] == ["/dev/vfio/vfio", "/dev/vfio/44"]
        assert maps.bdfToIommuMap["0000:07:00.0"] == "44"
    finally:
        for c in clients:
            c.close()
        for p in plugins.values():
            p.stop()
        kubelet.stop()
        shutil.rmtree(sockdir, ignore_errors=True)


def test_feed_follows_the_tree_numpy_reference():
    run_scenario(numpy_scan_delta())


@pytest.mark.gpu
def test_feed_follows_the_tree_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(util.pciids_text())
        run_scenario(ctx.scan_pci_delta)
