"""Register -> ListAndWatch -> Allocate replayed on the real scan (libkvgpu.so on an H100):
DiscoveryScan over a sysfs-shaped tree (BASELINE.json config 1), the plugin servers of kvgpu.serve,
the Allocate-time re-validation as one batched pass of the classification kernel, the health feed
through the K6 delta kernel — checked against the oracle's view of the same tree."""
import os
import shutil
import tempfile

import numpy as np
import pytest

import conftest  # noqa: F401
import util

pytestmark = pytest.mark.gpu


@pytest.fixture()
def world(tmp_path):
    import kvgpu
    from kvgpu import serve
    ids = tmp_path / "pci.ids"
    ids.write_bytes(util.pciids_text())
    base = util.make_pci_tree(str(tmp_path / "pci"), util.c1_tree_entries())
    ds = kvgpu.DiscoveryScan(str(ids), base, str(tmp_path / "nomdev"))
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")
    kubelet = serve.MockKubelet(sockdir).start()
    yield kvgpu, serve, ds, base, sockdir, kubelet
    kubelet.stop()
    ds.close()
    shutil.rmtree(sockdir, ignore_errors=True)


def test_scan_to_kubelet_round_trip(world):
    import grpc
    from oracle import oracle as O
    kvgpu, serve, ds, base, sockdir, kubelet = world
    maps = ds.create_iommu_device_map()
    m = O.Maps()
    m.create_iommu_device_map_tree(base)
    assert kvgpu.canonical_dump(maps) == m.dump(util.pciids_text())

    reval = serve.BatchRevalidator(ds.ctx.scan_pci, base)
    plugins = serve.plugins_from_specs(ds.create_device_plugins(), maps, reval, socket_dir=sockdir, base_path=base,
                                       root_path=sockdir, discover_egm=lambda: [])
    try:
        for p in plugins:
            p.start()
        regs = kubelet.wait_for(len(plugins))
        by_res = {r.resource_name: r for r in regs}
        assert "nvidia.com/GP102GL_TESLA_P40" in by_res
        c = kubelet.connect(by_res["nvidia.com/GP102GL_TESLA_P40"])
        first = next(c.list_and_watch())
        assert [d.ID for d in first.devices] == ["0000:%s:00.0" % b for b in ("04", "05", "06", "07", "84", "85", "86", "87")]
        assert [d.topology.nodes[0].ID for d in first.devices] == [0, 0, 0, 0, 1, 1, 1, 1]

        # group 40 = the GPU and its audio function: both are re-validated in one batch, both listed
        r = c.allocate(["0000:04:00.0"]).container_responses[0]
        assert dict(r.envs) == {"PCI_RESOURCE_NVIDIA_COM_GP102GL_TESLA_P40": "0000:04:00.0,0000:04:00.1"}
        assert [d.host_path for d in r.devices] == ["/dev/vfio/vfio", "/dev/vfio/40"]
        r = c.allocate(["0000:84:00.0", "0000:87:00.0"]).container_responses[0]
        assert r.envs["PCI_RESOURCE_NVIDIA_COM_GP102GL_TESLA_P40"].endswith("0000:84:00.0,0000:87:00.0")

        # the vendor of 0000:05:00.0 changes on the system -> refused with the reference's text
        real = os.path.realpath(os.path.join(base, "0000:05:00.0"))
        with open(os.path.join(real, "vendor"), "w") as f:
            f.write("0x8086\n")
        with pytest.raises(grpc.RpcError) as e:
            c.allocate(["0000:05:00.0"])
        assert e.value.details() == "invalid allocation request: unknown device: 0000:05:00.0"
        # the iommu group link of 0000:06:00.0 moves
        real = os.path.realpath(os.path.join(base, "0000:06:00.0"))
        os.remove(os.path.join(real, "iommu_group"))
        os.symlink("../../../kernel/iommu_groups/99", os.path.join(real, "iommu_group"))
        with pytest.raises(grpc.RpcError) as e:
            c.allocate(["0000:07:00.0", "0000:06:00.0"])
        assert e.value.details() == "invalid allocation request: unknown device: 0000:06:00.0"
        assert dict(c.allocate(["0000:07:00.0"]).container_responses[0].envs)   # unaffected devices still allocate
        c.close()
    finally:
        for p in plugins:
            p.stop()


def test_health_feed_through_the_delta_kernel(world):
    kvgpu, serve, ds, base, sockdir, kubelet = world
    maps = ds.create_iommu_device_map()
    plugins = serve.plugins_from_specs(ds.create_device_plugins(), maps, None, socket_dir=sockdir)
    p40 = [p for p in plugins if p.device_name == "GP102GL_TESLA_P40"][0]

    def snapshot():
        snap = kvgpu.snapshot_pci_tree(base)
        return snap.recs, snap.names
    ds.ctx.health_reset()
    feed = serve.HealthRescanFeed(ds.ctx.health_rescan, snapshot, plugins)
    assert feed.tick() == 0 and feed.tick() == 0
    # 0000:85:00.0 loses its vfio driver binding
    real = os.path.realpath(os.path.join(base, "0000:85:00.0"))
    os.remove(os.path.join(real, "driver"))
    assert feed.tick() == 1 and p40._events.get_nowait() == ("unhealthy", "0000:85:00.0")
    os.symlink("../../../bus/pci/drivers/vfio-pci", os.path.join(real, "driver"))
    assert feed.tick() == 1 and p40._events.get_nowait() == ("healthy", "0000:85:00.0")
    stream = p40.ListAndWatch(None, None)
    assert all(d.health == "Healthy" for d in next(stream).devices)
    p40.unhealthy("0000:85:00.0")
    assert [d.health for d in next(stream).devices].count("Unhealthy") == 1
