"""DiscoveryScan.create_iommu_device_map(raw=True) — the walk reads everything and the GPU decodes the reads — builds the
same Maps and the same plugin specs as the default path, on the config-1 tree and the golden Ginkgo entries."""
import dataclasses

import pytest

import util
import kvgpu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tree", ["c1", "ginkgo", "index"])
def test_raw_path_equals_default(tmp_path, tree):
    ent = {"c1": util.c1_tree_entries, "ginkgo": lambda: util.ginkgo()["create_iommu_device_map"]["entries"],
           "index": lambda: {"0000:00:01.0": dict(vendor="10de", device="1db6", driver="vfio-pci", iommu_group="g1",
                                                  numa_node="0"),
                             "zz": dict(vendor="10de", device="0x1db6x", driver="vfio-pci", iommu_group="7",
                                        numa_node="2")}}[tree]()
    base = util.make_pci_tree(str(tmp_path), ent)
    ids = str(tmp_path / "pci.ids")
    with open(ids, "wb") as f:
        f.write(util.pciids_text())
    specs = []
    for raw in (False, True):
        ds = kvgpu.DiscoveryScan(pci_ids_path=ids, base_path=base)
        try:
            maps = ds.create_iommu_device_map(raw=raw)
            specs.append((dataclasses.asdict(maps), [dataclasses.asdict(s) for s in ds.create_device_plugins()],
                          kvgpu.canonical_dump(maps)))
        finally:
            ds.close()
    assert specs[0] == specs[1]
