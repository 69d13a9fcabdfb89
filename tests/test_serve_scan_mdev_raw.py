"""DiscoveryScan.create_vgpu_id_map(raw=True) -- the walk reads everything and the GPU decodes the reads -- builds the
same Maps and plugin specs as the default path on the Ginkgo and a canonical mdev tree, and the oracle's gpuVgpuMap
keys on a tree with an empty parent component, where the default path keys the vGPU under "0000:00:00.0"."""
import dataclasses

import pytest

import util
import kvgpu
from oracle import oracle as O
from mdev_raw_cases import trees

pytestmark = pytest.mark.gpu


def scan(tmp_path, vbase, pbase, raw):
    ids = str(tmp_path / "pci.ids")
    with open(ids, "wb") as f:
        f.write(util.pciids_text())
    ds = kvgpu.DiscoveryScan(pci_ids_path=ids, base_path=pbase, vgpu_base_path=vbase)
    try:
        maps = ds.create_vgpu_id_map(raw=raw)
        return (dataclasses.asdict(maps), [dataclasses.asdict(s) for s in ds.create_device_plugins()],
                kvgpu.canonical_dump(maps))
    finally:
        ds.close()


@pytest.mark.parametrize("tree", ["ginkgo", "canonical", "empty-parent"])
def test_raw_path(tmp_path, tree):
    name, vbase, pbase, plain = next(t for t in trees(tmp_path) if t[0] == tree)
    got = scan(tmp_path, vbase, pbase, True)
    if plain:
        assert got == scan(tmp_path, vbase, pbase, False)
    else:
        om = O.Maps()
        om.create_vgpu_id_map_tree(vbase, pbase)
        assert got[2] == om.dump(util.pciids_text())
        assert "" in got[0]["gpuVgpuMap"] and "" not in scan(tmp_path, vbase, pbase, False)[0]["gpuVgpuMap"]
