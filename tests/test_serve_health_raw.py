"""KeyedGroupHealthFeed(raw=True) and KeyedVgpuHealthFeed(raw=True) over real trees: a tmp sysfs tree, a tmp VFIO
device directory and a tmp mdev bus, read each tick with plugin.read_pci_ids_raw / list_nodes_raw /
read_mdev_ids_raw.  The CPU variants run each tick through the string-level state machines of
tests/health_raw_ref.py (a CPU model of Context.health_rescan_*_raw), the GPU variants through the Context calls;
both must send the same events."""
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import health_raw_ref as HR
import kvgpu
import util
from kvgpu import dpapi, serve


class Plugin:
    """What the feeds use of a plugin: its devices, and the two health channels (logged, applied to the device)."""

    def __init__(self, ids, log):
        self.devs = [dpapi.Device(ID=i, health=dpapi.HEALTHY) for i in ids]
        self.log = log

    def _set(self, dev_id, h):
        self.log.append((h, dev_id))
        for d in self.devs:
            if d.ID == dev_id:
                d.health = h

    def healthy(self, dev_id):
        self._set(dev_id, dpapi.HEALTHY)

    def unhealthy(self, dev_id):
        self._set(dev_id, dpapi.UNHEALTHY)

    def relist(self, ids):
        have = {d.ID: d.health for d in self.devs}
        self.devs = [dpapi.Device(ID=i, health=have.get(i, dpapi.HEALTHY)) for i in ids]


def model_groups():
    ref = HR.RawGroupsRef()
    return lambda raw, nodes=(): _as_delta(ref.step(raw, [os.fsencode(n) if isinstance(n, str) else n for n in nodes]))


def model_mdev():
    ref = HR.RawMdevRef()
    return lambda raw, xids=(): _as_delta(ref.step(raw, [os.fsencode(x) if isinstance(x, str) else x for x in xids]))


def _as_delta(d):
    return kvgpu.HealthDelta(d.n_records, d.n_alive, d.changed)


# names the keyed feeds without raw reads refuse: neither canonical BDFs nor canonical UUIDs
A0, A1, B0, C0, X0 = "0000:3b:00.0", "0000:3b:00.1", "0000:86:00.0", "0000:af:00.0", "gpu-x"
GROUP = {A0: "40", A1: "40", B0: "41", C0: "042", X0: "41"}


def run_groups(rescan):
    tmp = tempfile.mkdtemp(prefix="kvg")
    try:
        base = util.make_pci_tree(os.path.join(tmp, "sys"), {
            a: dict(vendor="10de", device="2330", driver="vfio-pci", iommu_group=g, numa_node="0\n")
            for a, g in GROUP.items()})
        devdir = os.path.join(tmp, "vfio")
        os.makedirs(devdir)
        for name in ("vfio", "devices", "40", "41", "42"):      # "42" is not group "042"
            open(os.path.join(devdir, name), "w").close()
        log = []
        pa, pb = Plugin([A0, A1, C0], log), Plugin([B0, X0], log)
        feed = serve.KeyedGroupHealthFeed(rescan, lambda names: kvgpu.read_pci_ids_raw(base, names),
                                          lambda: kvgpu.list_nodes_raw(devdir), [pa, pb], raw=True)

        def tick():
            del log[:]
            assert feed.tick() == len(log)
            return sorted(log)

        assert tick() == [(dpapi.UNHEALTHY, C0)]                # its node does not exist
        assert tick() == []
        os.remove(os.path.join(devdir, "40"))                   # exactly the devices of group 40 flip
        assert tick() == [(dpapi.UNHEALTHY, A0), (dpapi.UNHEALTHY, A1)]
        open(os.path.join(devdir, "40"), "w").close()
        assert tick() == [(dpapi.HEALTHY, A0), (dpapi.HEALTHY, A1)]
        os.remove(os.path.join(devdir, "41"))                   # a non-canonical name flips with its group
        assert tick() == [(dpapi.UNHEALTHY, B0), (dpapi.UNHEALTHY, X0)]
        # a device hot-added elsewhere (a new group with a node): nothing for the others
        util.make_pci_tree(os.path.join(tmp, "sys"), {"0000:d8:00.0": dict(
            vendor="10de", device="2330", driver="vfio-pci", iommu_group="44", numa_node="0\n")})
        open(os.path.join(devdir, "44"), "w").close()
        pb.relist([B0, X0, "0000:d8:00.0"])
        assert tick() == []
        open(os.path.join(devdir, "41"), "w").close()
        assert tick() == [(dpapi.HEALTHY, B0), (dpapi.HEALTHY, X0)]
        # the VFIO directory vanishes: every device goes unhealthy
        shutil.rmtree(devdir)
        assert [d for _, d in tick()] == sorted([A0, A1, B0, X0, "0000:d8:00.0"])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(1, 6)]
V = "vgpu-7"                                                   # not a UUID
P1, P2 = "0000:3b:00.0", "0000:86:00.0"


def run_mdev(rescan):
    tmp = tempfile.mkdtemp(prefix="kvg")
    try:
        root = os.path.join(tmp, "sys")
        vbase, pbase = util.make_mdev_tree(root, {P1: "0\n", P2: "1\n"}, {
            U[0]: dict(type="GRID A100-1B\n", parent=P1), U[1]: dict(type="GRID A100-1B\n", parent=P2),
            U[2]: dict(type="GRID A100-2Q\n", parent=P1), V: dict(type="GRID A100-2Q\n", parent=P2)})
        log = []
        pa, pb = Plugin([U[0], U[1]], log), Plugin([U[2], V], log)
        feed = serve.KeyedVgpuHealthFeed(rescan, lambda names: kvgpu.read_mdev_ids_raw(vbase, pbase, names),
                                         [pa, pb], [("GPU-1", P1), ("GPU-2", P2)], raw=True)

        def tick():
            del log[:]
            assert feed.tick() == len(log)
            return sorted(log)

        assert tick() == [] and tick() == []
        assert feed.on_event(79, "GPU-1") == 1                  # exactly the vGPUs on GPU-1
        assert tick() == [(dpapi.UNHEALTHY, U[0]), (dpapi.UNHEALTHY, U[2])]
        assert tick() == []
        # a vGPU created on GPU-2 and one destroyed there: nothing for the others, the marks stay
        util.make_mdev_tree(root, {}, {U[3]: dict(type="GRID A100-1B\n", parent=P2)})
        pa.relist([U[0], U[1], U[3]])
        assert tick() == []
        os.remove(os.path.join(vbase, U[1]))
        pa.relist([U[0], U[3]])
        assert tick() == []
        assert feed.on_event(43, "GPU-2") == 0                  # an application error marks nothing
        assert tick() == []
        assert feed.on_event(48, "GPU-2") == 1                  # the non-UUID name is marked with its GPU
        assert tick() == [(dpapi.UNHEALTHY, U[3]), (dpapi.UNHEALTHY, V)]
        # only a re-created path clears a mark
        link = os.readlink(os.path.join(vbase, U[0]))
        os.remove(os.path.join(vbase, U[0]))
        assert tick() == []
        os.symlink(link, os.path.join(vbase, U[0]))
        assert tick() == [(dpapi.HEALTHY, U[0])]
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def test_raw_group_feed_cpu_model():
    run_groups(model_groups())


def test_raw_vgpu_feed_cpu_model():
    run_mdev(model_mdev())


def test_non_canonical_names_need_raw():
    fail = lambda *a: pytest.fail("no call for a list that has no keys")  # noqa: E731
    with pytest.raises(ValueError, match=X0):
        serve.KeyedGroupHealthFeed(fail, fail, fail, [Plugin([A0, X0], [])]).tick()
    with pytest.raises(ValueError, match=V):
        serve.KeyedVgpuHealthFeed(fail, fail, [Plugin([U[0], V], [])], []).tick()


@pytest.mark.gpu
def test_raw_group_feed_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        run_groups(ctx.health_rescan_groups_raw)


@pytest.mark.gpu
def test_raw_vgpu_feed_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        run_mdev(ctx.health_rescan_mdev_raw)
