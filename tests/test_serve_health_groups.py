"""GroupHealthFeed over real gRPC with MockKubelet: the passthrough health check of generic_device_plugin.go:611-690
driven by a PCI tree and a VFIO device directory under a temporary directory.  Two plugins, two groups of two
functions and one of one; a group node absent before the first tick, nodes removed, renamed and created, unrelated
names in the directory, a driver rebind the node watch cannot see, and an advertised list that grows (the feed
re-arms and reconciles).  DeviceNodeWatcher runs on the same directory beside the feed: while only nodes change, its
healthy / unhealthy stream with repeats removed is the feed's.  The CPU variant computes each tick with the numpy
state machine of tests/health_groups_ref.py; the GPU variant runs Context.health_rescan_groups."""
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import health_groups_ref
import kvgpu
import util
from kvgpu import dpapi, serve

A0, A1, B0, B1, C0 = "0000:3b:00.0", "0000:3b:00.1", "0000:86:00.0", "0000:86:00.1", "0000:af:00.0"
GROUP = {A0: "40", A1: "40", B0: "41", B1: "41", C0: "42"}


class LoggedPlugin(serve.GenericDevicePlugin):
    """A passthrough plugin that also logs what goes down its healthy / unhealthy channels."""

    def __init__(self, *a, log, **kw):
        super().__init__(*a, **kw)
        self.log = log

    def healthy(self, dev_id):
        self.log.append(("healthy", dev_id))
        super().healthy(dev_id)

    def unhealthy(self, dev_id):
        self.log.append(("unhealthy", dev_id))
        super().unhealthy(dev_id)


def health(stream, k=1):
    """The device list after k more ListAndWatch sends (one per health event)."""
    for _ in range(k):
        devs = next(stream).devices
    return [(d.ID, d.health) for d in devs]


def run_scenario(health_rescan_groups):
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")     # unix socket paths are limited to 107 bytes
    root = os.path.join(sockdir, "sys")
    base = util.make_pci_tree(root, {a: dict(vendor="10de", device="2330", driver="vfio-pci", iommu_group=g,
                                             numa_node="0\n") for a, g in GROUP.items()})
    devdir = os.path.join(sockdir, "vfio")
    os.makedirs(devdir)
    for name in ("vfio", "40", "41"):                          # the node of group 42 is absent from the start
        open(os.path.join(devdir, name), "w").close()
    kubelet = serve.MockKubelet(sockdir).start()
    feed_log, watch_log = [], []

    def plugin(name, bdfs, log, prefix=""):
        return LoggedPlugin(prefix + name, devdir, [dpapi.Device(ID=b, health=dpapi.HEALTHY) for b in bdfs],
                            serve.Maps(), log=log, socket_dir=sockdir, kubelet_socket=kubelet.socket_path)
    pa, pb = plugin("GH100_A", [A0, A1, C0], feed_log), plugin("GH100_B", [B0, B1], feed_log)
    clients, watchers = [], []
    try:
        for p in (pa, pb):
            p.start()
        regs = kubelet.wait_for(2)
        streams = []
        for p in (pa, pb):
            c = kubelet.connect(next(r for r in regs if r.endpoint == os.path.basename(p.socket_path)))
            clients.append(c)
            streams.append(c.list_and_watch())
        sa, sb = streams
        assert health(sa) == [(A0, "Healthy"), (A1, "Healthy"), (C0, "Healthy")]
        assert health(sb) == [(B0, "Healthy"), (B1, "Healthy")]
        feed = serve.GroupHealthFeed(health_rescan_groups,
                                     lambda bdfs, intern: kvgpu.snapshot_pci_ids(base, bdfs, intern),
                                     lambda intern: kvgpu.group_nodes(devdir, intern), [pa, pb])

        # arming: the device whose node is absent goes unhealthy at once
        assert feed.tick() == 1
        assert health(sa) == [(A0, "Healthy"), (A1, "Healthy"), (C0, "Unhealthy")]
        assert feed.tick() == 0
        assert feed.intern == {"40": 1, "42": 2, "41": 3}          # in the order the advertised devices meet them

        # the reference's own watch beside the feed, one per plugin, on recorders that are not served
        for p in (pa, pb):
            rec = plugin(p.device_name, [d.ID for d in p.devs], watch_log, prefix="watch-")
            watchers.append(serve.DeviceNodeWatcher(rec, bdf_to_iommu=GROUP))
        state = {b: b != C0 for b in GROUP}

        def step(change, sent):
            del feed_log[:], watch_log[:]
            change()
            assert feed.tick() == sent
            for w in watchers:
                w.poll_once()
            kept = []
            for kind, b in watch_log:                          # the watch's stream with repeats removed
                if state[b] != (kind == "healthy"):
                    state[b] = kind == "healthy"
                    kept.append((kind, b))
            assert sorted(feed_log) == sorted(kept), (feed_log, watch_log)

        def node(name):
            return os.path.join(devdir, name)

        step(lambda: open(node("42"), "w").close(), 1)                            # Create
        assert health(sa) == [(A0, "Healthy"), (A1, "Healthy"), (C0, "Healthy")]
        step(lambda: os.remove(node("40")), 2)                                   # Remove: both functions
        assert health(sa, 2) == [(A0, "Unhealthy"), (A1, "Unhealthy"), (C0, "Healthy")]
        step(lambda: os.rename(node("41"), node("41.gone")), 2)                  # Rename
        assert health(sb, 2) == [(B0, "Unhealthy"), (B1, "Unhealthy")]
        step(lambda: (open(node("99"), "w").close(), os.makedirs(node("devices"))), 0)   # nothing of ours
        step(lambda: (open(node("40"), "w").close(), open(node("41"), "w").close()), 4)  # both groups back
        assert health(sa, 2) == [(A0, "Healthy"), (A1, "Healthy"), (C0, "Healthy")]
        assert health(sb, 2) == [(B0, "Healthy"), (B1, "Healthy")]
        step(lambda: os.remove(node("42")), 1)
        assert health(sa) == [(A0, "Healthy"), (A1, "Healthy"), (C0, "Unhealthy")]

        # a driver rebind with the node in place: the feed sees it, the node watch cannot
        drv = os.path.join(root, "real", B1, "driver")
        os.remove(drv)
        os.symlink(os.path.join(root, "targets", "drivers", "nvidia"), drv)
        assert feed.tick() == 1
        assert health(sb) == [(B0, "Healthy"), (B1, "Unhealthy")]
        os.remove(drv)
        os.symlink(os.path.join(root, "targets", "drivers", "vfio-pci"), drv)
        assert feed.tick() == 1
        assert health(sb) == [(B0, "Healthy"), (B1, "Healthy")]

        # the advertised list grows by a device whose sysfs entry does not exist: the feed re-arms and sends what
        # differs from what the plugins advertise
        pb.set_devices([dpapi.Device(ID=B0, health=dpapi.HEALTHY), dpapi.Device(ID=B1, health=dpapi.HEALTHY),
                        dpapi.Device(ID="0000:d8:00.0", health=dpapi.HEALTHY)])
        assert health(sb) == [(B0, "Healthy"), (B1, "Healthy"), ("0000:d8:00.0", "Healthy")]
        assert feed.tick() == 1
        assert health(sb) == [(B0, "Healthy"), (B1, "Healthy"), ("0000:d8:00.0", "Unhealthy")]
        assert feed.tick() == 0
        for s in streams:
            s.cancel()
    finally:
        for w in watchers:
            w.stop()
        for c in clients:
            c.close()
        for p in (pa, pb):
            p.stop()
        kubelet.stop()
        shutil.rmtree(sockdir, ignore_errors=True)


def test_group_nodes_and_snapshot_by_address(tmp_path):
    """snapshot_pci_ids keeps the caller's order and the intern dict across snapshots; an address that is gone reads as
    a vendor error; group_nodes resolves node names through the same dict and drops every other name."""
    base = util.make_pci_tree(str(tmp_path / "sys"), {
        A0: dict(vendor="10de", device="2330", driver="vfio-pci", iommu_group="17", numa_node="1\n"),
        B0: dict(vendor="10de", device="2330", driver="vfio-pci", iommu_group="5", numa_node="0\n")})
    intern = {}
    snap = kvgpu.snapshot_pci_ids(base, [B0, "0000:00:01.0", A0], intern)
    assert intern == {"5": 1, "17": 2} and snap.group_names == ["", "5", "17"] and snap.names == [B0, "0000:00:01.0", A0]
    assert list(snap.recs["iommu_group"]) == [1, 0, 2] and list(snap.recs["addr"]) == [kvgpu.parse_bdf(b) for b in
                                                                                    (B0, "0000:00:01.0", A0)]
    assert list(snap.recs["flags"] & kvgpu._lib.PF_VENDOR_ERR) == [0, kvgpu._lib.PF_VENDOR_ERR, 0]
    assert list(snap.recs["numa"]) == [0, 0, 1] and list(snap.recs["device"]) == [0x2330, 0, 0x2330]
    assert list(kvgpu.snapshot_pci_ids(base, [A0], intern).recs["iommu_group"]) == [2]      # handles stay
    devdir = tmp_path / "vfio"
    assert list(kvgpu.group_nodes(str(devdir), intern)) == []                               # no directory, no node
    devdir.mkdir()
    for name in ("vfio", "17", "5", "99"):
        (devdir / name).touch()
    (devdir / "devices").mkdir()
    nodes = kvgpu.group_nodes(str(devdir), intern)
    assert nodes.dtype == "uint32" and list(nodes) == [1, 2]


def test_group_health_feed_numpy_reference():
    run_scenario(health_groups_ref.HealthGroupsRef().rescan)


@pytest.mark.gpu
def test_group_health_feed_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        run_scenario(ctx.health_rescan_groups)
