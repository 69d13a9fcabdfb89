"""KeyedVgpuHealthFeed and KeyedGroupHealthFeed over real gRPC with MockKubelet.

vGPUs: the scenario of VgpuHealthFeed (test_serve_health_mdev.py) up to the XID marks, then the advertised list grows
by a vGPU whose path does not exist.  The keyed feed sends exactly one event (the new vGPU goes unhealthy) and the
marked vGPUs stay unhealthy; only a re-created path clears a mark.

IOMMU groups: one sequence of trees and advertised lists (nodes created and removed, devices added to and dropped from
both plugins) run once through GroupHealthFeed and once through KeyedGroupHealthFeed.  The event streams are equal;
the keyed feed makes one kernel call per tick, where the index feed makes two on a tick whose list changed.

The CPU variants compute each tick with the numpy state machines of tests/health_*_ref.py; the GPU variants run the
Context calls."""
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import health_groups_ref
import health_keyed_ref
import kvgpu
import util
from kvgpu import dpapi, serve

U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(1, 6)]
P1, P2 = "0000:3b:00.0", "0000:86:00.0"


def health(stream, k=1):
    """The device list after k more ListAndWatch sends (one per health event or list change)."""
    for _ in range(k):
        devs = next(stream).devices
    return [(d.ID, d.health) for d in devs]


def run_vgpu_scenario(health_rescan_mdev_keyed):
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")     # unix socket paths are limited to 107 bytes
    root = os.path.join(sockdir, "sys")
    vbase, pbase = util.make_mdev_tree(root, {P1: "0\n", P2: "1\n"}, {
        U[0]: dict(type="GRID A100-1B\n", parent=P1),
        U[1]: dict(type="GRID A100-1B\n", parent=P2),
        U[2]: dict(type="GRID A100-2Q\n", parent=P1)})
    kubelet = serve.MockKubelet(sockdir).start()

    def plugin(name, ids):
        return serve.GenericVGpuDevicePlugin(name, "vgpu", [dpapi.Device(ID=u, health=dpapi.HEALTHY) for u in ids],
                                             vgpu_base_path=vbase, socket_dir=sockdir,
                                             kubelet_socket=kubelet.socket_path)
    pa, pb = plugin("GRID_A100-1B", U[:2]), plugin("GRID_A100-2Q", U[2:3])
    clients = []
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
        assert health(sa) == [(U[0], "Healthy"), (U[1], "Healthy")] and health(sb) == [(U[2], "Healthy")]
        gpus = [("GPU-1", P1), ("GPU-2", P2)]
        feed = serve.KeyedVgpuHealthFeed(health_rescan_mdev_keyed,
                                         lambda uuids, intern: kvgpu.snapshot_mdev_ids(vbase, pbase, uuids, intern),
                                         [pa, pb], gpus)

        # GPU-2 could not register for XID events: its vGPU is unhealthy from the first tick on
        assert feed.on_unsupported("GPU-2") == 1
        assert feed.tick() == 1
        assert health(sa) == [(U[0], "Healthy"), (U[1], "Unhealthy")]
        assert feed.tick() == 0

        # XID 79 on GPU-1 marks both of its vGPUs; the marks stay
        assert feed.on_event(79, "GPU-1") == 1
        assert feed.tick() == 2
        assert health(sa) == [(U[0], "Unhealthy"), (U[1], "Unhealthy")] and health(sb) == [(U[2], "Unhealthy")]
        assert feed.tick() == 0

        # the advertised list grows by a vGPU whose path does not exist: one event (it goes unhealthy), and the
        # marked vGPUs stay unhealthy
        pb.set_devices([dpapi.Device(ID=U[2], health=dpapi.UNHEALTHY), dpapi.Device(ID=U[3], health=dpapi.HEALTHY)])
        assert health(sb) == [(U[2], "Unhealthy"), (U[3], "Healthy")]
        assert feed.tick() == 1
        assert health(sb) == [(U[2], "Unhealthy"), (U[3], "Unhealthy")]
        assert feed.tick() == 0

        # and shrinks again: nothing to send, the marks still stay
        pb.set_devices([dpapi.Device(ID=U[2], health=dpapi.UNHEALTHY)])
        assert health(sb) == [(U[2], "Unhealthy")]
        assert feed.tick() == 0

        # only a re-created path clears a mark: U[0] removed (no transition), restored (healthy)
        link = os.readlink(os.path.join(vbase, U[0]))
        os.remove(os.path.join(vbase, U[0]))
        assert feed.tick() == 0
        os.symlink(link, os.path.join(vbase, U[0]))
        assert feed.tick() == 1
        assert health(sa) == [(U[0], "Healthy"), (U[1], "Unhealthy")]
        assert feed.tick() == 0
        for s in streams:
            s.cancel()
    finally:
        for c in clients:
            c.close()
        for p in (pa, pb):
            p.stop()
        kubelet.stop()
        shutil.rmtree(sockdir, ignore_errors=True)


A0, A1, B0, B1, C0, D0, E0 = ("0000:3b:00.0", "0000:3b:00.1", "0000:86:00.0", "0000:86:00.1", "0000:af:00.0",
                              "0000:d8:00.0", "0000:06:00.0")
GROUP = {A0: "40", A1: "40", B0: "41", B1: "41", C0: "42", E0: "43"}


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


def run_group_sequence(feed_cls, health_rescan_groups):
    """-> [(sorted events, kernel calls)] per tick of one fixed sequence of trees and advertised lists."""
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")
    root = os.path.join(sockdir, "sys")
    base = util.make_pci_tree(root, {a: dict(vendor="10de", device="2330", driver="vfio-pci", iommu_group=g,
                                             numa_node="0\n") for a, g in GROUP.items()})
    devdir = os.path.join(sockdir, "vfio")
    os.makedirs(devdir)
    for name in ("vfio", "40", "41", "43"):                    # the node of group 42 is absent from the start
        open(os.path.join(devdir, name), "w").close()
    kubelet = serve.MockKubelet(sockdir).start()
    log, calls = [], []

    def counted(recs, nodes=()):
        calls.append(len(recs))
        return health_rescan_groups(recs, nodes)

    def plugin(name, bdfs):
        return LoggedPlugin(name, devdir, [dpapi.Device(ID=b, health=dpapi.HEALTHY) for b in bdfs], serve.Maps(),
                            log=log, socket_dir=sockdir, kubelet_socket=kubelet.socket_path)
    pa, pb = plugin("GH100_A", [A0, A1, C0]), plugin("GH100_B", [B0, B1])
    clients, out = [], []
    try:
        for p in (pa, pb):
            p.start()
        regs = kubelet.wait_for(2)
        streams = {}
        for p in (pa, pb):
            c = kubelet.connect(next(r for r in regs if r.endpoint == os.path.basename(p.socket_path)))
            clients.append(c)
            streams[p] = c.list_and_watch()
            health(streams[p])
        feed = feed_cls(counted, lambda bdfs, intern: kvgpu.snapshot_pci_ids(base, bdfs, intern),
                        lambda intern: kvgpu.group_nodes(devdir, intern), [pa, pb])

        def node(name):
            return os.path.join(devdir, name)

        def relist(p, bdfs):
            p.set_devices([dpapi.Device(ID=b, health=dpapi.HEALTHY) for b in bdfs])
            health(streams[p])

        steps = [lambda: None,
                 lambda: open(node("42"), "w").close(),
                 lambda: os.remove(node("40")),
                 lambda: relist(pb, [B0, B1, D0]),                      # a device whose sysfs entry does not exist
                 lambda: None,
                 lambda: open(node("40"), "w").close(),
                 lambda: relist(pa, [A1, C0]),                          # A0 dropped
                 lambda: os.remove(node("41")),
                 lambda: relist(pb, [E0, B0, B1]),                      # E0 (ascends first) added, D0 dropped
                 lambda: (os.remove(node("43")), open(node("41"), "w").close()),
                 lambda: relist(pa, [A0, A1, C0]),                      # A0 back
                 lambda: None]
        for change in steps:
            del log[:], calls[:]
            change()
            sent = feed.tick()
            assert sent == len(log)
            for p in (pa, pb):                                          # ListAndWatch has applied every event
                mine = [b for _, b in log if any(d.ID == b for d in p.devs)]
                if mine:
                    health(streams[p], len(mine))
            out.append((sorted(log), len(calls)))
        for s in streams.values():
            s.cancel()
    finally:
        for c in clients:
            c.close()
        for p in (pa, pb):
            p.stop()
        kubelet.stop()
        shutil.rmtree(sockdir, ignore_errors=True)
    return out


LIST_CHANGES = {0, 3, 6, 8, 10}          # the ticks of run_group_sequence whose advertised list differs


def check_group_streams(index_rescan, keyed_rescan):
    old = run_group_sequence(serve.GroupHealthFeed, index_rescan)
    new = run_group_sequence(serve.KeyedGroupHealthFeed, keyed_rescan)
    assert [e for e, _ in new] == [e for e, _ in old]
    assert [c for _, c in new] == [1] * len(new)
    assert [c for _, c in old] == [2 if t in LIST_CHANGES else 1 for t in range(len(old))]
    assert sum(len(e) for e, _ in new) > 10


def test_keyed_vgpu_feed_numpy_reference():
    run_vgpu_scenario(health_keyed_ref.KeyedMdevRef().rescan)


def test_keyed_group_feed_numpy_reference():
    check_group_streams(health_groups_ref.HealthGroupsRef().rescan, health_keyed_ref.KeyedGroupsRef().rescan)


def test_keyed_feeds_refuse_names_that_are_not_keys():
    class P:
        def __init__(self, ids):
            self.devs = [dpapi.Device(ID=i, health=dpapi.HEALTHY) for i in ids]
    fail = lambda *a: pytest.fail("no call for a list that has no keys")  # noqa: E731
    bad = "0000000A-0000-4000-8000-00000000000A"             # upper-case hex: not the kernel's canonical name
    feed = serve.KeyedVgpuHealthFeed(fail, fail, [P([U[0], bad])], [])
    with pytest.raises(ValueError, match=bad):
        feed.tick()
    feed = serve.KeyedGroupHealthFeed(fail, fail, fail, [P([A0, "3b:00.1"])])
    with pytest.raises(ValueError, match="3b:00.1"):
        feed.tick()


@pytest.mark.gpu
def test_keyed_vgpu_feed_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        run_vgpu_scenario(ctx.health_rescan_mdev_keyed)


@pytest.mark.gpu
def test_keyed_group_feed_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        check_group_streams(ctx.health_rescan_groups, ctx.health_rescan_groups_keyed)
