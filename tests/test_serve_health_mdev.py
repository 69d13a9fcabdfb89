"""VgpuHealthFeed over real gRPC with MockKubelet: the vGPU health check of generic_vgpu_device_plugin.go:280-385 driven
by an mdev tree under a temporary directory and by XID events.  An mdev symlink removed and restored, XID 79 on one GPU
(31 / 43 / 45 ignored), an event without a UUID, a GPU marked by on_unsupported before the first tick, an NVML bus id
that matches no sysfs parent string, and an advertised UUID list that grows (the feed re-arms and reconciles).  The CPU
variant computes each tick with the numpy state machine of tests/health_mdev_ref.py; the GPU variant runs
Context.health_rescan_mdev."""
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import health_mdev_ref
import kvgpu
import util
from kvgpu import dpapi, serve

U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(1, 6)]
P1, P2 = "0000:3b:00.0", "0000:86:00.0"


def health(stream):
    return [(d.ID, d.health) for d in next(stream).devices]


def run_scenario(health_rescan_mdev):
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
        gpus = [("GPU-1", P1), ("GPU-2", P2), ("GPU-3", "00000000:3B:00.0")]   # GPU-3: NVML's spelling of P1
        feed = serve.VgpuHealthFeed(health_rescan_mdev,
                                    lambda uuids, intern: kvgpu.snapshot_mdev_ids(vbase, pbase, uuids, intern),
                                    [pa, pb], gpus)

        # GPU-2 could not register for XID events: its vGPU is unhealthy from the first tick on
        assert feed.on_unsupported("GPU-2") == 1
        assert feed.tick() == 1
        assert health(sa) == [(U[0], "Healthy"), (U[1], "Unhealthy")]
        assert feed.tick() == 0

        # an mdev symlink removed, then restored
        link = os.readlink(os.path.join(vbase, U[0]))
        os.remove(os.path.join(vbase, U[0]))
        assert feed.tick() == 1
        assert health(sa) == [(U[0], "Unhealthy"), (U[1], "Unhealthy")]
        os.symlink(link, os.path.join(vbase, U[0]))
        assert feed.tick() == 1
        assert health(sa) == [(U[0], "Healthy"), (U[1], "Unhealthy")]

        # application errors are ignored; XID 79 on GPU-1 marks both of its vGPUs
        for xid in serve.XID_APPLICATION_ERRORS:
            assert feed.on_event(xid, "GPU-1") == 0
        assert feed.tick() == 0
        assert feed.on_event(79, "GPU-1") == 1
        assert feed.tick() == 2
        assert health(sa) == [(U[0], "Unhealthy"), (U[1], "Unhealthy")] and health(sb) == [(U[2], "Unhealthy")]
        assert feed.tick() == 0                                     # the mark stays

        # a bus id string that is not the sysfs parent string marks nothing (the reference's map miss)
        assert feed.on_event(79, "GPU-3") == 1
        assert feed.tick() == 0

        # only a Create clears a mark: U[2] removed (no transition), restored (healthy)
        link2 = os.readlink(os.path.join(vbase, U[2]))
        os.remove(os.path.join(vbase, U[2]))
        assert feed.tick() == 0
        os.symlink(link2, os.path.join(vbase, U[2]))
        assert feed.tick() == 1
        assert health(sb) == [(U[2], "Healthy")]

        # an event without a UUID marks every GPU: U[2] goes (U[0] and U[1] are marked already)
        assert feed.on_event(48) == 3
        assert feed.tick() == 1
        assert health(sb) == [(U[2], "Unhealthy")]

        # the advertised list grows by a vGPU whose path does not exist: the feed re-arms and sends what differs
        # from what the plugins advertise.  The marks go with the old state: every present vGPU is healthy again.
        pb.set_devices([dpapi.Device(ID=U[2], health=dpapi.UNHEALTHY), dpapi.Device(ID=U[3], health=dpapi.HEALTHY)])
        assert health(sb) == [(U[2], "Unhealthy"), (U[3], "Healthy")]
        assert feed.tick() == 4
        assert health(sa) == [(U[0], "Healthy"), (U[1], "Unhealthy")]
        assert health(sa) == [(U[0], "Healthy"), (U[1], "Healthy")]
        got = [health(sb), health(sb)]
        assert got[-1] == [(U[2], "Healthy"), (U[3], "Unhealthy")]
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


def test_vgpu_health_feed_numpy_reference():
    run_scenario(health_mdev_ref.HealthMdevRef().rescan)


@pytest.mark.gpu
def test_vgpu_health_feed_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        run_scenario(ctx.health_rescan_mdev)
