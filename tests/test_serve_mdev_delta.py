"""MdevRescanFeed over real gRPC with MockKubelet: an mdev tree under a temporary directory changes between ticks and
the set of vGPU plugins follows it.  A new mdev of a new type registers a plugin; removing one of two mdevs of a type
makes its plugin re-send the shorter list; removing the last one stops the plugin; a parent's changed numa_node
re-sends the topology; the gpuVgpuMap object shared with an XidEventRouter is patched in place.  The CPU variant
computes each scan and delta with the numpy restatements of tests/util.py and tests/mdev_delta_ref.py; the GPU
variant runs Context.scan_mdev_delta."""
import os
import shutil
import tempfile

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import mdev_delta_ref
import util
from kvgpu import _lib as L
from kvgpu import serve


def numpy_scan_delta():
    """scan_mdev_delta restated in numpy: the result (no names joined) and the delta against the previous call."""
    prev = [np.zeros(0, dtype=L.MDEV_SURV), []]

    def ordering(keys):
        order = np.argsort(keys, kind="stable")
        uk, first = np.unique(keys[order], return_index=True)
        return uk, np.append(first, len(keys)).astype(np.uint32), order.astype(np.uint32)

    def scan(recs, raw_types):
        e = util.expect_mdev(recs, raw_types)
        labels, canon = util.mdev_labels(raw_types)
        s = np.zeros(len(e["src"]), dtype=L.MDEV_SURV)
        for f in ("uuid", "parent", "type_key", "numa", "src"):
            s[f] = e[f]
        tk, toff, tperm = ordering(s["type_key"])
        pk, poff, pperm = ordering(s["parent"])
        res = kvgpu.MdevResult(len(recs), s, tk.astype(np.uint16), toff, tperm, labels, canon.astype(np.uint16),
                               [""] * len(labels), pk.astype(np.uint32), poff, pperm)
        d = mdev_delta_ref.expect_mdev_delta(prev[0], s, prev[1], labels, L.MDEV_CHANGE)
        delta = kvgpu.MdevDelta(len(prev[0]), d["changes"], d["type_dirty"], d["type_gone"], d["par_dirty"],
                                d["par_gone"])
        prev[0], prev[1] = s, labels
        return res, delta
    return scan


U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(1, 8)]     # canonical UUIDs, ascending


def run_scenario(scan_delta):
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")     # unix socket paths are limited to 107 bytes
    root = os.path.join(sockdir, "sys")
    vbase, pbase = util.make_mdev_tree(root, {"0000:3b:00.0": "0\n", "0000:86:00.0": "1\n"}, {
        U[0]: dict(type="GRID A100-1B\n", parent="0000:3b:00.0"),
        U[1]: dict(type="GRID  A100-1B", parent="0000:86:00.0"),      # the same label after \s+ -> _
        U[2]: dict(type="GRID A100-2Q\n", parent="0000:3b:00.0")})
    kubelet = serve.MockKubelet(sockdir).start()
    maps, plugins = kvgpu.Maps(), {}
    shared = maps.gpuVgpuMap                                 # what an XidEventRouter would hold

    def make_plugin(spec):
        return serve.GenericVGpuDevicePlugin(spec.device_name, "vgpu", serve.devices_from_spec(spec),
                                             vgpu_base_path=vbase, socket_dir=sockdir,
                                             kubelet_socket=kubelet.socket_path)
    feed = serve.MdevRescanFeed(scan_delta, lambda: kvgpu.snapshot_mdev_tree(vbase, pbase), maps, plugins,
                                make_plugin)
    router = serve.XidEventRouter([], maps.gpuVgpuMap, [])
    clients = []
    try:
        feed.tick()
        assert sorted(plugins) == ["GRID_A100-1B", "GRID_A100-2Q"] and len(kubelet.wait_for(2)) == 2
        assert maps.gpuVgpuMap is shared and shared["0000:3b:00.0"] == [U[0], U[2]]
        c = kubelet.connect(next(r for r in kubelet.registrations
                                 if r.endpoint == os.path.basename(plugins["GRID_A100-1B"].socket_path)))
        clients.append(c)
        stream = c.list_and_watch()
        assert [d.ID for d in next(stream).devices] == [U[0], U[1]]
        plugins["GRID_A100-1B"].unhealthy(U[1])
        assert [d.health for d in next(stream).devices] == ["Healthy", "Unhealthy"]

        # a new mdev of a new type on a new GPU: a new plugin registers, the shared map has the GPU
        util.make_mdev_tree(root, {"0000:af:00.0": "1\n"}, {U[3]: dict(type="GRID A100-4C\n", parent="0000:af:00.0")})
        t = feed.tick()
        assert t.type_dirty == ["GRID_A100-4C"] and t.type_gone == [] and t.par_dirty == ["0000:af:00.0"]
        assert "GRID_A100-4C" in plugins and len(kubelet.wait_for(3)) == 3
        assert shared["0000:af:00.0"] == [U[3]] and router.gpu_vgpu_map is shared

        # the parent of U[1] moves to NUMA node 0: its type re-sends the topology, its GPU key stays clean
        with open(os.path.join(pbase, "0000:86:00.0", "numa_node"), "w") as f:
            f.write("0\n")
        t = feed.tick()
        assert t.type_dirty == ["GRID_A100-1B"] and t.par_dirty == [] and t.par_gone == []
        got = next(stream).devices
        assert [(d.ID, d.health, d.topology.nodes[0].ID) for d in got] == [(U[0], "Healthy", 0), (U[1], "Unhealthy", 0)]

        # one of the two mdevs of GRID_A100-1B goes: the plugin re-sends the shorter list, its GPU goes too
        os.remove(os.path.join(vbase, U[1]))
        t = feed.tick()
        assert t.type_dirty == ["GRID_A100-1B"] and t.par_gone == ["0000:86:00.0"]
        assert [d.ID for d in next(stream).devices] == [U[0]]
        assert "0000:86:00.0" not in shared
        stream.cancel()

        # the last mdev of GRID_A100-2Q goes: its plugin stops
        p2q = plugins["GRID_A100-2Q"]
        os.remove(os.path.join(vbase, U[2]))
        t = feed.tick()
        assert t.type_gone == ["GRID_A100-2Q"] and "GRID_A100-2Q" not in plugins and p2q.server is None
        assert "GRID_A100-2Q" not in maps.vGpuMap and shared["0000:3b:00.0"] == [U[0]]
        snap = feed.snapshot()
        assert kvgpu.canonical_dump(maps) == kvgpu.canonical_dump(
            kvgpu.mdev_maps_from_result(feed.scan_delta(snap.recs, snap.raw_types)[0]))
    finally:
        for c in clients:
            c.close()
        for p in plugins.values():
            p.stop()
        kubelet.stop()
        shutil.rmtree(sockdir, ignore_errors=True)


def test_mdev_feed_follows_the_tree_numpy_reference():
    run_scenario(numpy_scan_delta())


@pytest.mark.gpu
def test_mdev_feed_follows_the_tree_on_the_gpu():
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(util.pciids_text())
        run_scenario(ctx.scan_mdev_delta)
