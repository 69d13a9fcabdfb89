"""The passthrough plugin's GetPreferredAllocation with serve.NumaPacker, against the same plugin without it (the
reference rule serve.preferred_allocation): equal serialised PreferredAllocationResponses, or equal error texts, on every
call of tests/preferred_cases.py, with one packing call per PreferredAllocationRequest.

The CPU leg gives NumaPacker the C-ABI contract restated in Python; the gpu leg gives it Context.preferred_allocation on
an H100.  Both legs also run over gRPC against the mock kubelet: the CPU leg on the config-1 maps of tests/test_serve.py,
the gpu leg on the config-1 sysfs tree scanned by the real context."""
import shutil
import tempfile

import grpc
import pytest

import conftest  # noqa: F401
import preferred_cases as PC
import test_serve as TS
import util
import kvgpu
from kvgpu import dpapi, serve


@pytest.fixture(scope="module", params=["cpu", pytest.param("gpu", marks=pytest.mark.gpu)])
def leg(request):
    """The preferred_allocation call of the leg."""
    if request.param == "cpu":
        yield PC.contract
        return
    ctx = kvgpu.Context(0)
    yield ctx.preferred_allocation
    ctx.close()


def devices(devs):
    """[(id, node or None)] -> the plugin's []*pluginapi.Device (None: no topology)."""
    return [dpapi.Device(ID=i, health=dpapi.HEALTHY,
                         topology=dpapi.TopologyInfo(nodes=[] if n is None else [dpapi.NUMANode(ID=n)]))
            for i, n in devs]


def request_of(requests):
    return dpapi.PreferredAllocationRequest(container_requests=[dpapi.ContainerPreferredAllocationRequest(
        available_deviceIDs=list(a), must_include_deviceIDs=list(m), allocation_size=s) for a, m, s in requests])


def outcome(plugin, requests):
    try:
        return "response", plugin.GetPreferredAllocation(request_of(requests), None).SerializeToString()
    except serve.AllocateError as e:
        return "error", str(e)


def same(leg, devs, requests):
    """The plugin with NumaPacker answers as the plugin without it, in one packing call."""
    rec = PC.Recorder(leg)
    with_packer = serve.GenericDevicePlugin("n", "/", devices(devs), kvgpu.Maps(), prefer=serve.NumaPacker(rec))
    plain = serve.GenericDevicePlugin("n", "/", devices(devs), kvgpu.Maps())
    got, want = outcome(with_packer, requests), outcome(plain, requests)
    assert got == want, (devs, requests)
    assert len(rec.calls) == 1
    return got


def test_golden_vectors_and_edges(leg):
    for devs, requests in PC.golden_calls():
        same(leg, devs, requests)


@pytest.mark.parametrize("name", sorted(PC.named_calls()))
def test_named_quirks(leg, name):
    devs, requests = PC.named_calls()[name]
    kind, body = same(leg, devs, requests)
    if "error" in name or "negative size" in name or name == "size 0 with a must-include ID":
        assert kind == "error" and body.startswith("number of MustIncludeDeviceIDs (")


def test_seeded_calls(leg):
    import numpy as np
    rng = np.random.default_rng(3)
    for _ in range(200):
        same(leg, *PC.random_call(rng, int(rng.integers(1, 9)), int(rng.integers(1, 40))))


def test_no_container_requests(leg):
    assert same(leg, PC.DEVS, []) == ("response", b"")


def test_marshalling():
    """What NumaPacker hands the kernel: handles per request in first-seen order over must-include then available;
    nodes as dense indices per request, with -1, no topology and unknown IDs as PREF_NODE_NONE; -2 an ordinary node;
    the last entry with topology wins for a duplicate device."""
    rec = PC.Recorder()
    devs = [("a", 5), ("b", -2), ("c", -1), ("d", None), ("a", None), ("e", 0), ("e", 5)]
    serve.NumaPacker(rec)(devs, [(["b", "a", "c", "d", "u", "e", "b"], ["e", "a"], 3), ([], [], 0)])
    ids, n_must, n_avail, sizes, _ = rec.calls[0]
    none = kvgpu._lib.PREF_NODE_NONE
    assert (n_must, n_avail, sizes) == ([2, 0], [7, 0], [3, 0])
    assert ids["handle"].tolist() == [0, 1, 2, 1, 3, 4, 5, 0, 2]
    assert ids["node"].tolist() == [0, 0, 1, 0, none, none, none, 0, 1]


def test_first_failing_request_is_reported():
    with pytest.raises(serve.AllocateError) as e:
        serve.NumaPacker(PC.contract)(PC.DEVS, [(["a"], [], 1), (["a"], ["a", "b", "c"], 2), (["a"], ["a", "b"], 1)])
    assert str(e.value) == "number of MustIncludeDeviceIDs (3) exceeds allocation size (2)"


def test_plugins_from_specs_passes_prefer_to_passthrough_plugins():
    maps = TS.c1_maps()
    rec = PC.Recorder()
    plugins = serve.plugins_from_specs(kvgpu.plugin_specs_from_maps(maps), maps, None, prefer=serve.NumaPacker(rec))
    assert [type(p).__name__ for p in plugins] == ["GenericDevicePlugin", "GenericDevicePlugin",
                                                    "GenericVGpuDevicePlugin"]
    assert all(p.prefer is not None for p in plugins[:2]) and not hasattr(plugins[2], "prefer")
    assert serve.plugins_from_specs(kvgpu.plugin_specs_from_maps(maps), maps, None)[0].prefer is None


# ---- over gRPC against the mock kubelet ---------------------------------------------------------
P40 = "nvidia.com/GP102GL_TESLA_P40"
GRPC_REQUESTS = [
    ([["0000:04:00.0", "0000:05:00.0", "0000:84:00.0", "0000:85:00.0", "0000:86:00.0"], ["0000:86:00.0"], 3]),
    ([["0000:84:00.0", "0000:04:00.0", "0000:05:00.0", "0000:06:00.0"], [], 3]),
    ([["0000:04:00.0", "0000:84:00.0"], [], 2]),
    ([["0000:04:00.0", "0000:84:00.0", "0000:04:00.0"], ["0000:ff:00.0"], 2]),
    ([["0000:04:00.0"], [], 0]),
]


def _serve_and_compare(maps, specs, prefer, ref, **kw):
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")      # unix socket paths are limited to 107 bytes
    kubelet = serve.MockKubelet(sockdir).start()
    plugins = serve.plugins_from_specs(specs, maps, None, prefer=prefer, socket_dir=sockdir, root_path=sockdir,
                                       discover_egm=lambda: [], vgpu_base_path=sockdir, **kw)
    try:
        for p in plugins:
            p.start()
        regs = kubelet.wait_for(len(plugins))
        c = kubelet.connect(next(r for r in regs if r.resource_name == P40))
        assert c.options().get_preferred_allocation_available is True
        for available, must, size in GRPC_REQUESTS:
            want = outcome(ref, [(available, must, size)])
            try:
                r = c.preferred_allocation(available, must, size)
                got = ("response", r.SerializeToString())
            except grpc.RpcError as e:
                assert e.code() == grpc.StatusCode.UNKNOWN
                got = ("error", e.details())
            assert got == want, (available, must, size)
        # several container requests in one RPC, over the client's channel
        req = request_of([(a, m, s) for a, m, s in GRPC_REQUESTS[:3]])
        r = c._calls["GetPreferredAllocation"](req, timeout=serve.CONNECTION_TIMEOUT)
        assert r.SerializeToString() == ref.GetPreferredAllocation(req, None).SerializeToString()
        c.close()
    finally:
        for p in plugins:
            p.stop()
        kubelet.stop()
        shutil.rmtree(sockdir, ignore_errors=True)


def test_grpc_round_trip_on_config_1_maps():
    maps = TS.c1_maps()
    specs = kvgpu.plugin_specs_from_maps(maps)
    ref = serve.plugins_from_specs(specs, maps, None)[0]
    rec = PC.Recorder()
    _serve_and_compare(maps, specs, serve.NumaPacker(rec), ref)
    assert len(rec.calls) == len(GRPC_REQUESTS) + 1              # one packing call per RPC


@pytest.mark.gpu
def test_grpc_round_trip_on_the_config_1_tree(tmp_path):
    ids = tmp_path / "pci.ids"
    ids.write_bytes(util.pciids_text())
    base = util.make_pci_tree(str(tmp_path / "pci"), util.c1_tree_entries())
    ds = kvgpu.DiscoveryScan(str(ids), base, str(tmp_path / "nomdev"))
    try:
        maps = ds.create_iommu_device_map()
        specs = ds.create_device_plugins()
        ref = next(p for p in serve.plugins_from_specs(specs, maps, None) if p.device_name == "GP102GL_TESLA_P40")
        rec = PC.Recorder(ds.ctx.preferred_allocation)
        before = ds.ctx.launch_count
        _serve_and_compare(maps, specs, serve.NumaPacker(rec), ref, base_path=base)
        assert len(rec.calls) == len(GRPC_REQUESTS) + 1
        assert ds.ctx.launch_count - before == len(GRPC_REQUESTS) + 1    # one launch per RPC
        for call_ids, n_must, n_avail, sizes, raw in rec.calls:
            assert [(n, p, pos.tolist()) for n, p, pos in raw] == [
                (n, p, pos.tolist()) for n, p, pos in PC.contract(call_ids, n_must, n_avail, sizes)]
    finally:
        ds.close()
