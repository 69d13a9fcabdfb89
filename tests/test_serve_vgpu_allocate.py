"""The vGPU plugin's Allocate with its label check on the GPU (serve.MdevLabelCheck over Context.mdev_label_match):
one check call per AllocateRequest, the files read in the reference's order, unreadable IDs never checked, and
AllocateResponses byte-identical to the plugin's CPU path (generic_vgpu_device_plugin.go:208-245), in process and over
real gRPC with MockKubelet, on the reference's Ginkgo fixture and on the getDeviceName quirk of vGPU labels."""
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import label_match_cases as LM
import util
from kvgpu import dpapi, serve

P = "0000:06:00.0"
TREE = {  # the tree of test_serve.py::test_vgpu_allocate_skips_foreign_types
    "u1": dict(type="GRID P100X-1B\n", parent=P),
    "u2": dict(type="GRID  P100X-1B", parent=P),       # same label after \s+ -> _
    "u3": dict(type="GRID P100X-2B\n", parent=P),      # another type: skipped
    "u4": dict(type=None, parent=P)}                   # unreadable: skipped
REQUESTS = [[["u1", "u2", "u3", "u4", "missing"]], [["u3"]],
            [["u1", "u3"], ["u4", "u2", "missing"], [], ["u2", "u1"]]]


def allocate(plugin, *requests):
    req = dpapi.AllocateRequest(container_requests=[dpapi.ContainerAllocateRequest(devices_ids=r) for r in requests])
    return plugin.Allocate(req, None)


class FakeMatch:
    """label_match on the CPU: the plugin's own rule on the raw bytes; records every call."""

    def __init__(self):
        self.calls = []

    def __call__(self, files, name):
        self.calls.append((list(files), name))
        return [LM.ref_label(f) == name.encode("latin-1") for f in files]


class CountingCheck(serve.MdevLabelCheck):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.n_calls = 0

    def __call__(self, device_name, ids):
        self.n_calls += 1
        return super().__call__(device_name, ids)


def test_one_check_per_request_in_reference_order(tmp_path):
    mdev, _ = util.make_mdev_tree(str(tmp_path), {P: "0\n"}, TREE)
    raw = {u: e["type"].encode() for u, e in TREE.items() if e["type"] is not None}
    cpu = serve.GenericVGpuDevicePlugin("GRID_P100X-1B", "vgpu", [], vgpu_base_path=mdev)
    for reqs in REQUESTS:
        fake = FakeMatch()
        check = CountingCheck(fake, mdev)
        gpu = serve.GenericVGpuDevicePlugin("GRID_P100X-1B", "vgpu", [], vgpu_base_path=mdev, check=check)
        got = allocate(gpu, *reqs)
        assert got.SerializeToString() == allocate(cpu, *reqs).SerializeToString(), reqs
        assert check.n_calls == 1
        ids = [i for r in reqs for i in r]
        readable = [i for i in ids if i in raw]                 # u4 and "missing" fail to read: never checked
        assert fake.calls == [([raw[i] for i in readable], "GRID_P100X-1B")]
    r = allocate(gpu, *REQUESTS[0]).container_responses[0]
    assert dict(r.envs) == {"MDEV_PCI_RESOURCE_NVIDIA_COM_GRID_P100X-1B": "u1,u2"}


def test_check_without_readable_ids_makes_no_match_call(tmp_path):
    mdev, _ = util.make_mdev_tree(str(tmp_path), {P: "0\n"}, TREE)
    fake = FakeMatch()
    check = serve.MdevLabelCheck(fake, mdev)
    assert check("GRID_P100X-1B", ["u4", "missing"]) == [False, False]
    assert check("GRID_P100X-1B", []) == []
    assert fake.calls == []


# ---- on the GPU, over gRPC ----------------------------------------------------------------------
@pytest.fixture()
def grpc_world():
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")     # unix socket paths are limited to 107 bytes
    kubelet = serve.MockKubelet(sockdir).start()
    started = []

    def serve_plugins(plugins):
        for p in plugins:
            p.start()
            started.append(p)
        regs = kubelet.wait_for(len(started))
        return [kubelet.connect(next(r for r in regs if r.endpoint == os.path.basename(p.socket_path)))
                for p in plugins]
    yield sockdir, kubelet, serve_plugins
    for p in started:
        p.stop()
    kubelet.stop()
    shutil.rmtree(sockdir, ignore_errors=True)


def _pair(name, mdev, sockdir, kubelet, check):
    """The plugin with the GPU check, served over gRPC, and its CPU-path twin, called in process."""
    gpu = serve.GenericVGpuDevicePlugin(name, "vgpu", [], check=check, vgpu_base_path=mdev, socket_dir=sockdir,
                                        kubelet_socket=kubelet.socket_path)
    return gpu, serve.GenericVGpuDevicePlugin(name, "vgpu", [], vgpu_base_path=mdev)


def _same_responses(client, cpu, reqs):
    a = client.allocate(*reqs)
    assert a.SerializeToString() == allocate(cpu, *reqs).SerializeToString(), reqs
    return a


@pytest.mark.gpu
def test_grpc_responses_equal_the_cpu_path(grpc_world):
    import kvgpu
    sockdir, kubelet, serve_plugins = grpc_world
    mdev, _ = util.make_mdev_tree(os.path.join(sockdir, "sys"), {P: "0\n"}, TREE)
    with kvgpu.Context(0) as ctx:
        gpu, cpu = _pair("GRID_P100X-1B", mdev, sockdir, kubelet, serve.MdevLabelCheck(ctx.mdev_label_match, mdev))
        cg, = serve_plugins([gpu])
        for reqs in REQUESTS:
            _same_responses(cg, cpu, reqs)
        r = cg.allocate(*REQUESTS[0]).container_responses[0]
        assert dict(r.envs) == {"MDEV_PCI_RESOURCE_NVIDIA_COM_GRID_P100X-1B": "u1,u2"}
        r = cg.allocate(*REQUESTS[2]).container_responses
        assert [dict(x.envs) for x in r] == [{"MDEV_PCI_RESOURCE_NVIDIA_COM_GRID_P100X-1B": x} for x in ("u1", "u2")] + [
            {}, {"MDEV_PCI_RESOURCE_NVIDIA_COM_GRID_P100X-1B": "u2,u1"}]


@pytest.mark.gpu
def test_grpc_ginkgo_fixture(grpc_world):
    """generic_vgpu_device_plugin_test.go:134-156: IDs "1" and "2" are vGPUs of type "vGPUId", "3" does not exist."""
    import kvgpu
    sockdir, kubelet, serve_plugins = grpc_world
    mdev, _ = util.make_mdev_tree(os.path.join(sockdir, "sys"), {P: "0\n"}, {
        "1": dict(type="vGPUId", parent=P), "2": dict(type="vGPUId\n", parent=P)})
    with kvgpu.Context(0) as ctx:
        gpu, cpu = _pair("vGPUId", mdev, sockdir, kubelet, serve.MdevLabelCheck(ctx.mdev_label_match, mdev))
        cg, = serve_plugins([gpu])
        r = _same_responses(cg, cpu, [["1"]]).container_responses[0]
        assert r.envs["MDEV_PCI_RESOURCE_NVIDIA_COM_VGPUID"] == "1"
        r = _same_responses(cg, cpu, [["3"]]).container_responses[0]
        assert dict(r.envs) == {}
        assert r.devices[0].host_path == "/dev/vfio"


@pytest.mark.gpu
def test_grpc_plugins_from_specs_and_the_getdevicename_quirk(grpc_world, tmp_path):
    """A vGPU label that is a pci.ids device-line prefix resolves through getDeviceName (device_plugin.go:152), so its
    plugin is named after the pci.ids name and the reference skips every ID at Allocate; a label that resolves to
    nothing names its plugin itself and keeps its IDs."""
    import kvgpu
    sockdir, kubelet, serve_plugins = grpc_world
    ids = tmp_path / "pci.ids"
    ids.write_bytes(util.pciids_text())
    ua, ub, uc = ("%08x-0000-4000-8000-%012x" % (k, k) for k in (1, 2, 3))
    mdev, pci = util.make_mdev_tree(os.path.join(sockdir, "sys"), {P: "0\n"}, {
        ua: dict(type="1b38\n", parent=P), ub: dict(type="GRID A100-4C\n", parent=P),
        uc: dict(type="GRID  A100-4C", parent=P)})
    ds = kvgpu.DiscoveryScan(str(ids), pci, mdev)
    try:
        ds.create_iommu_device_map()
        maps = ds.create_vgpu_id_map()
        specs = ds.create_device_plugins()
        assert sorted(s.device_name for s in specs) == ["GP102GL_TESLA_P40", "GRID_A100-4C"]
        kw = dict(socket_dir=sockdir, kubelet_socket=kubelet.socket_path, vgpu_base_path=mdev)
        check = CountingCheck(ds.ctx.mdev_label_match, mdev)
        gpu = serve.plugins_from_specs(specs, maps, None, vgpu_check=check, **kw)
        assert all(p.check is check for p in gpu)
        clients = dict(zip((p.device_name for p in gpu), serve_plugins(gpu)))
        cpu = serve.plugins_from_specs(specs, maps, None, **kw)
        assert all(p.check is None for p in cpu)
        for reqs in ([[ua, ub, uc]], [[ua], [uc, ub]]):
            want = {p.device_name: allocate(p, *reqs).SerializeToString() for p in cpu}
            for name, c in clients.items():
                assert c.allocate(*reqs).SerializeToString() == want[name], (name, reqs)
        r = clients["GP102GL_TESLA_P40"].allocate([ua, ub, uc]).container_responses[0]
        assert dict(r.envs) == {} and [d.host_path for d in r.devices] == ["/dev/vfio"]
        r = clients["GRID_A100-4C"].allocate([ua, ub, uc]).container_responses[0]
        assert dict(r.envs) == {"MDEV_PCI_RESOURCE_NVIDIA_COM_GRID_A100-4C": "%s,%s" % (ub, uc)}
        assert check.n_calls == 2 * 2 + 2
    finally:
        ds.close()
