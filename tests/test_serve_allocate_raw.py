"""The passthrough plugin with serve.AllocateRawCheck and serve.discover_egm_raw (every Allocate decision of an
AllocateRequest from the raw reads, in one call), against the same plugin with serve.AllocateCheck and
serve.discover_egm_devices on the same sysfs tree: equal serialised AllocateResponses, error texts and ReferencePanics
on every Allocate case of the reference's vectors and on the cases of test_serve_allocate_check.py.  On trees whose
gpu_devices hold \\x1c, "İ" or an invalid byte the raw plugin follows the Go rules restated in
tests/allocate_raw_cases.py, and the test records where AllocateCheck's Python decoding differs.

The CPU leg gives AllocateRawCheck the restatement and AllocateCheck the contract of tests/allocate_check_cases.py; the
gpu leg gives them Context.pci_allocate_raw and Context.pci_allocate_check on an H100.  The last test replays Register
-> Allocate over gRPC on the config-1 tree with the raw plugin on the real context."""
import json
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import allocate_check_cases as AC
import allocate_raw_cases as AR
import test_serve as TS
import util
import kvgpu
from kvgpu import dpapi, serve


@pytest.fixture(scope="module", params=["cpu", pytest.param("gpu", marks=pytest.mark.gpu)])
def leg(request):
    """(allocate_raw call, allocate_check call) of the leg"""
    if request.param == "cpu":
        yield AR.contract, AC.contract
        return
    ctx = kvgpu.Context(0)
    yield ctx.pci_allocate_raw, ctx.pci_allocate_check
    ctx.close()


class Calls:
    def __init__(self, fn):
        self.fn, self.n = fn, 0

    def __call__(self, *a):
        self.n += 1
        return self.fn(*a)


def tree(root, links, vendors, egm=(), panic=()):
    """bus/<addr>/iommu_group -> ../../kernel/iommu_groups/<group> and bus/<addr>/vendor = "0x<vendor>\\n" (a read
    that fails: no entry; a panic: one byte); sys/class/egm/<name>/gpu_devices and dev/<name> per (dev path, gpu
    devices bytes or list, node present)"""
    base = os.path.join(root, "bus")
    for addr in set(links) | set(vendors) | set(panic):
        os.makedirs(os.path.join(base, addr), exist_ok=True)
    for addr, g in links.items():
        if g is not None:
            os.symlink("../../kernel/iommu_groups/" + g, os.path.join(base, addr, "iommu_group"))
    for addr, v in vendors.items():
        if v is not None and addr not in panic:
            with open(os.path.join(base, addr, "vendor"), "w") as f:
                f.write("0x%s\n" % v)
    for addr in panic:
        with open(os.path.join(base, addr, "vendor"), "w") as f:
            f.write("x")
    for item in egm:
        path, gpus = item[0], item[1]
        node = item[2] if len(item) > 2 else True
        name = os.path.basename(path)
        d = os.path.join(root, "sys", "class", "egm", name)
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "gpu_devices"), "wb") as f:
            f.write(gpus if isinstance(gpus, bytes) else ("\n".join(gpus) + "\n").encode())
        if node:
            os.makedirs(os.path.join(root, "dev"), exist_ok=True)
            open(os.path.join(root, "dev", name), "w").close()
    os.makedirs(base, exist_ok=True)
    return base


def outcome(plugin, *requests):
    try:
        return "response", TS.allocate(plugin, *requests).SerializeToString()
    except serve.AllocateError as e:
        return "error", str(e)
    except kvgpu.ReferencePanic as e:
        return "panic", str(e)


def same(plugin, leg, *requests, raising=False):
    """Allocate through AllocateCheck and discover_egm_devices, then through AllocateRawCheck and discover_egm_raw:
    equal outcomes, and the raw check made one call"""
    raw_call, check_call = leg
    root = plugin.root_path

    def fail():
        raise RuntimeError("egm discovery failed")
    plugin.allocate_check = serve.AllocateCheck(check_call, plugin.base_path)
    plugin.discover_egm = fail if raising else (lambda: serve.discover_egm_devices(root))
    want = outcome(plugin, *requests)
    calls = Calls(raw_call)
    plugin.allocate_check = serve.AllocateRawCheck(calls, plugin.base_path)
    plugin.discover_egm = fail if raising else (lambda: serve.discover_egm_raw(root))
    got = outcome(plugin, *requests)
    assert got == want, requests
    assert calls.n == 1, requests
    return got


def make_plugin(root, maps, devs=(), name="n"):
    m = kvgpu.Maps()
    m.iommuMap = {g: [kvgpu.NvidiaGpuDevice(x, 0) for x in d] for g, d in maps.items()}
    m.bdfToIommuMap = {x: g for g, d in maps.items() for x in d}
    return serve.GenericDevicePlugin(name, "/", list(devs), m, base_path=os.path.join(root, "bus"), root_path=root)


def test_reference_vectors(leg, tmp_path):
    a = json.load(open(os.path.join(TS.HERE, "golden", "plugin_vectors.json")))["allocate"]
    kinds = []
    for k, case in enumerate(a["cases"]):
        root = str(tmp_path / ("case%d" % k))
        egm = case["egm"]
        entries = [(e["dev_path"], e["gpus"]) for e in a[egm]] if egm and egm != "error" else []
        tree(root, a["read_link"], a["read_vendor_" + case["vendor"]], entries)
        p = TS.plugin_for_case(a, case, root)
        p.revalidate = None
        if case.get("iommufd"):
            os.makedirs(os.path.join(root, "bus", case["request"][0], "vfio-dev", case["iommufd"]), exist_ok=True)
        kinds.append(same(p, leg, case["request"], raising=egm == "error")[0])
    assert kinds.count("response") == 6 and kinds.count("error") == 3


A, A1, B, C, D = "0000:0a:00.0", "0000:0a:00.1", "0000:0b:00.0", "0000:0c:00.0", "0000:0D:00.0"
MAPS = {"7": [A, A1], "8": [B], "9": [C], "10": [D]}
LINKS = {x: g for g, d in MAPS.items() for x in d}


def own(root, links=None, vendors=None, panic=(), egm=()):
    tree(root, dict(LINKS, **(links or {})), dict({x: "10de" for x in LINKS}, **(vendors or {})), egm, panic)
    return make_plugin(root, MAPS)


def test_own_cases(leg, tmp_path):
    egm = [("/dev/egm4", (" 0000:0A:00.0", "0000:0B:00.0\t")), ("/dev/egm5", ("0000:0d:00.0",)),
           ("/dev/egm6", ("0000:0c:00.0 ", "0000:0C:00.0")), ("/dev/egm2", ("0000:0a:00.1",)),
           ("/dev/egm7", ("0000:0c:00.0",), False), ("/dev/gpu1", ("0000:0c:00.0",))]
    p = own(str(tmp_path / "a"), egm=egm)
    for reqs in (([A, B],), ([A],), ([D],), ([C],), ([D, C, B, A],), ([A1],), ([A], [B]), ([A, B], [C], [D]),
                 ([A], [], [B]), ([A, B], ["nope"])):
        same(p, leg, *reqs)
    p = own(str(tmp_path / "b"), egm=egm[:2], links={C: "8"}, vendors={D: "8086"})
    for reqs in (([A], [B], [C]), ([A, B], [D, A]), ([D], [C])):
        assert same(p, leg, *reqs)[0] == "error"
    p = own(str(tmp_path / "c"), panic={B}, links={C: "7"}, vendors={D: None})
    assert same(p, leg, [B])[0] == "panic" and same(p, leg, [A], [B])[0] == "panic"
    for first in ([C], [D], ["nope"], [A, C]):
        assert same(p, leg, first, [B])[0] == "error"
    p = own(str(tmp_path / "d"), panic={A1}, links={A1: "8"})
    assert same(p, leg, [A]) == ("error", "invalid allocation request: unknown device: %s" % A1)
    p = own(str(tmp_path / "e"), links={A: None, B: "08"})
    assert same(p, leg, [A])[0] == "error" and same(p, leg, [B])[0] == "error"


# gpu_devices whose Python decoding (str.split after a "replace" decode, str.strip().lower()) differs from Go's
GO_ONLY = [("x1c", b"0000:0a:00.0\x1c0000:0b:00.0\n", [[A, B], ["0000:0a:00.0\x1c0000:0b:00.0"]]),
           ("dotted_i", "İd\n".encode(), [["id"], ["İd"], ["i̇d"]]),
           ("invalid", b"\xe2\x82x\n", [["�x"], ["��x"]])]


@pytest.mark.parametrize("name,gpus,id_sets", GO_ONLY, ids=[g[0] for g in GO_ONLY])
def test_go_decoding_where_python_differs(leg, tmp_path, name, gpus, id_sets):
    root = str(tmp_path)
    tree(root, LINKS, {x: "10de" for x in LINKS}, [("/dev/egm1", gpus)])
    base = os.path.join(root, "bus")
    raw_call, check_call = leg
    differs = []
    for ids in id_sets:
        got = serve.AllocateRawCheck(raw_call, base)([([(A, "7")], ids)], serve.discover_egm_raw(root))
        want_take = AR.allocate_raw([([(b"../7", b"0x10de\n", b"7")], [i.encode() for i in ids])],
                                    [(b"egm1", gpus, True)])[3][0, 0]
        assert got[0][2] == (["/dev/egm1"] if want_take else [])
        old = serve.AllocateCheck(check_call, base)([([(A, "7")], ids)], serve.discover_egm_devices(root))
        differs.append(old[0][2] != got[0][2])
    # where AllocateCheck's host decoding differs from the reference (DESIGN §4.11.2)
    assert differs == {"x1c": [True, True], "dotted_i": [True, False, True], "invalid": [True, True]}[name]


@pytest.mark.gpu
def test_scan_to_kubelet_round_trip_with_allocate_raw(tmp_path):
    import grpc
    ids = tmp_path / "pci.ids"
    ids.write_bytes(util.pciids_text())
    base = util.make_pci_tree(str(tmp_path / "pci"), util.c1_tree_entries())
    ds = kvgpu.DiscoveryScan(str(ids), base, str(tmp_path / "nomdev"))
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")
    root = str(tmp_path / "root")
    tree(root, {}, {}, [("/dev/egm0", ["0000:84:00.0", " 0000:87:00.0"]), ("/dev/egm1", ["0000:04:00.0"])])
    kubelet = serve.MockKubelet(sockdir).start()
    plugins = []
    try:
        maps = ds.create_iommu_device_map()
        calls = Calls(ds.ctx.pci_allocate_raw)
        plugins = serve.plugins_from_specs(ds.create_device_plugins(), maps, None,
                                           allocate_check=serve.AllocateRawCheck(calls, base), socket_dir=sockdir,
                                           base_path=base, root_path=root,
                                           discover_egm=lambda: serve.discover_egm_raw(root))
        ref = {p.device_name: p for p in serve.plugins_from_specs(
            ds.create_device_plugins(), maps, None, allocate_check=serve.AllocateCheck(ds.ctx.pci_allocate_check, base),
            socket_dir=sockdir, base_path=base, root_path=root)}["GP102GL_TESLA_P40"]
        for p in plugins:
            p.start()
        regs = kubelet.wait_for(len(plugins))
        c = kubelet.connect(next(r for r in regs if r.resource_name == "nvidia.com/GP102GL_TESLA_P40"))

        def both(*reqs):
            want = outcome(ref, *reqs)
            try:
                got = ("response", c.allocate(*reqs).SerializeToString())
            except grpc.RpcError as e:
                got = ("error", e.details())
            assert got == want, reqs
            return got
        r = dpapi.AllocateResponse.FromString(both(["0000:04:00.0"])[1]).container_responses[0]
        assert [d.host_path for d in r.devices] == ["/dev/vfio/vfio", "/dev/vfio/40", "/dev/egm1"]
        r = dpapi.AllocateResponse.FromString(both(["0000:84:00.0", "0000:87:00.0"])[1]).container_responses[0]
        assert [d.host_path for d in r.devices][-1] == "/dev/egm0"
        both(["0000:84:00.0"], ["0000:87:00.0"])
        assert calls.n == 3
        c.close()
    finally:
        for p in plugins:
            p.stop()
        kubelet.stop()
        ds.close()
        shutil.rmtree(sockdir, ignore_errors=True)
