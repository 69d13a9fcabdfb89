"""The passthrough plugin with serve.AllocateResponder (the whole AllocateResponse in one call after the plan) against
the same plugin with serve.AllocateRawCheck and the host replay of GenericDevicePlugin.Allocate, both with
discover_egm_raw, on real sysfs trees with vfio-dev directories and /dev/iommu: equal serialised AllocateResponses,
error texts and ReferencePanics on the reference's vectors and on the cases of test_serve_allocate_raw.py, with iommufd
off and on.  On trees where the host replay differs from Go (a vfio-dev entry that is a link to a directory, names
that are not UTF-8) the responder follows the restatement of tests/allocate_response_cases.py, and the test records
where the replay differs.

The CPU leg gives the responder the restatement and AllocateRawCheck allocate_raw_cases' contract; the gpu leg gives
them Context.pci_allocate_response and Context.pci_allocate_raw on an H100.  The last test replays Register ->
Allocate over gRPC with the responder on the real context."""
import json
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import allocate_raw_cases as AR
import allocate_response_cases as RC
import test_serve as TS
import test_serve_allocate_raw as SR
import util
import kvgpu
from kvgpu import dpapi, serve


def restated(raw, resp):
    """allocate_response_cases.allocate_response on a packed call, as Context.pci_allocate_response returns it"""
    requests, egm = AR.unpack(raw)
    out, m, v = [], 0, 0
    for r, (members, ids) in enumerate(requests):
        visits, e = [], 0
        for _ in range(int(resp.n_visited[r])):
            visit = []
            for _ in range(int(resp.id_members[v])):
                st = int(resp.vfio_state[m])
                first, last = int(resp.vfio_first[m]), int(resp.vfio_first[m + 1])
                listing = (kvgpu.NOT_READ if not st & 1 else None if st & 2 else
                           [(resp.vfio_bytes[resp.vfio_off[k]:resp.vfio_off[k + 1]], bool(resp.vfio_dir[k]))
                            for k in range(first, last)])
                addr = resp.addr_bytes[resp.addr_off[m]:resp.addr_off[m + 1]]
                visit.append((addr,) + members[e] + (listing,))
                m, e = m + 1, e + 1
            visits.append(visit)
            v += 1
        out.append((ids, visits, bool(resp.lookup_error[r])))
    return RC.allocate_response(out, egm, bool(resp.iommufd))


@pytest.fixture(scope="module", params=["cpu", pytest.param("gpu", marks=pytest.mark.gpu)])
def leg(request):
    """(allocate_response call, allocate_raw call) of the leg"""
    if request.param == "cpu":
        yield restated, AR.contract
        return
    ctx = kvgpu.Context(0)
    yield ctx.pci_allocate_response, ctx.pci_allocate_raw
    ctx.close()


def same(plugin, leg, *requests):
    """Allocate through the replay with AllocateRawCheck, then through AllocateResponder: equal outcomes, one call"""
    resp_call, raw_call = leg
    root = plugin.root_path
    plugin.discover_egm = lambda: serve.discover_egm_raw(root)
    plugin.allocate_check = serve.AllocateRawCheck(raw_call, plugin.base_path)
    want = SR.outcome(plugin, *requests)
    calls = SR.Calls(resp_call)
    plugin.allocate_response = serve.AllocateResponder(calls, plugin.base_path)
    got = SR.outcome(plugin, *requests)
    plugin.allocate_response = None
    assert got == want, requests
    assert calls.n == 1, requests
    return got


def vfio_dev(root, addr, *names, link=()):
    d = os.path.join(root, "bus", addr, "vfio-dev")
    os.makedirs(d, exist_ok=True)
    for n in names:
        os.makedirs(os.path.join(d, n), exist_ok=True)
    for n, target in link:
        os.symlink(target, os.path.join(d, n))


def iommu(root):
    os.makedirs(os.path.join(root, "dev"), exist_ok=True)
    open(os.path.join(root, "dev", "iommu"), "w").close()


def test_reference_vectors(leg, tmp_path):
    a = json.load(open(os.path.join(TS.HERE, "golden", "plugin_vectors.json")))["allocate"]
    kinds = []
    for k, case in enumerate(a["cases"]):
        if case["egm"] == "error":
            continue
        root = str(tmp_path / ("case%d" % k))
        entries = [(e["dev_path"], e["gpus"]) for e in a[case["egm"]]] if case["egm"] else []
        SR.tree(root, a["read_link"], a["read_vendor_" + case["vendor"]], entries)
        p = TS.plugin_for_case(a, case, root)
        p.revalidate = None
        kinds.append(same(p, leg, case["request"])[0])
    assert "response" in kinds and "error" in kinds


@pytest.mark.parametrize("iommufd", [False, True])
def test_own_cases(leg, tmp_path, iommufd):
    def own(name, **kw):
        root = str(tmp_path / name)
        p = SR.own(root, **kw)
        if iommufd:
            iommu(root)
            for x in SR.LINKS:
                vfio_dev(root, x, "vfio%d" % (len(x) + ord(x[-4])))
        return p
    egm = [("/dev/egm4", (" 0000:0A:00.0", "0000:0B:00.0\t")), ("/dev/egm5", ("0000:0d:00.0",)),
           ("/dev/egm6", ("0000:0c:00.0 ", "0000:0C:00.0")), ("/dev/egm2", ("0000:0a:00.1",)),
           ("/dev/egm7", ("0000:0c:00.0",), False), ("/dev/gpu1", ("0000:0c:00.0",))]
    A, A1, B, C, D = SR.A, SR.A1, SR.B, SR.C, SR.D
    p = own("a", egm=egm)
    for reqs in (([A, B],), ([A],), ([D],), ([C],), ([D, C, B, A],), ([A1],), ([A], [B]), ([A, B], [C], [D]),
                 ([A], [], [B]), ([A, B], ["nope"]), ([A, A],), ([A, A1],), ([], [A])):
        same(p, leg, *reqs)
    p = own("b", egm=egm[:2], links={C: "8"}, vendors={D: "8086"})
    for reqs in (([A], [B], [C]), ([A, B], [D, A]), ([D], [C])):
        assert same(p, leg, *reqs)[0] == "error"
    p = own("c", panic={B}, links={C: "7"}, vendors={D: None})
    assert same(p, leg, [B])[0] == "panic" and same(p, leg, [A], [B])[0] == "panic"
    for first in ([C], [D], ["nope"], [A, C]):
        assert same(p, leg, first, [B])[0] == "error"
    if iommufd:   # listing errors: a missing vfio-dev, an empty one, a file named vfio*
        p = own("d")
        shutil.rmtree(os.path.join(str(tmp_path / "d"), "bus", A1, "vfio-dev"))
        assert same(p, leg, [A])[1].startswith("could not determine iommufd device for device %s: [Errno" % A1)
        shutil.rmtree(os.path.join(str(tmp_path / "d"), "bus", B, "vfio-dev"))
        os.makedirs(os.path.join(str(tmp_path / "d"), "bus", B, "vfio-dev"))
        open(os.path.join(str(tmp_path / "d"), "bus", B, "vfio-dev", "vfio0"), "w").close()
        assert same(p, leg, [B])[1] == "could not determine iommufd device for device %s: no iommufd device found" % B


def test_where_the_host_replay_differs(leg, tmp_path):
    """a vfio-dev entry that links to a directory, and names that are not UTF-8: the responder follows Go"""
    resp_call, _ = leg
    root = str(tmp_path)
    p = SR.own(root)
    iommu(root)
    A, B = SR.A, SR.B
    vfio_dev(root, A, "vfio9", link=[("vfio1", "vfio9")])            # Go skips the link; isdir() follows it
    vfio_dev(root, SR.A1, "vfio2")
    # bytes order: b"vfio\xee\x80\x80" (U+E000) < b"vfio\xff"; str order: "vfio\udcff" < "vfio\ue000"
    vfio_dev(root, B, os.fsdecode(b"vfio\xff"), "vfio\ue000")
    p.discover_egm = lambda: serve.discover_egm_raw(root)
    p.allocate_response = serve.AllocateResponder(resp_call, p.base_path)
    got = [TS.allocate(p, [x]).container_responses[0].devices[0].host_path for x in (A, B)]
    assert got == ["/dev/vfio/devices/vfio9", "/dev/vfio/devices/vfio\ue000"]
    # where the host replay's reader differs: it follows the link, and it sorts str
    assert [serve.read_vfio_dev(p.base_path, x) for x in (A, B)] == ["vfio1", os.fsdecode(b"vfio\xff")]


@pytest.mark.gpu
def test_register_allocate_round_trip_with_the_responder(tmp_path):
    import grpc
    ids = tmp_path / "pci.ids"
    ids.write_bytes(util.pciids_text())
    base = util.make_pci_tree(str(tmp_path / "pci"), util.c1_tree_entries())
    ds = kvgpu.DiscoveryScan(str(ids), base, str(tmp_path / "nomdev"))
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")
    root = str(tmp_path / "root")
    SR.tree(root, {}, {}, [("/dev/egm1", ["0000:04:00.0"])])
    kubelet = serve.MockKubelet(sockdir).start()
    plugins = []
    try:
        maps = ds.create_iommu_device_map()
        calls = SR.Calls(ds.ctx.pci_allocate_response)
        kw = dict(socket_dir=sockdir, base_path=base, root_path=root, discover_egm=lambda: serve.discover_egm_raw(root))
        plugins = serve.plugins_from_specs(ds.create_device_plugins(), maps, None,
                                           allocate_response=serve.AllocateResponder(calls, base), **kw)
        ref = {p.device_name: p for p in serve.plugins_from_specs(
            ds.create_device_plugins(), maps, None, allocate_check=serve.AllocateRawCheck(ds.ctx.pci_allocate_raw, base),
            **kw)}["GP102GL_TESLA_P40"]
        for p in plugins:
            p.start()
        regs = kubelet.wait_for(len(plugins))
        c = kubelet.connect(next(r for r in regs if r.resource_name == "nvidia.com/GP102GL_TESLA_P40"))
        want = SR.outcome(ref, ["0000:04:00.0"])
        got = ("response", c.allocate(["0000:04:00.0"]).SerializeToString())
        assert got == want
        r = dpapi.AllocateResponse.FromString(got[1]).container_responses[0]
        assert [d.host_path for d in r.devices] == ["/dev/vfio/vfio", "/dev/vfio/40", "/dev/egm1"]
        with pytest.raises(grpc.RpcError) as e:
            c.allocate(["nope"])
        assert e.value.details() == SR.outcome(ref, ["nope"])[1]
        assert calls.n == 2
        c.close()
    finally:
        for p in plugins:
            p.stop()
        kubelet.stop()
        ds.close()
        shutil.rmtree(sockdir, ignore_errors=True)
