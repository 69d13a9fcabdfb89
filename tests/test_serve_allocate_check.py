"""The passthrough plugin's Allocate with serve.AllocateCheck (every decision of an AllocateRequest in one call), against
the same plugin with serve.GroupCheck and the CPU EGM rule: equal serialised AllocateResponses, or equal error texts, or
equal ReferencePanics, with one call per AllocateRequest.  The cases: every Allocate case of the reference's vectors
(the shared, subset and multi-socket EGM cases and failed discovery among them), EGM strings with surrounding
whitespace and upper-case hex on either side, iommufd together with EGM, several container requests where a later one
fails, and an earlier request that fails while a later one would panic.

The CPU leg gives AllocateCheck the C-ABI contract restated in tests/allocate_check_cases.py and GroupCheck the rule
of tests/group_check_cases.py; the gpu leg gives them Context.pci_allocate_check and Context.pci_group_check on an
H100.  The last test replays Register -> ListAndWatch -> Allocate over gRPC on the config-1 tree with AllocateCheck on
the real context."""
import json
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import allocate_check_cases as AC
import group_check_cases as GC
import test_serve as TS
import util
import kvgpu
from kvgpu import dpapi, serve


def fake_group_check(recs, want):
    bad = GC.first_bad(recs, want)
    return None if bad == len(recs) else bad


class Calls:
    """Counts the calls of `fn` and keeps their request counts."""

    def __init__(self, fn):
        self.fn, self.n_reqs = fn, []

    def __call__(self, recs, want, n_members, *rest):
        self.n_reqs.append(len(n_members))
        return self.fn(recs, want, n_members, *rest)


@pytest.fixture(scope="module", params=["cpu", pytest.param("gpu", marks=pytest.mark.gpu)])
def leg(request):
    """(allocate_check, group_check) of the leg."""
    if request.param == "cpu":
        yield AC.contract, fake_group_check
        return
    ctx = kvgpu.Context(0)
    yield ctx.pci_allocate_check, ctx.pci_group_check
    ctx.close()


def outcome(plugin, *requests):
    try:
        return "response", TS.allocate(plugin, *requests).SerializeToString()
    except serve.AllocateError as e:
        return "error", str(e)
    except kvgpu.ReferencePanic as e:
        return "panic", str(e)


def same(plugin, leg, *requests):
    """Allocate through GroupCheck and the CPU EGM rule, then through AllocateCheck with the same readers: the outcomes
    are equal, and AllocateCheck made one call."""
    allocate_check, group_check = leg
    rv = plugin.revalidate
    plugin.revalidate = serve.GroupCheck(group_check, rv.base_path, rv.read_link, rv.read_id)
    want = outcome(plugin, *requests)
    calls = Calls(allocate_check)
    plugin.allocate_check = serve.AllocateCheck(calls, rv.base_path, rv.read_link, rv.read_id)
    got = outcome(plugin, *requests)
    plugin.revalidate, plugin.allocate_check = rv, None
    assert got == want, requests
    assert calls.n_reqs == [len(requests)], requests
    return got


def host_paths(got, k=0):
    return [d.host_path for d in dpapi.AllocateResponse.FromString(got[1]).container_responses[k].devices]


def test_reference_vectors(leg, tmp_path):
    a = json.load(open(os.path.join(TS.HERE, "golden", "plugin_vectors.json")))["allocate"]
    kinds = []
    for k, case in enumerate(a["cases"]):
        root = str(tmp_path / ("case%d" % k))
        os.makedirs(root)
        plugin = TS.plugin_for_case(a, case, root)
        got = same(plugin, leg, case["request"])
        kinds.append(got[0])
        if got[0] == "response":
            paths = host_paths(got)
            for p, n in case.get("want_host_path_count", {}).items():
                assert paths.count(p) == n, case["cite"]
            for p in case.get("want_absent", []):
                assert p not in paths, case["cite"]
            if "want_devices" in case:
                assert paths == case["want_devices"], case["cite"]
    assert kinds.count("response") == 6 and kinds.count("error") == 3


# ---- a plugin of its own: groups "7" = a and its audio function, "8" = b, "9" = c, "10" = D (upper-case hex) -------
A, A1, B, C, D = "0000:0a:00.0", "0000:0a:00.1", "0000:0b:00.0", "0000:0c:00.0", "0000:0D:00.0"
MAPS = {"7": [A, A1], "8": [B], "9": [C], "10": [D]}


def plugin(root, links=None, vendors=None, panic=(), egm=(), iommufd=None):
    m = kvgpu.Maps()
    m.iommuMap = {g: [kvgpu.NvidiaGpuDevice(x, 0) for x in devs] for g, devs in MAPS.items()}
    m.bdfToIommuMap = {x: g for g, devs in MAPS.items() for x in devs}
    all_links = {x: g for g, devs in MAPS.items() for x in devs}
    rl, ri = TS.dict_readers({k: v for k, v in dict(all_links, **(links or {})).items() if v is not None},
                             {k: v for k, v in dict({x: "10de" for x in all_links}, **(vendors or {})).items()
                              if v is not None})

    def read_id(base, addr, prop):
        if addr in panic:
            raise kvgpu.ReferencePanic("slice bounds out of range reading %s/%s" % (addr, prop))
        return ri(base, addr, prop)
    base = os.path.join(root, "bus")
    os.makedirs(base, exist_ok=True)
    if iommufd is not None:
        os.makedirs(os.path.join(root, "dev"), exist_ok=True)
        open(os.path.join(root, "dev", "iommu"), "w").close()
        for addr, vfio in iommufd.items():
            os.makedirs(os.path.join(base, addr, "vfio-dev", vfio))
    egm_devs = [serve.EGMDeviceInfo(p, list(g)) for p, g in egm]
    reval = serve.GroupCheck(fake_group_check, base, rl, read_id)
    return serve.GenericDevicePlugin("n", "/", [], m, revalidate=reval, base_path=base, root_path=root,
                                     discover_egm=lambda: egm_devs)


def test_egm_strings_are_normalised_on_both_sides(leg, tmp_path):
    # the EGM lists carry whitespace and upper-case hex; D's DevicesID is upper case itself
    egm = [("/dev/egm4", (" 0000:0A:00.0\n", "0000:0B:00.0\t")), ("/dev/egm5", ("0000:0d:00.0",)),
           ("/dev/egm6", ("0000:0c:00.0 ", "0000:0C:00.0")), ("/dev/egm2", ("0000:0a:00.1",))]
    p = plugin(str(tmp_path), egm=egm)
    assert "/dev/egm4" in host_paths(same(p, leg, [A, B]))
    assert "/dev/egm4" not in host_paths(same(p, leg, [A]))
    assert host_paths(same(p, leg, [D]))[-1:] == ["/dev/egm5"]
    assert host_paths(same(p, leg, [C]))[-1:] == ["/dev/egm6"]
    got = same(p, leg, [D, C, B, A])
    assert host_paths(got)[-3:] == ["/dev/egm4", "/dev/egm5", "/dev/egm6"]      # sorted; egm2 lists A1, not requested
    for reqs in ([A1], [A, A1], [C, D], [B, D, A]):
        same(p, leg, reqs)


def test_iommufd_with_egm(leg, tmp_path):
    egm = [("/dev/egm4", (A, B)), ("/dev/egm5", (C,))]
    p = plugin(str(tmp_path / "ok"), egm=egm, iommufd={A: "vfio3", A1: "vfio4", B: "vfio5", C: "vfio6"})
    got = same(p, leg, [A, B, C])
    assert host_paths(got)[-2:] == ["/dev/egm4", "/dev/egm5"] and "/dev/iommu" in host_paths(got)
    same(p, leg, [C], [A, B])
    p = plugin(str(tmp_path / "bad"), egm=egm, iommufd={A: "vfio3", B: "vfio5"})
    assert same(p, leg, [A, B])[0] == "error"                                # A1 has no vfio-dev directory
    assert same(p, leg, [B], [C]) == ("error", "could not determine iommufd device for device %s: "
                                      "[Errno 2] No such file or directory: '%s'"
                                      % (C, os.path.join(str(tmp_path / "bad"), "bus", C, "vfio-dev")))


def test_several_container_requests(leg, tmp_path):
    egm = [("/dev/egm4", (A, B)), ("/dev/egm5", (C,))]
    p = plugin(str(tmp_path / "ok"), egm=egm)
    for reqs in (([A], [B]), ([A, B], [C], [D]), ([C], [A, B]), ([A], [], [B]), ([A, B], [A, B])):
        got = same(p, leg, *reqs)
        assert got[0] == "response"
    r = dpapi.AllocateResponse.FromString(same(p, leg, [A, B], [C])[1]).container_responses
    assert r[1].envs["PCI_RESOURCE_NVIDIA_COM_N"] == ",".join([A, A1, B, C])  # env_list spans the requests (:361)
    assert [d.host_path for d in r[0].devices][-1] == "/dev/egm4" and [d.host_path for d in r[1].devices][-1] == \
        "/dev/egm5"
    # a later request fails: its lookup, a moved link, a changed vendor
    p = plugin(str(tmp_path / "bad"), egm=egm, links={C: "8"}, vendors={D: "8086"})
    assert same(p, leg, [A, B], ["nope"]) == ("error", "invalid allocation request: unknown device: nope")
    assert same(p, leg, [A], [B], [C]) == ("error", "invalid allocation request: unknown device: %s" % C)
    assert same(p, leg, [A, B], [D, A]) == ("error", "invalid allocation request: unknown device: %s" % D)
    assert same(p, leg, [D], [C])[1].endswith(D)                              # the first failing request wins


def test_an_earlier_failure_hides_a_later_panic(leg, tmp_path):
    p = plugin(str(tmp_path / "p"), panic={B}, links={C: "7"}, vendors={D: None})
    assert same(p, leg, [B])[0] == "panic"
    assert same(p, leg, [A], [B])[0] == "panic"
    for first in ([C], [D], ["nope"], [A, C]):
        got = same(p, leg, first, [B])
        assert got[0] == "error", first
    # the panicking member is behind a moved link in its own request: the link check fails first
    p = plugin(str(tmp_path / "q"), panic={A1}, links={A1: "8"})
    assert same(p, leg, [A]) == ("error", "invalid allocation request: unknown device: %s" % A1)


def test_a_panic_surfaces_where_the_reference_reads(tmp_path):
    """AllocateCheck raises a member's panic where the reference reads that vendor file.  An earlier member of the
    same request whose iommufd device cannot be read stops the reference first; GroupCheck, which raises before the
    request is replayed, surfaces the panic there instead."""
    p = plugin(str(tmp_path), panic={A1}, iommufd={A1: "vfio4"})      # A, read before A1, has no vfio-dev directory
    rv = p.revalidate
    p.allocate_check = serve.AllocateCheck(AC.contract, rv.base_path, rv.read_link, rv.read_id)
    kind, text = outcome(p, [A])
    assert kind == "error" and text.startswith("could not determine iommufd device for device %s: " % A)
    p.allocate_check = None
    assert outcome(p, [A])[0] == "panic"


def test_one_call_per_allocate_request(tmp_path):
    p = plugin(str(tmp_path), egm=[("/dev/egm4", (A, B))])
    rv = p.revalidate
    calls = Calls(AC.contract)
    p.allocate_check = serve.AllocateCheck(calls, rv.base_path, rv.read_link, rv.read_id)
    TS.allocate(p, [A], [B, A], [D])
    TS.allocate(p)
    with pytest.raises(serve.AllocateError):
        TS.allocate(p, ["nope"], [A])                     # a lookup error stops the first request; the call is made
    assert calls.n_reqs == [3, 0, 2]


def test_what_the_call_is_given(tmp_path):
    """The group handles of one table, the reads as GroupCheck records them, the EGM GPU strings interned first by
    egm_key, and DevicesIDs no device lists as n_egm_gpus."""
    seen = []

    def capture(*args):
        seen.append(args)
        return AC.contract(*args)
    p = plugin(str(tmp_path), links={B: None}, vendors={C: "10DE"})
    rv = p.revalidate
    check = serve.AllocateCheck(capture, rv.base_path, rv.read_link, rv.read_id)
    egm = [serve.EGMDeviceInfo("/dev/egm9", [" 0000:0B:00.0", "0000:0c:00.0"]),
           serve.EGMDeviceInfo("/dev/egm1", []), serve.EGMDeviceInfo("/dev/egm3", ["0000:0b:00.0 "])]
    out = check([([(A, "7"), (A1, "7")], [A]), ([(B, "8")], [B, "x", "0000:0B:00.0"]), ([(C, "9")], [C])], egm)
    recs, want, n_members, ids, n_ids, egm_off, egm_gpu, n_egm_gpus = seen[0]
    assert list(want) == [0, 0, 1, 2] and list(recs["iommu_group"]) == [0, 0, 0, 2]
    assert list(recs["flags"]) == [0, 0, kvgpu._lib.PF_IOMMU_ERR, 0] and list(recs["vendor"])[3] == 0xffff
    assert n_members == [2, 1, 1] and n_ids == [1, 3, 1]
    assert list(egm_off) == [0, 2, 2, 3] and list(egm_gpu) == [0, 1, 0] and n_egm_gpus == 2
    assert list(ids) == [2, 0, 2, 0, 1]
    assert out == [(None, None, ["/dev/egm1"]), (0, None, ["/dev/egm1", "/dev/egm3"]), (0, None, ["/dev/egm1"])]
    assert check([], None) == [] and len(seen) == 2
    assert list(seen[1][5]) == [] and seen[1][7] == 0


# ---- over gRPC on the config-1 tree, with the real context ---------------------------------------
@pytest.mark.gpu
def test_scan_to_kubelet_round_trip_with_allocate_check(tmp_path):
    import grpc
    ids = tmp_path / "pci.ids"
    ids.write_bytes(util.pciids_text())
    base = util.make_pci_tree(str(tmp_path / "pci"), util.c1_tree_entries())
    ds = kvgpu.DiscoveryScan(str(ids), base, str(tmp_path / "nomdev"))
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")
    kubelet = serve.MockKubelet(sockdir).start()
    plugins = []
    egm = [serve.EGMDeviceInfo("/dev/egm0", ["0000:84:00.0", " 0000:87:00.0"]),
           serve.EGMDeviceInfo("/dev/egm1", ["0000:04:00.0\n"])]
    try:
        maps = ds.create_iommu_device_map()
        calls = Calls(ds.ctx.pci_allocate_check)
        plugins = serve.plugins_from_specs(ds.create_device_plugins(), maps, None,
                                           allocate_check=serve.AllocateCheck(calls, base), socket_dir=sockdir,
                                           base_path=base, root_path=sockdir, discover_egm=lambda: egm)
        ref = serve.plugins_from_specs(ds.create_device_plugins(), maps, serve.GroupCheck(ds.ctx.pci_group_check, base),
                                       socket_dir=sockdir, base_path=base, root_path=sockdir, discover_egm=lambda: egm)
        ref = {p.device_name: p for p in ref}
        for p in plugins:
            p.start()
        regs = kubelet.wait_for(len(plugins))
        c = kubelet.connect(next(r for r in regs if r.resource_name == "nvidia.com/GP102GL_TESLA_P40"))
        ref = ref["GP102GL_TESLA_P40"]

        def both(*reqs):
            want = outcome(ref, *reqs)
            try:
                got = ("response", c.allocate(*reqs).SerializeToString())
            except grpc.RpcError as e:
                got = ("error", e.details())
            assert got == want, reqs
            return got

        r = dpapi.AllocateResponse.FromString(both(["0000:04:00.0"])[1]).container_responses[0]
        assert dict(r.envs) == {"PCI_RESOURCE_NVIDIA_COM_GP102GL_TESLA_P40": "0000:04:00.0,0000:04:00.1"}
        assert [d.host_path for d in r.devices] == ["/dev/vfio/vfio", "/dev/vfio/40", "/dev/egm1"]
        r = dpapi.AllocateResponse.FromString(both(["0000:84:00.0", "0000:87:00.0"])[1]).container_responses[0]
        assert [d.host_path for d in r.devices][-1] == "/dev/egm0"
        both(["0000:84:00.0"], ["0000:87:00.0"])
        real = os.path.realpath(os.path.join(base, "0000:05:00.0"))
        with open(os.path.join(real, "vendor"), "w") as f:
            f.write("0x8086\n")
        assert both(["0000:04:00.0"], ["0000:05:00.0"]) == (
            "error", "invalid allocation request: unknown device: 0000:05:00.0")
        assert calls.n_reqs == [1, 1, 2, 2]                        # one call per AllocateRequest
        c.close()
    finally:
        for p in plugins:
            p.stop()
        kubelet.stop()
        ds.close()
        shutil.rmtree(sockdir, ignore_errors=True)
