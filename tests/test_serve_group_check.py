"""The passthrough plugin's Allocate with serve.GroupCheck as its re-check, against the same plugin with
serve.BatchRevalidator: equal serialised AllocateResponses, or equal error texts, or equal ReferencePanics, on every
Allocate case of the reference's vectors and on the reads the re-check exists for (a group link that moved or cannot be
read, a vendor that changed or cannot be read, a short vendor file before and after an earlier rejection, "042"
against "42"), beside lookup errors, iommufd, EGM and several container requests.

The CPU leg gives GroupCheck the rule restated in numpy (tests/group_check_cases.py) and BatchRevalidator the numpy
scan of tests/test_serve.py; the gpu leg gives them Context.pci_group_check and Context.scan_pci on an H100.  The last
test replays Register -> ListAndWatch -> Allocate over gRPC on the config-1 tree with GroupCheck on the real context."""
import json
import os
import shutil
import tempfile

import pytest

import conftest  # noqa: F401
import group_check_cases as GC
import test_serve as TS
import util
import kvgpu
from kvgpu import dpapi, serve


class FakeGroupCheck:
    """Context.pci_group_check on the CPU; records the size of every call."""

    def __init__(self):
        self.calls = []

    def __call__(self, recs, want):
        self.calls.append(len(recs))
        bad = GC.first_bad(recs, want)
        return None if bad == len(recs) else bad


@pytest.fixture(scope="module", params=["cpu", pytest.param("gpu", marks=pytest.mark.gpu)])
def leg(request):
    """(group_check, scan_pci) of the leg."""
    if request.param == "cpu":
        yield FakeGroupCheck(), TS.fake_scan_pci
        return
    ctx = kvgpu.Context(0)
    ctx.pciids_load(util.pciids_text())          # kvg_scan_pci joins names; kvg_pci_group_check needs none
    yield ctx.pci_group_check, ctx.scan_pci
    ctx.close()


def outcome(plugin, *requests):
    try:
        return "response", TS.allocate(plugin, *requests).SerializeToString()
    except serve.AllocateError as e:
        return "error", str(e)
    except kvgpu.ReferencePanic as e:
        return "panic", str(e)


class Counting(serve.GroupCheck):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.n_calls = 0

    def __call__(self, pairs):
        self.n_calls += 1
        return super().__call__(pairs)


def same(plugin, leg, *requests):
    """Allocate through BatchRevalidator, then through GroupCheck with the same readers: the outcomes are equal."""
    group_check, scan_pci = leg
    rv = plugin.revalidate
    plugin.revalidate = serve.BatchRevalidator(scan_pci, rv.base_path, rv.read_link, rv.read_id)
    want = outcome(plugin, *requests)
    plugin.revalidate = serve.GroupCheck(group_check, rv.base_path, rv.read_link, rv.read_id)
    got = outcome(plugin, *requests)
    plugin.revalidate = rv
    assert got == want, requests
    return got


def test_reference_vectors(leg, tmp_path):
    a = json.load(open(os.path.join(TS.HERE, "golden", "plugin_vectors.json")))["allocate"]
    kinds = []
    for k, case in enumerate(a["cases"]):
        root = str(tmp_path / ("case%d" % k))
        os.makedirs(root)
        plugin = TS.plugin_for_case(a, case, root)
        kind, body = same(plugin, leg, case["request"])
        kinds.append(kind)
        if case.get("want_error"):
            assert kind == "error" and body.startswith("invalid allocation request: unknown device: ")
    assert kinds.count("response") == 6 and kinds.count("error") == 3


# ---- the reads the re-check exists for ----------------------------------------------------------
# groups: "7" = a GPU and its audio function, "8" = b, "042" = c (its link reads "42"), "42" = d, "9" = no member
MAPS = {"7": ["a", "a1"], "8": ["b"], "042": ["c"], "42": ["d"], "9": []}
BDF = {"a": "7", "a1": "7", "b": "8", "c": "042", "d": "42", "e": "9", "ghost": "7"}
LINKS = {"a": "7", "a1": "7", "b": "8", "c": "42", "d": "42"}
VENDORS = {"a": "10de", "a1": "10de", "b": "10de", "c": "10de", "d": "10de"}
REQUESTS = [["a"], ["a1"], ["b"], ["a", "b"], ["b", "a"], ["c"], ["d"], ["d", "c"], ["e"], ["ghost"],
            ["nope"], ["a", "nope"], ["b", "nope"], ["a", "ghost"]]


def plugin(root, links=None, vendors=None, panic=(), egm=(), iommufd=None):
    m = kvgpu.Maps()
    m.iommuMap = {g: [kvgpu.NvidiaGpuDevice(x, 0) for x in devs] for g, devs in MAPS.items()}
    m.bdfToIommuMap = dict(BDF)
    rl, ri = TS.dict_readers({k: v for k, v in dict(LINKS, **(links or {})).items() if v is not None},
                             {k: v for k, v in dict(VENDORS, **(vendors or {})).items() if v is not None})

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
    reval = serve.BatchRevalidator(TS.fake_scan_pci, base, rl, read_id)
    return serve.GenericDevicePlugin("n", "/", [], m, revalidate=reval, base_path=base, root_path=root,
                                     discover_egm=lambda: egm_devs)


SCENARIOS = {
    "unchanged": {},
    "link moved": dict(links={"a1": "8"}),
    "link unreadable": dict(links={"b": None}),
    "vendor changed": dict(vendors={"a1": "8086"}),
    "vendor upper case": dict(vendors={"b": "10DE"}),
    "vendor unreadable": dict(vendors={"a": None}),
    "short vendor file": dict(panic={"a1"}),
    "short vendor file after a rejected device": dict(panic={"a1"}, links={"a": "8"}),
    "short vendor file behind a moved link": dict(panic={"a1"}, links={"a1": "9"}),
    "042 against 42 both ways": dict(links={"d": "042"}),
}


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_reads(leg, tmp_path, name):
    p = plugin(str(tmp_path), **SCENARIOS[name])
    kinds = {outcome_kind for outcome_kind, _ in (same(p, leg, r) for r in REQUESTS)}
    assert "error" in kinds
    if name == "unchanged":
        assert outcome(p, ["a"])[0] == "response" and outcome(p, ["c"])[0] == "error"      # "42" is not "042"
    if name == "short vendor file":
        assert outcome(p, ["a"])[0] == "panic" and outcome(p, ["b", "a"])[0] == "panic"
    if name in ("short vendor file after a rejected device", "short vendor file behind a moved link"):
        assert "panic" not in kinds


def test_iommufd_and_egm(leg, tmp_path):
    p = plugin(str(tmp_path / "fd"), iommufd={"a": "vfio3", "b": "vfio5"})
    for reqs in (["a"], ["a1"], ["b", "a"]):
        assert same(p, leg, reqs)[0] == "error"                    # a1 has no vfio-dev directory
    assert same(p, leg, ["b"])[0] == "response"
    p = plugin(str(tmp_path / "fd2"), iommufd={"a": "vfio3", "a1": "vfio4", "b": "vfio5"})
    for reqs in (["a"], ["b"], ["a", "b"]):
        assert same(p, leg, reqs)[0] == "response"
    p = plugin(str(tmp_path / "fd3"), iommufd={"a": "vfio3", "a1": "vfio4", "b": "vfio5"}, links={"a1": "8"})
    assert same(p, leg, ["a"]) == ("error", "invalid allocation request: unknown device: a1")
    p = plugin(str(tmp_path / "egm"), egm=[("/dev/egm4", ("a", "b")), ("/dev/egm5", ("d",))])
    for reqs in (["a"], ["a", "b"], ["b", "a"], ["d"], ["a", "b", "d"]):
        same(p, leg, reqs)
    r = dpapi.AllocateResponse.FromString(same(p, leg, ["a", "b"])[1]).container_responses[0]
    assert "/dev/egm4" in [d.host_path for d in r.devices]


def test_several_container_requests(leg, tmp_path):
    p = plugin(str(tmp_path / "ok"))
    for reqs in ((["a"], ["b"]), (["b"], ["a"], ["d"]), (["a"], ["c"]), (["nope"], ["a"]), (["a"], [], ["b"])):
        got = same(p, leg, *reqs)
        if reqs == (["a"], ["b"]):
            r = dpapi.AllocateResponse.FromString(got[1]).container_responses
            assert r[1].envs["PCI_RESOURCE_NVIDIA_COM_N"] == "a,a1,b"    # env_list spans the requests (:361)
    p = plugin(str(tmp_path / "bad"), vendors={"b": "8086"}, panic={"d"})
    for reqs in ((["a"], ["b"]), (["a"], ["d"]), (["b"], ["d"]), (["d"], ["b"])):
        same(p, leg, *reqs)


def test_one_group_check_call_per_container_request(tmp_path):
    fake = FakeGroupCheck()
    p = plugin(str(tmp_path))
    rv = p.revalidate
    check = Counting(fake, rv.base_path, rv.read_link, rv.read_id)
    p.revalidate = check
    TS.allocate(p, ["a"], ["b", "a"], ["d"])
    assert check.n_calls == 3 and fake.calls == [2, 3, 1]
    with pytest.raises(serve.AllocateError):
        TS.allocate(p, ["nope"], ["a"])                          # the first request fails its lookup before any read
    assert check.n_calls == 4 and fake.calls == [2, 3, 1]        # no device to check: no call


def test_records_carry_only_the_reads(tmp_path):
    """What GroupCheck hands the rule: the interned groups (link and maps from one table), the read errors, and the
    vendor as 0x10de only for the exact string "10de"; driver, device and NUMA stay zero."""
    seen = []

    def capture(recs, want):
        seen.append((recs.copy(), want.copy()))
        return FakeGroupCheck()(recs, want)
    p = plugin(str(tmp_path), links={"b": None, "d": "042"}, vendors={"a1": "10DE", "c": None})
    rv = p.revalidate
    check = serve.GroupCheck(capture, rv.base_path, rv.read_link, rv.read_id)
    assert check([("a", "7"), ("a1", "7"), ("b", "8"), ("c", "042"), ("d", "42")]) == 1
    recs, want = seen[0]
    assert list(want) == [0, 0, 1, 2, 3]                          # "7", "8", "042", "42" in first-seen order
    assert list(recs["addr"]) == [0, 1, 2, 3, 4]
    assert list(recs["iommu_group"]) == [0, 0, 0, 3, 2]           # c's link reads "42", d's reads "042"
    assert list(recs["flags"]) == [0, 0, kvgpu._lib.PF_IOMMU_ERR, kvgpu._lib.PF_VENDOR_ERR, 0]
    assert list(recs["vendor"]) == [0x10de, 0xffff, 0x10de, 0xffff, 0x10de]
    assert not recs["driver"].any() and not recs["device"].any() and not recs["numa"].any()
    assert check([]) is None and len(seen) == 1


# ---- over gRPC on the config-1 tree, with the real context ---------------------------------------
@pytest.mark.gpu
def test_scan_to_kubelet_round_trip_with_group_check(tmp_path):
    import grpc
    ids = tmp_path / "pci.ids"
    ids.write_bytes(util.pciids_text())
    base = util.make_pci_tree(str(tmp_path / "pci"), util.c1_tree_entries())
    ds = kvgpu.DiscoveryScan(str(ids), base, str(tmp_path / "nomdev"))
    sockdir = tempfile.mkdtemp(prefix="kvg", dir="/tmp")
    kubelet = serve.MockKubelet(sockdir).start()
    plugins = []
    try:
        maps = ds.create_iommu_device_map()
        check = Counting(ds.ctx.pci_group_check, base)
        plugins = serve.plugins_from_specs(ds.create_device_plugins(), maps, check, socket_dir=sockdir,
                                           base_path=base, root_path=sockdir, discover_egm=lambda: [])
        ref = serve.plugins_from_specs(ds.create_device_plugins(), maps, serve.BatchRevalidator(ds.ctx.scan_pci, base),
                                       socket_dir=sockdir, base_path=base, root_path=sockdir,
                                       discover_egm=lambda: [])
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

        # group 40 = the GPU and its audio function: both checked in one launch, both listed
        r = dpapi.AllocateResponse.FromString(both(["0000:04:00.0"])[1]).container_responses[0]
        assert dict(r.envs) == {"PCI_RESOURCE_NVIDIA_COM_GP102GL_TESLA_P40": "0000:04:00.0,0000:04:00.1"}
        assert [d.host_path for d in r.devices] == ["/dev/vfio/vfio", "/dev/vfio/40"]
        both(["0000:84:00.0", "0000:87:00.0"])
        both(["0000:84:00.0"], ["0000:85:00.0"])
        # the audio function's driver changes: Allocate does not re-check drivers
        real = os.path.realpath(os.path.join(base, "0000:04:00.1"))
        os.remove(os.path.join(real, "driver"))
        assert both(["0000:04:00.0"])[0] == "response"
        # the vendor of 0000:05:00.0 changes -> refused with the reference's text
        real = os.path.realpath(os.path.join(base, "0000:05:00.0"))
        with open(os.path.join(real, "vendor"), "w") as f:
            f.write("0x8086\n")
        assert both(["0000:05:00.0"]) == ("error", "invalid allocation request: unknown device: 0000:05:00.0")
        # the iommu group link of 0000:06:00.0 moves
        real = os.path.realpath(os.path.join(base, "0000:06:00.0"))
        os.remove(os.path.join(real, "iommu_group"))
        os.symlink("../../../kernel/iommu_groups/99", os.path.join(real, "iommu_group"))
        assert both(["0000:07:00.0", "0000:06:00.0"]) == (
            "error", "invalid allocation request: unknown device: 0000:06:00.0")
        assert both(["0000:07:00.0"])[0] == "response"
        assert check.n_calls == 8                                 # one per container request
        c.close()
    finally:
        for p in plugins:
            p.stop()
        kubelet.stop()
        ds.close()
        shutil.rmtree(sockdir, ignore_errors=True)
