"""GPU parity: the CUDA path (through the C-ABI of libkvgpu.so) against the CPU oracle, bit for bit.

Every test here needs an H100 (`-m gpu`).  The oracle is only ever the checker.
"""
import hashlib
import os

import numpy as np
import pytest

import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


@pytest.fixture(scope="module")
def ctx(kv):
    c = kv.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pciids():
    return util.pciids_text()


@pytest.fixture(scope="module")
def loaded(kv, pciids):
    """a context that keeps the shipped pci.ids table (scratch loads go to `ctx`)"""
    c = kv.Context(0)
    c.pciids_load(pciids)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------
# getDeviceName
# ------------------------------------------------------------------------------------------------
def test_ginkgo_get_device_name_kats(ctx):
    G = util.ginkgo()["get_device_name"]
    ctx.pciids_load(G["fixture"].encode())
    for kat in G["kats"]:
        if kat["missing_file"]:
            continue
        assert ctx.name_lookup(kat["key"]) == kat["want"], kat
    # unreadable file -> "" for every key (device_plugin_test.go:405-409): an empty table
    ctx.pciids_load(b"")
    assert ctx.name_lookup("118c") == ""
    assert ctx.name_lookup("") == ""


def test_full_pciids_table_matches_golden(loaded, pciids):
    assert loaded.name_lookup("1b38") == "GP102GL_TESLA_P40"
    d = util.pciids_names()
    info = loaded.pciids_info()
    assert info["vendor_off"] == pciids.index(b"\n10de  NVIDIA") + 1
    assert info["n_lines"] == pciids.count(b"\n")
    names = loaded.name_table(0, 65536)
    got = {"%04x" % i: n for i, n in enumerate(names) if n}
    assert got == {k: v for k, v in d["names"].items() if v}
    table = "".join("%s %s\n" % (k, got.get(k, "")) for k in sorted(d["names"])).encode()
    assert hashlib.sha256(table).hexdigest() == d["table_sha256"]
    # hash path == oracle on hits, misses and other vendors' ids
    rng = np.random.default_rng(7)
    for k in list(rng.integers(0, 65536, 300)) + [0x2331, 0x2330, 0xffff, 0x0000, 0x10de]:
        key = "%04x" % int(k)
        assert loaded.name_lookup(key) == O.get_device_name(pciids, key), key


def test_general_keys_prefix_semantics(loaded, pciids):
    keys = ["", "1", "1b", "1b3", "1b38 ", "1b38  GP102GL", "\t1043", "1B38", "2901  ", "x", "10de",
            "0008  NV1 [STG2000X-B Series]", "0008  NV1 [STG2000X-B Series]x", "#", "\n", "1b38\n",
            "ffffff", "2f", "334", "3340  GB120", "é", "1b3\r"]
    for k in keys:
        assert loaded.name_lookup(k.encode("utf-8")) == O.get_device_name(pciids, k.encode("utf-8")), repr(k)


def _random_pciids(rng, n_lines):
    vend = ["10de", "8086", "10de", "1002", "ffff", "10dx", "C 03", "", "10de  dup", "abcd"]
    alphabet = [b"a", b"B", b"7", b" ", b"  ", b"\t", b"/", b".", b"[", b"]", b"-", b"_", b"\r", b"\x0b",
                b"\x0c", b"\xc4\xb1", b"\xc5\xbf", b"\xc3\xa9", b"\xc2\xa0", b"\xe2\x80\x80", b"\xff",
                b"\xe3\x80\x80", b"(", b"x"]
    out = []
    for _ in range(n_lines):
        r = rng.integers(0, 100)
        if r < 6:
            out.append(rng.choice(vend).encode() + b"  Vendor " + bytes(rng.integers(65, 91, 3).tolist()))
        elif r < 12:
            out.append(b"# comment " + bytes(rng.integers(97, 123, 4).tolist()))
        elif r < 14:
            out.append(b"")
        elif r < 30:
            out.append(b"\t\t" + b"%04x %04x  sub" % (rng.integers(0, 65536), rng.integers(0, 65536)))
        else:
            idv = b"%04x" % rng.integers(0, 40)
            if r > 95:
                idv = idv.upper() if rng.integers(0, 2) else idv[:3]
            sep = [b"  ", b" ", b"\t", b"", b" \xc2\xa0 "][int(rng.integers(0, 5))]
            body = b"".join(alphabet[int(i)] for i in rng.integers(0, len(alphabet), rng.integers(0, 12)))
            out.append(b"\t" + idv + sep + body)
    text = b"\n".join(out)
    if rng.integers(0, 2):
        text += b"\n"
    if rng.integers(0, 4) == 0:
        text = text.replace(b"\n", b"\r\n")
    return text


def test_random_grammar_fuzz(ctx):
    rng = np.random.default_rng(20250711)
    keys = ["%04x" % i for i in range(0, 40)] + ["", "0", "00", "000", "0001 ", "\t", "001\r", "0001\r"]
    for it in range(60):
        text = _random_pciids(rng, int(rng.integers(1, 400)))
        ctx.pciids_load(text)
        for k in keys:
            want = O.get_device_name(text, k.encode())
            got = ctx.name_lookup(k.encode())
            assert got == want, (it, k, text[:200])


def test_tile_boundaries_and_scanner_limit(ctx):
    TILE = 8192
    base = b"8086  Intel\n\t1234  wrong vendor\n"
    # the 10de line, device lines and a section end placed on every offset around a tile edge
    for delta in list(range(-8, 9)) + [8192 - 8, 8192, 8192 + 5]:
        pad_len = TILE - len(base) + delta - 2
        text = base + b"#" + b"c" * pad_len + b"\n" + b"10de  NVIDIA\n\t1234  Edge [case]\n" + \
            b"#" + b"d" * (TILE - 40) + b"\n\t5678  second tile\n10df  next\n\t9999  other\n"
        ctx.pciids_load(text)
        for k in ("1234", "5678", "9999", "abcd"):
            assert ctx.name_lookup(k) == O.get_device_name(text, k.encode()), (delta, k)
    # vendor context carried across many tiles without any header line
    many = b"10de  NVIDIA\n" + b"".join(b"\t%04x  dev %d\n" % (i, i) for i in range(0, 9000)) + b"1000 x\n\t0001  y\n"
    ctx.pciids_load(many)
    for k in ("0000", "0100", "1fff", "2327", "2328", "0001"):
        assert ctx.name_lookup(k) == O.get_device_name(many, k.encode()), k
    # bufio.Scanner 64 KiB token limit
    tail = b"10de  NVIDIA\n\t1234  name\n"
    for n, _ in ((65535, "NAME"), (65536, ""), (70000, "")):
        text = b"x" * n + b"\n" + tail
        ctx.pciids_load(text)
        assert ctx.name_lookup("1234") == O.get_device_name(text, b"1234"), n
    text = b"10de\n\t1234  name\n\t" + b"y" * 65536
    ctx.pciids_load(text)
    assert ctx.name_lookup("1234") == "NAME"
    text = b"10de\n\t" + b"y" * 65536 + b"\n\t1234  name\n"
    ctx.pciids_load(text)
    assert ctx.name_lookup("1234") == ""
    assert ctx.name_lookup("yyyy") == O.get_device_name(text, b"yyyy") == ""


# ------------------------------------------------------------------------------------------------
# createIommuDeviceMap on flat snapshots
# ------------------------------------------------------------------------------------------------
def _explain(got: bytes, want: bytes) -> str:
    g, w = got.split(b"\n"), want.split(b"\n")
    for i, (a, b) in enumerate(zip(g, w)):
        if a != b:
            return "first differing dump line %d of %d/%d: got %r want %r" % (i, len(g), len(w), a, b)
    return "dumps differ in length only: %d vs %d lines" % (len(g), len(w))


def _pci_dump_gpu(kv, ctx, recs):
    res = ctx.scan_pci(recs)
    return kv.canonical_dump(kv.pci_maps_from_result(res)), res


def _pci_dump_oracle(recs, pciids):
    m = O.Maps()
    m.create_iommu_device_map_flat(recs)
    return m.dump(pciids)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 6000, 100_003])
@pytest.mark.parametrize("group_bits", [0, 12])
def test_scan_pci_matches_oracle(kv, loaded, pciids, n, group_bits):
    ids = O.nv_ids(pciids)
    recs = O.gen_pci(0, n, ids, group_bits)
    got, res = _pci_dump_gpu(kv, loaded, recs)
    want = _pci_dump_oracle(recs, pciids)
    assert hashlib.sha256(got).hexdigest() == hashlib.sha256(want).hexdigest()
    assert got == want
    assert res.n_records == n


@pytest.mark.parametrize("bits", [1, 8, 9, 11, 12, 16, 17, 21, 22, 23, 24, 31, 32])
def test_orderings_at_key_width_boundaries(kv, loaded, pciids, bits):
    """The radix digit width is derived on the device from the largest key: walk the plan through
    every pass-count boundary (11 / 22 bits), narrow and full-width keys, and a small device-id range."""
    ids = O.nv_ids(pciids)
    n = 40_000
    recs = O.gen_pci(0, n, ids, 0)
    rng = np.random.default_rng(bits)
    hi = (1 << bits) - 1
    recs["iommu_group"] = rng.integers(0, hi + 1, n, dtype=np.uint64).astype(np.uint32)
    recs[0] = (0x0100, 0x10de, int(ids[0]), hi, 1, 0, 0)      # a certain survivor carrying the widest key
    recs[n - 1] = (0x0200, 0x10de, int(ids[1]), 0, 1, 0, 0)   # ... and the narrowest
    if bits == 8:   # few distinct small device ids: a single-pass ordering 0
        recs["device"] = (recs["device"] & 0x3f).astype(np.uint16)
    got, res = _pci_dump_gpu(kv, loaded, recs)
    assert got == _pci_dump_oracle(recs, pciids)


def test_speculated_pass_sets_are_verified(kv, loaded, pciids):
    """The number of radix pass sets launched for the wide ordering is speculated from the previous scan's largest
    key and verified when the control block comes home (ctrl_fetch): a scan whose keys are wider than the previous
    scan's must re-run its orderings and still match the oracle, through the host entry point and through the
    device-resident entry point + count."""
    import torch
    ids = O.nv_ids(pciids)
    n = 30_000
    for bits in (5, 30, 7, 32, 23, 22):
        recs = O.gen_pci(0, n, ids, 0)
        rng = np.random.default_rng(bits)
        recs["iommu_group"] = rng.integers(0, 1 << bits, n, dtype=np.uint64).astype(np.uint32)
        recs[0] = (0x0100, 0x10de, int(ids[0]), (1 << bits) - 1, 1, 0, 0)
        got, _ = _pci_dump_gpu(kv, loaded, recs)
        assert got == _pci_dump_oracle(recs, pciids), bits
    # device-resident: narrow keys first (the hint), then wide keys; the count call is what verifies
    for bits in (6, 31):
        recs = O.gen_pci(0, n, ids, 0)
        recs["iommu_group"] = np.random.default_rng(bits).integers(0, 1 << bits, n, dtype=np.uint64).astype(np.uint32)
        recs[0] = (0x0100, 0x10de, int(ids[0]), (1 << bits) - 1, 1, 0, 0)
        d = torch.from_numpy(np.frombuffer(recs.tobytes(), dtype=np.uint8).copy()).cuda()
        loaded.dev_scan_pci(d.data_ptr(), n)
        loaded.dev_scan_pci_count()
        res = loaded.dev_scan_pci_fetch()
        assert kv.canonical_dump(kv.pci_maps_from_result(res)) == _pci_dump_oracle(recs, pciids), bits
        del d


def test_scan_beside_a_reparse_on_the_side_stream(kv, pciids):
    """A re-parse of the published image runs on the context's side stream; the PCI scan that follows classifies and
    sorts beside it and joins the names in its final kernel.  Results must equal the oracle's, scan after scan, and
    everything else that needs the table (name lookups, the host entry points, an mdev scan) must wait for it."""
    import torch
    ctx = kv.Context(0)
    try:
        ids = O.nv_ids(pciids)
        pad = ctx.text_pad(len(pciids))
        h = np.full(pad + 16, 10, dtype=np.uint8)
        h[:len(pciids)] = np.frombuffer(pciids, dtype=np.uint8)
        d_text = torch.from_numpy(h).cuda()
        ctx.dev_pciids_parse(d_text.data_ptr(), len(pciids), pad + 16, 1)          # publishes (synchronous)
        for rep, n in enumerate((50_000, 3, 200_001, 0, 2049)):
            recs = O.gen_pci(7 * rep, n, ids, 9)
            d = torch.from_numpy(np.frombuffer(recs.tobytes(), dtype=np.uint8).copy()).cuda() if n else torch.zeros(16, dtype=torch.uint8).cuda()
            ctx.dev_pciids_parse(d_text.data_ptr(), len(pciids), pad + 16, 1)      # re-parse: side stream
            ctx.dev_scan_pci(d.data_ptr(), n)
            res = ctx.dev_scan_pci_fetch()
            assert kv.canonical_dump(kv.pci_maps_from_result(res)) == _pci_dump_oracle(recs, pciids), (rep, n)
            del d
        # the split classify / split final path (>= 2 Mi records): the deferred result must equal the plain one
        n = 2_200_000
        big = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
        ctx.dev_gen_pci(big.data_ptr(), 0, n, ids, 21)
        ctx.dev_scan_pci(big.data_ptr(), n)
        plain = ctx.dev_scan_pci_fetch()
        ctx.dev_pciids_parse(d_text.data_ptr(), len(pciids), pad + 16, 1)
        ctx.dev_scan_pci(big.data_ptr(), n)
        late = ctx.dev_scan_pci_fetch()
        assert np.array_equal(plain.survivors, late.survivors)
        for f in ("dev_keys", "dev_off", "dev_perm", "dev_name_slot", "grp_keys", "grp_off", "grp_perm"):
            assert np.array_equal(getattr(plain, f), getattr(late, f)), f
        assert int((plain.survivors["name_slot"] != 0xffffffff).sum()) > 0
        del big, plain, late
        # a consumer that is not the PCI device scan right after a re-parse
        ctx.dev_pciids_parse(d_text.data_ptr(), len(pciids), pad + 16, 1)
        assert ctx.name_lookup(b"1b38") == O.get_device_name(pciids, b"1b38")
        ctx.dev_pciids_parse(d_text.data_ptr(), len(pciids), pad + 16, 1)
        recs = O.gen_pci(0, 5000, ids, 0)
        got, _ = _pci_dump_gpu(kv, ctx, recs)
        assert got == _pci_dump_oracle(recs, pciids)
        del d_text
    finally:
        torch.cuda.synchronize()
        ctx.close()


@pytest.mark.parametrize("n", [131_072, 131_077, 300_001, 1_048_576 + 1])
def test_pipelined_host_entry_matches_oracle(kv, loaded, pciids, n):
    """kvg_scan_pci switches to the chunked copy / classify / copy-back pipeline at 128 Ki records:
    sizes on and off the tile and chunk boundaries, plus the plain path forced on the same input."""
    ids = O.nv_ids(pciids)
    recs = O.gen_pci(7, n, ids, 18)
    want = _pci_dump_oracle(recs, pciids)
    for rep in range(2):
        got, res = _pci_dump_gpu(kv, loaded, recs)
        assert got == want and res.n_records == n


def test_scan_pci_config2_one_million(kv, loaded, pciids):
    """BASELINE.json config 2: full pci.ids + 1,000,000 synthetic PCI records."""
    ids = O.nv_ids(pciids)
    recs = O.gen_pci(0, 1_000_000, ids, 19)
    want = _pci_dump_oracle(recs, pciids)
    for rep in range(3):   # repeated: a race would not fail every time
        got, res = _pci_dump_gpu(kv, loaded, recs)
        assert hashlib.sha256(got).hexdigest() == hashlib.sha256(want).hexdigest(), (rep, _explain(got, want))
    assert 330_000 < len(res.survivors) < 360_000


def test_scan_pci_edge_populations(kv, loaded, pciids):
    n = 5000
    recs = np.zeros(n, dtype=kv.PCI_REC)
    recs["addr"] = np.arange(n)
    recs["vendor"], recs["device"], recs["driver"] = 0x10de, 0x1b38, 1
    recs["iommu_group"] = 7          # one giant IOMMU group
    recs["numa"] = -1
    got, res = _pci_dump_gpu(kv, loaded, recs)
    assert got == _pci_dump_oracle(recs, pciids)
    assert len(res.survivors) == n and len(res.grp_keys) == 1 and len(res.dev_keys) == 1
    recs["flags"] = 8                # device read fails everywhere -> nothing survives
    got, res = _pci_dump_gpu(kv, loaded, recs)
    assert got == b"" == _pci_dump_oracle(recs, pciids)
    recs["flags"] = 16               # numa unreadable -> kept with numa 0
    recs["numa"] = 5
    recs["iommu_group"] = np.arange(n)[::-1] * 977 % 4099 + 0xFFFF0000  # 32-bit group keys
    recs["device"] = np.arange(n) % 300 + 0x1b00
    got, res = _pci_dump_gpu(kv, loaded, recs)
    assert got == _pci_dump_oracle(recs, pciids)
    assert (res.survivors["numa"] == 0).all()


def test_scan_requires_table(kv):
    c = kv.Context(0)
    with pytest.raises(kv.KvgError) as e:
        c.scan_pci(np.zeros(4, dtype=kv.PCI_REC))
    assert e.value.rc == -5
    c.close()


# ------------------------------------------------------------------------------------------------
# createVgpuIDMap on flat snapshots (BASELINE.json config 3)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 100, 2049, 65536])
def test_scan_mdev_matches_oracle(kv, loaded, pciids, n):
    recs = O.gen_mdev(0, n)
    types = O.gen_type_names(256)
    res = loaded.scan_mdev(recs, types)
    got = kv.canonical_dump(kv.mdev_maps_from_result(res))
    m = O.Maps()
    m.create_vgpu_id_map_flat(recs, types)
    want = m.dump(pciids)
    assert got == want
    if n == 65536:
        assert len(res.type_keys) == 128          # 256 raw names, pairs merge after sanitising
        assert all(nm == "" for nm in res.type_names)  # vGPU labels never match pci.ids (:152-155)


def test_scan_mdev_label_that_matches_pciids(kv, loaded, pciids):
    """A type label that happens to be a device-line prefix DOES resolve (prefix semantics)."""
    recs = O.gen_mdev(0, 64)
    recs["type_idx"] = np.arange(64) % 3
    types = [b"1b38\n", b"GRID  P100X-1B\n", b"\n\n0008  NV1\n"]
    res = loaded.scan_mdev(recs, types)
    got = kv.canonical_dump(kv.mdev_maps_from_result(res))
    m = O.Maps()
    m.create_vgpu_id_map_flat(recs, types)
    assert got == m.dump(pciids)
    assert res.type_names[0] == "GP102GL_TESLA_P40"
    assert res.labels[1] == b"GRID_P100X-1B"


# ------------------------------------------------------------------------------------------------
# health re-scan (BASELINE.json config 5)
# ------------------------------------------------------------------------------------------------
def _alive(recs):
    drop = 1 | 2 | 4 | 8
    return (recs["vendor"] == 0x10de) & ((recs["flags"] & drop) == 0) & (
        (recs["driver"] == 1) | (recs["driver"] == 2))


def test_health_rescan_transitions(kv, loaded, pciids):
    ids = O.nv_ids(pciids)
    n = 10_000
    recs = O.gen_pci(0, n, ids, 0)
    loaded.health_reset()
    prev = np.zeros(n, dtype=bool)
    rng = np.random.default_rng(5)
    for tick in range(6):
        if tick:
            flip = rng.integers(0, n, 10)
            recs["driver"][flip] = rng.integers(0, 5, 10)
            recs["flags"][flip] ^= rng.integers(0, 32, 10).astype(np.uint8)
        d = loaded.health_rescan(recs)
        now = _alive(recs)
        idx = np.nonzero(now != prev)[0]
        want = (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)
        assert d.n_alive == int(now.sum())
        assert np.array_equal(d.changed, want)
        prev = now


# ------------------------------------------------------------------------------------------------
# real directory trees through the plugin-shaped interface
# ------------------------------------------------------------------------------------------------
def test_discovery_scan_on_trees(kv, tmp_path, pciids):
    G = util.ginkgo()
    ids_path = tmp_path / "pci.ids"
    ids_path.write_bytes(pciids)
    # config 1: 8 Tesla P40 + decoys
    base = util.make_pci_tree(str(tmp_path / "c1"), util.c1_tree_entries())
    ds = kv.DiscoveryScan(str(ids_path), base, str(tmp_path / "nomdev"))
    ds.create_iommu_device_map()
    ds.create_vgpu_id_map()
    m = O.Maps()
    m.create_iommu_device_map_tree(base)
    m.create_vgpu_id_map_tree(str(tmp_path / "nomdev"), base)
    assert kv.canonical_dump(ds.maps) == m.dump(pciids)
    specs = {s.key: s for s in ds.create_device_plugins()}
    p40 = specs["1b38"]
    assert p40.resource_name == "nvidia.com/GP102GL_TESLA_P40"
    assert p40.socket_path == "/var/lib/kubelet/device-plugins/kubevirt-GP102GL_TESLA_P40.sock"
    assert p40.env_key == "PCI_RESOURCE_NVIDIA_COM_GP102GL_TESLA_P40"
    assert [d["ID"] for d in p40.devs] == ["0000:%s:00.0" % b for b in
                                           ("04", "05", "06", "07", "84", "85", "86", "87")]
    assert [d["Topology"]["Nodes"][0]["ID"] for d in p40.devs] == [0, 0, 0, 0, 1, 1, 1, 1]
    assert ds.get_device_name("1b38") == "GP102GL_TESLA_P40"
    # the Ginkgo createIommuDeviceMap fixture: non-BDF names, non-numeric groups (index mode)
    base2 = util.make_pci_tree(str(tmp_path / "gk"), G["create_iommu_device_map"]["entries"])
    ds.basePath = base2
    ds.create_iommu_device_map()
    assert ds.maps.iommuMap["io_1"][0].addr == "1"
    assert ds.maps.deviceMap["1b80"][0].addr == "1"
    assert ds.maps.deviceMap["1b81"][0].addr == "2"
    assert ds.maps.bdfToIommuMap["1"] == "io_1"
    assert set(ds.maps.deviceMap) == {"1b80", "1b81"}
    # the Ginkgo createVgpuIDMap fixture
    spec = G["create_vgpu_id_map"]
    mdev, pci = util.make_mdev_tree(str(tmp_path / "vg"), {spec["parent_dir"]: spec["parent_numa_content"]},
                                    spec["entries"])
    ds.vGpuBasePath, ds.basePath = mdev, pci
    ds.create_vgpu_id_map()
    assert ds.maps.gpuVgpuMap["GpuId"][0] == "1"
    assert ds.maps.vGpuMap["vGPUId"][0].addr == "1" and ds.maps.vGpuMap["vGPUId"][0].numaNode == 2
    m2 = O.Maps()
    m2.create_vgpu_id_map_tree(mdev, pci)
    ds.maps.iommuMap, ds.maps.deviceMap, ds.maps.bdfToIommuMap = {}, {}, {}
    assert kv.canonical_dump(ds.maps) == m2.dump(pciids)
    ds.close()


def test_non_canonical_device_strings_are_kept_as_keys(kv, tmp_path, pciids):
    """readIDFromFile returns string(data[2:]) for ANY file content (device_plugin.go:294-302) and that string is
    the deviceMap key (:240) and the getDeviceName argument (:124, prefix match :388-402).  The snapshotter
    carries such strings in index mode; the dump must equal the oracle's on the same tree."""
    ids_path = tmp_path / "pci.ids"
    ids_path.write_bytes(pciids)
    ent = {}
    for i, dev in enumerate(("0x1b38\n", "0X1B38\n", "0x1b3\n", "0x1b38 \n", "garbage\n", "0x\n", "0x1b38\n", "0x2901\n\n")):
        ent["0000:%02x:00.0" % (4 + i)] = dict(vendor="10de", device=dev, driver="vfio-pci", iommu_group=str(40 + i),
                                              numa_node="%d\n" % (i & 1))
    base = util.make_pci_tree(str(tmp_path / "odd"), ent)
    ds = kv.DiscoveryScan(str(ids_path), base, str(tmp_path / "nomdev"))
    ds.create_iommu_device_map()
    m = O.Maps()
    m.create_iommu_device_map_tree(base)
    assert kv.canonical_dump(ds.maps) == m.dump(pciids)
    assert set(ds.maps.deviceMap) == {"1b38", "0X1B38", "1b3", "1b38 ", "garbage", "", "2901"}
    assert ds.maps.deviceNames["1b3"] == "0_GP102GL_QUADRO_P6000"       # prefix semantics (:388)
    assert len(ds.maps.deviceMap["1b38"]) == 2
    ds.close()
    # the native host layer (C++ above the same C-ABI) carries them the same way
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "kubevirt-gpu-device-plugin_b200", "kvg-discover")
    r = subprocess.run([exe, "--pci-ids", str(ids_path), "--sysfs-pci", base, "--sysfs-mdev", str(tmp_path / "nomdev"), "--dump"],
                       capture_output=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert r.stdout == m.dump(pciids)


# ------------------------------------------------------------------------------------------------
# device-resident path, generators, batch parse, full-size properties
# ------------------------------------------------------------------------------------------------
def test_device_generators_match_oracle(kv, loaded, pciids):
    import torch
    ids = O.nv_ids(pciids)
    n = 50_001
    buf = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    for bits in (0, 15):
        loaded.dev_gen_pci(buf.data_ptr(), 1234567, n, ids, bits)
        loaded.dev_scan_pci(buf.data_ptr(), 0)  # stream sync via fetch
        loaded.dev_scan_pci_count()
        got = np.frombuffer(buf.cpu().numpy().tobytes(), dtype=kv.PCI_REC)
        assert np.array_equal(got, O.gen_pci(1234567, n, ids, bits))
    mb = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
    loaded.dev_gen_mdev(mb.data_ptr(), 99, n)
    loaded.dev_scan_pci_count()
    got = np.frombuffer(mb.cpu().numpy().tobytes(), dtype=kv.MDEV_REC)
    want = O.gen_mdev(99, n)
    assert got.tobytes() == want.tobytes()


def test_batch_parse_device_resident(kv, pciids):
    import torch
    c = kv.Context(0)
    n_files = 5
    stride = c.text_pad(len(pciids)) + 16
    host = np.full(stride * n_files, 10, dtype=np.uint8)
    for f in range(n_files):
        host[f * stride:f * stride + len(pciids)] = np.frombuffer(pciids, dtype=np.uint8)
    dev = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    c.dev_pciids_parse(dev.data_ptr(), len(pciids), stride, n_files)
    info = c.pciids_info()
    assert info["n_lines"] == pciids.count(b"\n")
    d = util.pciids_names()
    names = c.name_table(0, 65536)
    assert {"%04x" % i: n for i, n in enumerate(names) if n} == {k: v for k, v in d["names"].items() if v}
    # the table holds the device lines under vendor 10de only (nothing else is ever looked up)
    assert sum(1 for v in d["names"].values() if v) <= info["n_entries"] < 4000
    c.dev_pciids_parse(dev.data_ptr(), len(pciids), stride, n_files)  # steady-state path
    assert c.name_lookup("2901") == "GB100_B200"
    c.close()


def test_full_size_properties(kv, loaded, pciids):
    """16,777,216 records (> L2): size-independent properties instead of the oracle."""
    import torch
    ids = O.nv_ids(pciids)
    n = 1 << 24
    buf = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    loaded.dev_gen_pci(buf.data_ptr(), 0, n, ids, 23)
    loaded.dev_scan_pci(buf.data_ptr(), n)
    res = loaded.dev_scan_pci_fetch()
    recs = np.frombuffer(buf.cpu().numpy().tobytes(), dtype=kv.PCI_REC)
    alive = _alive(recs)
    S = int(alive.sum())
    assert len(res.survivors) == S
    # stable compaction: survivors are exactly the alive records, in order
    assert np.array_equal(res.survivors["addr"], recs["addr"][alive])
    assert np.array_equal(res.survivors["iommu_group"], recs["iommu_group"][alive])
    assert np.array_equal(res.survivors["device"], recs["device"][alive])
    for keys, off, perm, field in ((res.dev_keys, res.dev_off, res.dev_perm, "device"),
                                   (res.grp_keys, res.grp_off, res.grp_perm, "iommu_group")):
        assert np.all(np.diff(keys.astype(np.int64)) > 0)            # distinct, ascending
        assert off[0] == 0 and off[-1] == S and np.all(np.diff(off.astype(np.int64)) > 0)
        assert np.array_equal(np.sort(perm), np.arange(S, dtype=np.uint32))  # a permutation
        k_of = res.survivors[field][perm]
        assert np.array_equal(k_of, np.repeat(keys, np.diff(off)))   # bucket k holds key k only
        same = k_of[1:] == k_of[:-1]
        assert np.all(perm[1:][same] > perm[:-1][same])              # stable inside a bucket
    # the join: name slots agree with the table for every distinct device id
    names = loaded.name_table(0, 65536)
    for k in range(0, len(res.dev_keys), 97):
        assert res.name_at(int(res.dev_name_slot[k])) == names[int(res.dev_keys[k])]


# ------------------------------------------------------------------------------------------------
# multi-GPU (BASELINE.json config 4): sharded scan == single scan == oracle
# ------------------------------------------------------------------------------------------------
def _gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("n", [200_003, 5])
def test_sharded_scan_matches_oracle(n, mode):
    """One process per GPU of the box (world 1 on a single-GPU box: the exchange kernels — multisplit by
    owner, window stores, flags, gather, acks — still run, with one owner).  PCI and mdev records."""
    import subprocess
    import sys
    world = max(1, min(_gpu_count(), 8))
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29600 + n % 300 + (0 if mode == "p2p" else 301)),
           os.path.join(here, "_nccl_worker.py"), str(n), mode]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=400)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "nccl-ok world=%d n=%d" % (world, n) in r.stdout


def test_native_host_layer_matches_oracle(tmp_path, pciids):
    """libkvghost.so / kvg-discover (C++ host above the C-ABI) on real trees == oracle dump."""
    import subprocess
    ids_path = tmp_path / "pci.ids"
    ids_path.write_bytes(pciids)
    G = util.ginkgo()
    ent = util.c1_tree_entries()
    ent.update(G["create_iommu_device_map"]["entries"])
    base = util.make_pci_tree(str(tmp_path / "pci"), ent)
    spec = G["create_vgpu_id_map"]
    mdev, mpci = util.make_mdev_tree(str(tmp_path / "vg"), {spec["parent_dir"]: spec["parent_numa_content"]},
                                     spec["entries"])
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "kubevirt-gpu-device-plugin_b200", "kvg-discover")
    r = subprocess.run([exe, "--pci-ids", str(ids_path), "--sysfs-pci", base, "--sysfs-mdev", mdev, "--dump"],
                       capture_output=True, timeout=120)
    assert r.returncode == 0, r.stderr
    m = O.Maps()
    m.create_iommu_device_map_tree(base)
    m.create_vgpu_id_map_tree(mdev, base)   # parents' numa is read under the PCI base (:280)
    assert r.stdout == m.dump(pciids)
    r = subprocess.run([exe, "--pci-ids", str(ids_path), "--sysfs-pci", base, "--sysfs-mdev", mdev],
                       capture_output=True, text=True, timeout=120)
    assert ("P 1b38 GP102GL_TESLA_P40 nvidia.com/GP102GL_TESLA_P40 "
            "/var/lib/kubelet/device-plugins/kubevirt-GP102GL_TESLA_P40.sock "
            "PCI_RESOURCE_NVIDIA_COM_GP102GL_TESLA_P40 8\n  0000:04:00.0 Healthy 0\n") in r.stdout
    assert "P vGPUId vGPUId nvidia.com/vGPUId " in r.stdout and "MDEV_PCI_RESOURCE_NVIDIA_COM_VGPUID 2" in r.stdout
