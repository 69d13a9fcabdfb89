"""The health re-scans from raw reads (kvg_health_rescan_groups_raw / kvg_health_rescan_mdev_raw), both kernel forms
of both kinds executed on the CPU from their real source under the warp emulator of tools/emu/: k_health_raw_small
and k_compact<RawHealthOp>, against the string-level reference of tests/health_raw_ref.py.  The harness keeps the
previous list as the host driver does: a call writes this call's bytes, and its names and bytes become the previous
list only when the call is not refused."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import health_raw_ref as HR
import mdev_raw_cases as MC
import raw_scan_cases as RC
from kvgpu import _lib as L
from raw_scan_cases import MISSING, RawError

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

vp, u32, i32 = C.c_void_p, C.c_uint32, C.c_int
SMALL, COMPACT = 0, 1
MAX_GROUPS, MAX_XID = 4096, 1024


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("health_raw"))
    for f in (lib.emu_health_groups_raw, lib.emu_health_mdev_raw):
        f.argtypes = [i32, vp, vp, vp, u32, vp, vp, u32, vp, vp, vp, u32, vp, vp, vp]
    return lib


def strings(xs):
    """a list of byte strings -> (offsets, blob) with room for the empty list"""
    off = np.zeros(len(xs) + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(x) for x in xs], dtype=np.uint64)
    return off, np.frombuffer(b"".join(xs) + b"\0", dtype=np.uint8).copy()


class Harness:
    """One kind's previous list as the library keeps it, run through either kernel form and checked against the
    reference after every call."""

    def __init__(self, emu, kind):
        self.kind = kind
        self.fn = emu.emu_health_groups_raw if kind == "groups" else emu.emu_health_mdev_raw
        self.fields = L.RAW_FIELDS if kind == "groups" else L.MRAW_FIELDS
        self.ref = HR.RawGroupsRef() if kind == "groups" else HR.RawMdevRef()
        self.prev = (np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint8), np.zeros(1, dtype=np.uint8), 0)

    def kernel(self, raw, sets, form):
        """-> (refusal kind or None, n_alive, changed)"""
        n = len(raw.state)
        if n == 0:   # the library's reset: nothing launched
            self.prev = (self.prev[0], self.prev[1], self.prev[2], 0)
            return None, 0, []
        off = np.ascontiguousarray(raw.off, dtype=np.uint32)
        st = np.ascontiguousarray(raw.state, dtype=np.uint16)
        blob = np.frombuffer(bytes(raw.bytes) + b"\0", dtype=np.uint8).copy()
        soff, sblob = strings(sets)
        state_out = np.zeros(n + 1, dtype=np.uint8)
        changed = np.zeros(n + 1, dtype=np.uint32)
        hdr = np.zeros(10, dtype=np.uint32)
        poff, pbytes, pstate, pn = self.prev
        assert self.fn(form, off.ctypes.data, st.ctypes.data, blob.ctypes.data, n, soff.ctypes.data, sblob.ctypes.data,
                       len(sets), poff.ctypes.data, pbytes.ctypes.data, pstate.ctypes.data, pn, state_out.ctypes.data,
                       changed.ctypes.data, hdr.ctypes.data) == 0
        v = hdr[4:].view(np.uint64)
        for kind, word in (("miss", v[0]), ("panic", v[1]), ("range", v[2])):
            if int(word) != (1 << 64) - 1:
                return kind, 0, []
        if hdr[3]:
            return "order", 0, []
        self.prev = (off, blob, state_out, n)
        return None, int(hdr[0]), [int(x) for x in changed[:int(hdr[1])]]

    def call(self, raw, sets, form):
        """one call, checked against the reference; -> the refusal kind or the Delta"""
        got = self.kernel(raw, sets, form)
        if len(raw.state) == 0:
            self.ref.prev = {}
            return HR.Delta(0, 0, [])
        try:
            want = self.ref.step(raw, sets)
        except RawError as e:
            assert got[0] == e.kind, (got, e)
            return e.kind
        assert got[0] is None, got
        assert (got[1], got[2]) == (want.n_alive, want.changed)
        return want


# ---- passthrough GPUs by IOMMU group --------------------------------------------------------------------------------
def bdf_name(k):
    return b"0000:%02x:%02x.%d" % (k >> 8 & 0xFF, k >> 3 & 31, k & 7)


def pci_entry(group, vendor=b"0x10de\n", driver=b"../../../bus/pci/drivers/vfio-pci", numa=b"0\n",
              device=b"0x20b0\n"):
    return {"vendor": vendor, "driver": driver, "iommu_group": b"../../../kernel/iommu_groups/" + group,
            "numa_node": numa, "device": device}


def pci_raw(names_groups, **kw):
    return RC.raw_of([(nm, pci_entry(g, **kw)) for nm, g in names_groups])


def gen_groups(rng, n, name_kind="canonical"):
    """n alive-ish entries with random group strings (some decimal, some not), names ascending byte-wise"""
    pool = [b"%d" % k for k in range(40)] + [b"042", b"vfio", b"devices", b"g-7", b""]
    if name_kind == "canonical":
        names = [bdf_name(k) for k in sorted(rng.choice(1 << 16, size=n, replace=False))]
    else:   # non-canonical and prefixes of each other
        names = sorted({b"gpu" + b"x" * int(rng.integers(0, 3)) + b"%d" % int(rng.integers(0, 4 * n))
                        for _ in range(3 * n)})[:n]
    out = []
    for nm in names:
        e = pci_entry(pool[rng.integers(len(pool))])
        r = rng.random()
        if r < 0.05:
            e["vendor"] = b"0x8086\n"
        elif r < 0.1:
            e["driver"] = b"../nvidia"
        elif r < 0.13:
            e["iommu_group"] = None
        elif r < 0.2:
            e["numa_node"] = RC.NUMAS[rng.integers(len(RC.NUMAS))]
            if e["numa_node"] in (b"9223372036854775807", b"-9223372036854775808", b"32768", b"-32769"):
                e["numa_node"] = b"-1\n"
        out.append((nm, e))
    return RC.raw_of(out)


def node_list(rng, k=20):
    pool = [b"%d" % j for j in range(40)] + [b"42", b"vfio", b"devices", b"g-7"]
    xs = [pool[rng.integers(len(pool))] for _ in range(k)]
    return xs + xs[: k // 3]   # duplicates


@pytest.mark.parametrize("form", [SMALL, COMPACT])
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 2047, 2048, 2049])
def test_groups_sizes(emu, form, n):
    rng = np.random.default_rng(n + 7 * form)
    h = Harness(emu, "groups")
    raw = gen_groups(rng, n)
    for _ in range(3):
        h.call(raw, node_list(rng), form)


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_groups_non_canonical_names_and_list_changes(emu, form):
    rng = np.random.default_rng(3 + form)
    h = Harness(emu, "groups")
    raw = gen_groups(rng, 300, name_kind="other")
    nodes = node_list(rng)
    h.call(raw, nodes, form)
    names = [raw.bytes[raw.off[i * L.RAW_FIELDS]:raw.off[i * L.RAW_FIELDS + 1]] for i in range(len(raw.state))]
    assert any(names[i + 1].startswith(names[i]) for i in range(len(names) - 1))
    # remove and add entries in the middle of the list: the others keep their state (nothing listed for them)
    entries = [(names[i], _entry_of(raw, i)) for i in range(len(names))]
    entries2 = entries[:100] + entries[120:] + [(names[150] + b"~new", pci_entry(b"1"))]
    entries2.sort(key=lambda x: x[0])
    d = h.call(RC.raw_of(entries2), nodes, form)
    new_i = [k for k, (nm, _) in enumerate(entries2) if nm.endswith(b"~new")][0]
    assert all(w >> 1 == new_i for w in d.changed)


def _entry_of(raw, i, fields=L.RAW_FIELDS, keys=RC.FIELDS):
    st = int(raw.state[i])
    e = {}
    for f, key in enumerate(keys, start=1):
        if not (st >> f) & 1:
            e[key] = MISSING
        elif (st >> (8 + f)) & 1:
            e[key] = None
        else:
            e[key] = raw.bytes[raw.off[i * fields + f]:raw.off[i * fields + f + 1]]
    return e


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_groups_string_identity(emu, form):
    h = Harness(emu, "groups")
    raw = pci_raw([(bdf_name(1), b"042"), (bdf_name(2), b"42"), (bdf_name(3), b"vfio"), (bdf_name(4), b"devices"),
                   (bdf_name(5), b"7")])
    assert h.call(raw, [b"42"], form).changed == [3]
    assert h.call(raw, [b"042", b"vfio", b"7", b"7"], form).changed == [1, 2, 5, 9]
    assert h.call(raw, [], form).changed == [0, 4, 8]      # an empty listing: no node exists
    assert h.call(raw, [b"devices"], form).changed == [7]


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_groups_node_vanishes_and_returns(emu, form):
    h = Harness(emu, "groups")
    raw = pci_raw([(bdf_name(k), b"%d" % (k // 4)) for k in range(16)])
    all_nodes = [b"%d" % g for g in range(4)]
    assert len(h.call(raw, all_nodes, form).changed) == 16
    d = h.call(raw, [b"0", b"1", b"3"], form)
    assert d.changed == [(k << 1) for k in range(8, 12)]
    d = h.call(raw, all_nodes, form)
    assert d.changed == [(k << 1) | 1 for k in range(8, 12)]


def refusal_cases_groups():
    ok = [(bdf_name(k), pci_entry(b"1")) for k in range(4)]
    miss = [ok[0], (bdf_name(1), dict(pci_entry(b"1"), driver=MISSING))] + ok[2:]
    panic = [ok[0], (bdf_name(1), dict(pci_entry(b"1"), device=b"0"))] + ok[2:]
    rng = [ok[0], (bdf_name(1), dict(pci_entry(b"1"), numa_node=b"32768"))] + ok[2:]
    desc = [ok[1], ok[0]] + ok[2:]
    dup = [ok[0], ok[0]] + ok[2:]
    return {"miss": miss, "panic": panic, "range": rng, "order": desc, "order_dup": dup}


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_groups_refusals_leave_the_list(emu, form):
    h = Harness(emu, "groups")
    base = pci_raw([(bdf_name(k), b"1") for k in range(4)])
    h.call(base, [b"1"], form)
    for case, ents in refusal_cases_groups().items():
        assert h.call(RC.raw_of(ents), [b"1"], form) == case.split("_")[0]
        assert h.call(base, [b"1"], form).changed == []    # the list is still the base's
    # the order check spans a row / tile edge too
    n = 2049
    names = [bdf_name(k) for k in range(n)]
    names[1024], names[1023] = names[1023], names[1024]
    names[2048], names[2047] = names[2047], names[2048]
    assert h.call(pci_raw([(x, b"1") for x in names]), [b"1"], form) == "order"
    # a precedence: a miss beats a panic of an earlier entry
    ents = refusal_cases_groups()
    mixed = [ents["panic"][1], (bdf_name(2), dict(pci_entry(b"1"), numa_node=MISSING))]
    assert h.call(RC.raw_of(mixed), [], form) == "miss"


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_groups_reset_and_caps(emu, form):
    h = Harness(emu, "groups")
    raw = pci_raw([(bdf_name(k), b"%d" % k) for k in range(8)])
    assert len(h.call(raw, [b"%d" % k for k in range(8)], form).changed) == 8
    h.call(RC.raw_of([]), [], form)    # n = 0: the reset
    assert len(h.call(raw, [b"%d" % k for k in range(8)], form).changed) == 8
    at = [b"%d" % k for k in range(MAX_GROUPS)]
    d = h.call(raw, at, form)
    assert d.changed == []
    assert h.fn(form, None, None, None, 1, None, None, MAX_GROUPS + 1, None, None, None, 0, None, None, None) == -1


# ---- vGPUs ---------------------------------------------------------------------------------------------------------
def mdev_entry(parent, name, typ=b"GRID T4-1Q\n", numa=b"0\n"):
    return {"type": typ, "link": MC.link_to(parent, name), "numa_node": numa}


def uuid(k):
    return b"%08x-0000-4000-8000-%012x" % (k, k)


@pytest.mark.parametrize("form", [SMALL, COMPACT])
@pytest.mark.parametrize("n", [1, 1024, 1025, 2048, 2049])
def test_mdev_sizes(emu, form, n):
    rng = np.random.default_rng(100 + n + form)
    h = Harness(emu, "mdev")
    ents = MC.gen_entries(rng, n, parents="mixed")
    for nm, e in ents:
        if e["numa_node"] in (b"9223372036854775807", b"-9223372036854775808", b"32768", b"-32769"):
            e["numa_node"] = b"1\n"
    ents.sort(key=lambda x: x[0])
    ents = [x for k, x in enumerate(ents) if k == 0 or x[0] != ents[k - 1][0]]
    raw = MC.raw_of(ents)
    buses = [b"0000:%02x:00.0" % k for k in range(64)] + [b"", b"\n", b"0000:0A:00.0"]
    for _ in range(3):
        xs = [buses[rng.integers(len(buses))] for _ in range(int(rng.integers(0, 6)))]
        h.call(raw, xs + xs[:1], form)


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_mdev_xid_marks_survive_list_changes(emu, form):
    h = Harness(emu, "mdev")
    gpu = [b"0000:%02x:00.0" % k for k in range(3)]
    ents = [(uuid(k), mdev_entry(gpu[k % 3], uuid(k))) for k in range(9)]
    raw = MC.raw_of(ents)
    assert len(h.call(raw, [], form).changed) == 9
    d = h.call(raw, [gpu[1], gpu[1]], form)                 # duplicates mark once
    assert d.changed == [(k << 1) for k in (1, 4, 7)]
    # a vGPU created on another GPU and one destroyed: the marks stay, nothing else is listed
    ents2 = [e for k, e in enumerate(ents) if k != 3] + [(uuid(5) + b"x", mdev_entry(gpu[2], uuid(5) + b"x"))]
    ents2.sort(key=lambda x: x[0])
    d = h.call(MC.raw_of(ents2), [], form)
    new_i = [k for k, (nm, _) in enumerate(ents2) if nm.endswith(b"x")][0]
    assert d.changed == [(new_i << 1) | 1]
    # a marked vGPU that leaves and returns starts unmarked
    ents3 = [e for e in ents2 if e[0] != uuid(4)]
    h.call(MC.raw_of(ents3), [], form)
    d = h.call(MC.raw_of(ents2), [], form)
    back = [k for k, (nm, _) in enumerate(ents2) if nm == uuid(4)][0]
    assert d.changed == [(back << 1) | 1]


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_mdev_non_canonical_names_and_empty_parent(emu, form):
    h = Harness(emu, "mdev")
    ents = [(b"1", mdev_entry(b"0000:01:00.0", b"1")), (b"10", mdev_entry(b"", b"10")),
            (b"2", {"type": b"x", "link": b"a//2", "numa_node": b"1\n"}), (b"ABC", mdev_entry(b"0000:01:00.0", b"ABC"))]
    raw = MC.raw_of(ents)
    h.call(raw, [], form)
    d = h.call(raw, [b"", b"0000:01:00.0"], form)
    assert d.changed == [0, 6]       # the empty parents are marked by nothing


@pytest.mark.parametrize("form", [SMALL, COMPACT])
def test_mdev_refusals(emu, form):
    h = Harness(emu, "mdev")
    ok = [(uuid(k), mdev_entry(b"0000:01:00.0", uuid(k))) for k in range(3)]
    base = MC.raw_of(ok)
    h.call(base, [b"0000:01:00.0"], form)
    cases = {"miss": [ok[0], (uuid(1), dict(ok[1][1], link=MISSING)), ok[2]],
             "panic": [ok[0], (uuid(1), dict(ok[1][1], link=b"nolash")), ok[2]],
             "range": [ok[0], (uuid(1), dict(ok[1][1], numa_node=b"-32769")), ok[2]],
             "order": [ok[1], ok[0], ok[2]]}
    for kind, ents in cases.items():
        assert h.call(MC.raw_of(ents), [], form) == kind
        assert h.call(base, [], form).changed == []     # still the base's list: every vGPU marked, none listed
    h.call(MC.raw_of([]), [], form)
    assert len(h.call(base, [b"%d" % k for k in range(MAX_XID)], form).changed) == 3
    assert h.fn(form, None, None, None, 1, None, None, MAX_XID + 1, None, None, None, 0, None, None, None) == -1
