"""kvg_health_rescan_groups_raw / kvg_health_rescan_mdev_raw on the H100.

  equivalence  canonical names (BDFs / UUIDs), group and parent strings interned through one dict kept across ticks,
               nodes and bus ids resolved through it: every delta equals, byte for byte, that of
               kvg_health_rescan_groups_keyed / kvg_health_rescan_mdev_keyed on the decoded records
  sequences    against the string-level reference (tests/health_raw_ref.py) at every size regime, any names
  refusals     each leaves the list unchanged
  isolation    the other health states, the raw scans and raw deltas are not disturbed, and do not disturb
  launches     a poll-loop tick is one kernel launch

The call stages its inputs in every case, so pinned and pageable inputs take the same path and are not told apart."""
import gzip
import os

import numpy as np
import pytest

import conftest
import health_keyed_ref
import health_raw_ref as HR
import kvgpu
import mdev_raw_cases as MC
import raw_scan_cases as RC
from kvgpu import _lib as L
from raw_scan_cases import MISSING

pytestmark = pytest.mark.gpu
GROUP_POOL = [b"%d" % k for k in range(60)] + [b"042", b"vfio", b"devices", b"g-7", b""]
NODE_POOL = [b"%d" % k for k in range(60)] + [b"42", b"vfio", b"devices", b"g-7"]
BUS_POOL = [b"0000:%02x:00.0" % k for k in range(64)] + [b"", b"0000:0A:00.0"]


@pytest.fixture(scope="module")
def ctx():
    with kvgpu.Context(0) as c:
        yield c


def bdf_names(rng, n):
    return [kvgpu.format_bdf(int(a)).encode() for a in np.sort(rng.choice(1 << 24, size=n, replace=False))]


def pci_entries(rng, n, names):
    out = []
    for nm in names:
        e = {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "numa_node": b"0\n", "device": b"0x2330\n",
             "iommu_group": b"../iommu_groups/" + GROUP_POOL[rng.integers(len(GROUP_POOL))]}
        r = rng.random()
        if r < 0.04:
            e["vendor"] = b"0x8086\n"
        elif r < 0.08:
            e["driver"] = None
        elif r < 0.11:
            e["iommu_group"] = None
        elif r < 0.14:
            e["device"] = None
        out.append((nm, e))
    return out


def nodes_of(rng):
    xs = [NODE_POOL[rng.integers(len(NODE_POOL))] for _ in range(int(rng.integers(0, 50)))]
    return xs + xs[:3]


def changed(d):
    return [int(x) for x in d.changed]


def decode_pci(raw, intern):
    """the decoded records with group handles from `intern` (string -> handle from 1; no group -> 0)"""
    recs = RC.go_snapshot(raw)[0].copy()
    for i, (_, _, g) in enumerate(HR.pci_entries(raw)):
        recs[i]["iommu_group"] = intern.setdefault(g, len(intern) + 1) if g else 0
    return recs


def decode_mdev(raw, intern):
    recs, _, _, types, _ = MC.go_mdev_snapshot(raw)
    recs = recs.copy()
    for i, (_, _, p) in enumerate(HR.mdev_entries(raw)):
        recs[i]["parent"] = intern.setdefault(p, len(intern) + 1) if p else 0
    return recs, len(types)


@pytest.mark.parametrize("n", [1000, 10_000, 40_000])
def test_groups_equal_keyed_on_canonical_input(ctx, n):
    rng = np.random.default_rng(n)
    names = bdf_names(rng, n + n // 10)
    intern = {}
    ctx.health_rescan_groups_raw(RC.raw_of([])), ctx.health_rescan_groups_keyed(np.zeros(0, L.PCI_REC))
    for t in range(5):
        keep = np.sort(rng.choice(len(names), size=n, replace=False))
        raw = RC.raw_of(pci_entries(rng, n, [names[k] for k in keep]))
        nodes = nodes_of(rng)
        a = ctx.health_rescan_groups_raw(raw, nodes)
        recs = decode_pci(raw, intern)
        b = ctx.health_rescan_groups_keyed(recs, [intern[x] for x in nodes if x in intern])
        assert (a.n_records, a.n_alive) == (b.n_records, b.n_alive)
        assert np.array_equal(a.changed, b.changed)


def mdev_entries(rng, names):
    ents = []
    for nm in names:
        parent = BUS_POOL[rng.integers(len(BUS_POOL) - 2)]
        e = {"type": b"GRID T4-%dQ\n" % rng.integers(4), "link": MC.link_to(parent, nm), "numa_node": b"0\n"}
        r = rng.random()
        if r < 0.05:
            e["type"] = None
        elif r < 0.1:
            e["link"] = None
        ents.append((nm, e))
    return ents


@pytest.mark.parametrize("n", [1000, 10_000, 40_000])
def test_mdev_equal_keyed_on_canonical_input(ctx, n):
    rng = np.random.default_rng(n + 1)
    names = MC.canonical_names(rng, n + n // 10)
    intern = {}
    ctx.health_rescan_mdev_raw(MC.raw_of([])), ctx.health_rescan_mdev_keyed(np.zeros(0, L.MDEV_REC), 0)
    for t in range(6):
        keep = np.sort(rng.choice(len(names), size=n, replace=False))
        raw = MC.raw_of(mdev_entries(rng, [names[k] for k in keep]))
        xids = [BUS_POOL[rng.integers(len(BUS_POOL))] for _ in range(int(rng.integers(0, 4)))]
        a = ctx.health_rescan_mdev_raw(raw, xids)
        recs, n_types = decode_mdev(raw, intern)
        b = ctx.health_rescan_mdev_keyed(recs, n_types, [intern[x] for x in xids if x in intern])
        assert (a.n_records, a.n_alive) == (b.n_records, b.n_alive)
        assert np.array_equal(a.changed, b.changed)


def any_names(rng, n):
    """byte-wise ascending names of any form, prefixes of each other among them"""
    xs = set()
    while len(xs) < n:
        xs.add(b"dev" + b"-" * int(rng.integers(0, 2)) + b"%x" % int(rng.integers(0, 8 * n)))
    return sorted(xs)


@pytest.mark.parametrize("n", [1, 1000, 10_000, 32_768, 32_769, 200_000])
def test_groups_sequences(ctx, n):
    rng = np.random.default_rng(10 + n)
    names = any_names(rng, n + n // 20 + 1)
    ref = HR.RawGroupsRef()
    ctx.health_rescan_groups_raw(RC.raw_of([]))
    for t in range(4):
        keep = np.sort(rng.choice(len(names), size=n, replace=False))
        raw = RC.raw_of(pci_entries(rng, n, [names[k] for k in keep]))
        nodes = nodes_of(rng)
        d, w = ctx.health_rescan_groups_raw(raw, nodes), ref.step(raw, nodes)
        assert (d.n_records, d.n_alive, changed(d)) == (w.n_records, w.n_alive, w.changed)


@pytest.mark.parametrize("n", [1, 1000, 10_000, 32_768, 32_769, 200_000])
def test_mdev_sequences(ctx, n):
    rng = np.random.default_rng(20 + n)
    names = any_names(rng, n + n // 20 + 1)
    ref = HR.RawMdevRef()
    ctx.health_rescan_mdev_raw(MC.raw_of([]))
    for t in range(4):
        keep = np.sort(rng.choice(len(names), size=n, replace=False))
        raw = MC.raw_of(mdev_entries(rng, [names[k] for k in keep]))
        xids = [BUS_POOL[rng.integers(len(BUS_POOL))] for _ in range(int(rng.integers(0, 4)))]
        d, w = ctx.health_rescan_mdev_raw(raw, xids), ref.step(raw, xids)
        assert (d.n_records, d.n_alive, changed(d)) == (w.n_records, w.n_alive, w.changed)


def pci_ok(k, group=b"1"):
    return (b"0000:00:%02x.0" % k, {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "numa_node": b"0\n",
                                    "device": b"0x2330\n", "iommu_group": b"../" + group})


@pytest.mark.parametrize("n", [4, 40_000])
def test_refusals_leave_the_list(ctx, n):
    base_e = [(b"e%06d" % k, pci_ok(0)[1]) for k in range(n)]
    base = RC.raw_of(base_e)
    ctx.health_rescan_groups_raw(RC.raw_of([]))
    assert len(ctx.health_rescan_groups_raw(base, [b"1"]).changed) == n
    bad = {L.KVG_EINVAL: [dict(base_e[1][1], driver=MISSING)], L.KVG_EPANIC: [dict(base_e[1][1], vendor=b"0")],
           L.KVG_ERANGE: [dict(base_e[1][1], numa_node=b"32768")]}
    for rc, (e,) in bad.items():
        ents = list(base_e)
        ents[n - 1] = (ents[n - 1][0], e)
        with pytest.raises((kvgpu.KvgError, kvgpu.ReferencePanic)) as ex:
            ctx.health_rescan_groups_raw(RC.raw_of(ents), [b"1"])
        assert rc == (L.KVG_EPANIC if isinstance(ex.value, kvgpu.ReferencePanic) else ex.value.rc)
        assert len(ctx.health_rescan_groups_raw(base, [b"1"]).changed) == 0
    for ents in ([base_e[1], base_e[0]] + base_e[2:], [base_e[0]] + base_e[:-1]):   # descending, duplicate
        with pytest.raises(kvgpu.KvgError, match="ascend"):
            ctx.health_rescan_groups_raw(RC.raw_of(ents), [b"1"])
        assert len(ctx.health_rescan_groups_raw(base, [b"1"]).changed) == 0
    # the caps, exactly at and one past
    assert len(ctx.health_rescan_groups_raw(base, [b"%d" % k for k in range(4096)]).changed) == 0
    with pytest.raises(kvgpu.KvgError):
        ctx.health_rescan_groups_raw(base, [b"%d" % k for k in range(4097)])
    mraw = MC.raw_of([(b"m%d" % k, {"type": b"t", "link": b"a/b/m", "numa_node": b"0\n"}) for k in range(3)])
    ctx.health_rescan_mdev_raw(mraw, [b"%d" % k for k in range(1024)])
    with pytest.raises(kvgpu.KvgError):
        ctx.health_rescan_mdev_raw(mraw, [b"%d" % k for k in range(1025)])
    assert len(ctx.health_rescan_groups_raw(base, [b"1"]).changed) == 0


def test_isolation_and_launches(ctx):
    rng = np.random.default_rng(5)
    ctx.pciids_load(gzip.open(os.path.join(conftest.ROOT, "tests", "golden", "pci.ids.gz"), "rb").read())
    ctx.health_rescan_groups_raw(RC.raw_of([])), ctx.health_rescan_mdev_raw(MC.raw_of([]))
    raw = RC.raw_of([pci_ok(k, b"%d" % (k % 3)) for k in range(30)])
    mraw = MC.raw_of(mdev_entries(rng, MC.canonical_names(rng, 20)))
    ref_g, ref_m = HR.RawGroupsRef(), HR.RawMdevRef()
    keyed_ref = health_keyed_ref.KeyedGroupsRef()
    krecs = decode_pci(raw, {})
    for t in range(4):
        nodes = [b"%d" % k for k in range(3) if (t + k) % 2]
        before = ctx.launch_count
        d = ctx.health_rescan_groups_raw(raw, nodes)
        assert ctx.launch_count - before == 1                       # a poll-loop tick: one kernel launch
        w = ref_g.step(raw, nodes)
        assert changed(d) == w.changed
        dm = ctx.health_rescan_mdev_raw(mraw, [BUS_POOL[t]])
        assert changed(dm) == ref_m.step(mraw, [BUS_POOL[t]]).changed
        # the other states, the raw scans and the raw deltas in between leave the raw lists alone, and are left alone
        g = [k for k in range(1, 4)]
        kd = ctx.health_rescan_groups_keyed(krecs, g)
        assert changed(kd) == [int(x) for x in keyed_ref.rescan(krecs, g).changed]
        ctx.health_rescan_groups(krecs, g)
        ctx.health_rescan(krecs)
        ctx.scan_pci_raw(raw)
        ctx.scan_pci_raw_delta(raw)
        ctx.scan_mdev_raw(mraw)
        ctx.scan_mdev_raw_delta(mraw)
