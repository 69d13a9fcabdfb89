"""kvg_scan_pci_raw_delta on the H100: over sequences of raw snapshots, *res and *snap against kvg_scan_pci_raw, every
delta against the string-level restatement raw_delta_ref.expect with each column (names, groups, devices) numeric on
one side and index on the other in both directions and all in index mode on both sides, fully numeric pairs byte for
byte against kvg_scan_pci_delta, 1 M numeric and 70 k index-mode entries, refusals that leave the slot unchanged, the
reset, the launch counts of the header, and isolation from the other deltas, scans, health and Allocate calls."""
import numpy as np
import pytest

import raw_delta_ref
import raw_scan_cases as RC
import util
import kvgpu
from kvgpu import _lib as L
from oracle import oracle as O

pytestmark = pytest.mark.gpu

SURVIVOR = {"vendor": b"0x10de\n", "driver": b"../vfio-pci", "iommu_group": b"../g/3", "numa_node": b"1\n",
            "device": b"0x1db6\n"}


@pytest.fixture(scope="module")
def ctxs():
    """the context under test, and one that runs kvg_scan_pci_delta on the decoded records in lockstep"""
    cs = [kvgpu.Context(0), kvgpu.Context(0)]
    for c in cs:
        c.pciids_load(util.pciids_text())
    yield cs
    for c in cs:
        c.close()


def same_result(a, b):
    for f in ("n_records", "name_pool"):
        assert getattr(a, f) == getattr(b, f), f
    for f in ("survivors", "dev_keys", "dev_off", "dev_perm", "dev_name_slot", "grp_keys", "grp_off", "grp_perm"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def numeric(snap):
    return snap.packed_addr and snap.group_names is None and snap.device_names is None


class Walker:
    """Feeds a sequence of raw snapshots to both contexts and checks each step."""

    def __init__(self, ctxs, reset=True):
        self.ctx, self.ref = ctxs
        if reset:
            self.ctx.scan_pci_raw_delta_reset()
            self.ref.scan_pci_delta_reset()
        self.prev = None   # (side, snapshot)

    def step(self, raw, string_ref=True):
        want_res, want_snap = self.ctx.scan_pci_raw(raw)   # also the first scan after a table load, which joins more
        c0 = self.ctx.launch_count
        res, snap, delta = self.ctx.scan_pci_raw_delta(raw)
        c1 = self.ctx.launch_count
        self.ctx.scan_pci_raw(raw)
        c2 = self.ctx.launch_count
        same_result(res, want_res)
        assert snap.recs.tobytes() == want_snap.recs.tobytes()
        assert (snap.packed_addr, snap.group_names, snap.device_names) == \
            (want_snap.packed_addr, want_snap.group_names, want_snap.device_names)
        both = numeric(snap) and (self.prev is None or numeric(self.prev[1]))
        assert c1 - c0 == c2 - c1 + (2 if both else 4), (c0, c1, c2, both)
        ref_res, ref_delta = self.ref.scan_pci_delta(snap.recs)
        if both:
            for f in ("changes", "dev_dirty", "dev_gone", "grp_dirty", "grp_gone"):
                assert getattr(delta, f).tobytes() == getattr(ref_delta, f).tobytes(), f
        side = raw_delta_ref.side_of(res, snap)
        prev_side = self.prev[0] if self.prev else raw_delta_ref.empty_side()
        assert delta.n_prev == len(prev_side["names"])
        if string_ref:
            want = raw_delta_ref.expect(prev_side, side)
            for f in ("changes", "dev_dirty", "dev_gone", "grp_dirty", "grp_gone"):
                assert np.array_equal(getattr(delta, f), want[f]), (f, getattr(delta, f)[:6], want[f][:6])
        self.prev = (side, snap)
        return res, snap, delta


def bump(name: bytes) -> bytes:
    return kvgpu.format_bdf(kvgpu.parse_bdf(name.decode()) + 1).encode()


def mutate(rng, entries, k):
    """k random hot-adds, removals, regroups, device changes and NUMA moves on canonical, ascending entries"""
    out = [(n, dict(e)) for n, e in entries]
    for _ in range(k):
        i = int(rng.integers(len(out)))
        n, e = out[i]
        op = int(rng.integers(5))
        if op == 0:
            e["iommu_group"] = b"../g/%d" % rng.integers(0, 64)
        elif op == 1:
            e["device"] = RC.DEVICES[rng.integers(3)]
        elif op == 2:
            e["numa_node"] = b"%d\n" % rng.integers(0, 4)
        elif op == 3 and len(out) > 1:
            del out[i]
        else:
            nn = bump(n)
            if kvgpu.parse_bdf(nn.decode()) is not None and (i + 1 == len(out) or nn < out[i + 1][0]):
                out.insert(i + 1, (nn, dict(SURVIVOR, iommu_group=b"../g/%d" % rng.integers(0, 64))))
    return out


def in_modes(entries, modes, rng):
    """the same entries with the listed columns forced into index mode: a non-canonical name appended, one group
    written with a leading zero, one device id in upper case"""
    out = [(n, dict(e)) for n, e in entries]
    if "group" in modes:
        out[int(rng.integers(len(out)))][1]["iommu_group"] = b"../g/042"
    if "device" in modes:
        out[int(rng.integers(len(out)))][1]["device"] = b"0x1DB6\n"
    if "name" in modes:
        out.append((b"zz-not-a-bdf", dict(SURVIVOR)))
    return out


ALL = ("name", "group", "device")
SEQUENCE = [(), ("name",), (), ("group",), (), ("device",), (), ALL, ALL, (), ("name", "device"), ("group",)]


@pytest.mark.parametrize("n", [40, 3000])
def test_sequence_through_every_mode_pair(ctxs, n):
    rng = np.random.default_rng(n)
    cur = [(nm, dict(SURVIVOR, iommu_group=b"../g/%d" % rng.integers(0, 64), device=RC.DEVICES[rng.integers(3)],
                     numa_node=b"%d\n" % rng.integers(0, 4)) if rng.random() < 0.8 else
            dict(e, numa_node=e["numa_node"] and b"0\n"))   # other entries as generated, without numa_node range errors
           for nm, e in RC.gen_entries(rng, n, modes=(True, True))]
    w = Walker(ctxs)
    for modes in SEQUENCE:
        cur = mutate(rng, cur, max(1, n // 100))
        w.step(RC.raw_of(in_modes(cur, modes, rng)))


def test_random_entries_any_mode(ctxs):
    """gen_entries' own mix (non-canonical groups and devices), names sorted so that survivors ascend"""
    rng = np.random.default_rng(11)
    w = Walker(ctxs)
    for step in range(4):
        ent = sorted(((n, dict(e, numa_node=e["numa_node"] and b"1\n")) for n, e in
                      RC.gen_entries(rng, 2000, names="mixed")), key=lambda x: x[0])   # no numa_node range error
        dedup = [x for k, x in enumerate(ent) if k == 0 or x[0] != ent[k - 1][0]]
        w.step(RC.raw_of(dedup))


def test_one_million_numeric(ctxs):
    recs = O.gen_pci(0, 1_000_000, O.nv_ids(util.pciids_text()), 16)
    w = Walker(ctxs)
    w.step(RC.render_records(recs), string_ref=False)
    rng = np.random.default_rng(12)
    nxt = recs.copy()
    sel = rng.choice(len(nxt), 1000, replace=False)
    nxt["numa"][sel[:500]] ^= 1
    nxt["iommu_group"][sel[500:]] += 7
    nxt = np.delete(nxt, rng.choice(len(nxt), 500, replace=False))
    res, snap, delta = w.step(RC.render_records(nxt), string_ref=False)
    assert numeric(snap) and len(delta.changes) > 0


def test_seventy_thousand_index_mode(ctxs):
    rng = np.random.default_rng(13)
    cur = [(nm, dict(SURVIVOR, iommu_group=b"../g/%d" % rng.integers(0, 5000), device=RC.DEVICES[rng.integers(3)]))
           for nm, _ in RC.gen_entries(rng, 72_000, modes=(True, True))]
    w = Walker(ctxs)
    w.step(RC.raw_of(in_modes(cur, ALL, rng)))
    front = kvgpu.format_bdf(0).encode()
    assert front < cur[0][0]
    nxt = [(front, dict(SURVIVOR, iommu_group=b"../g/new"))] + mutate(rng, cur, 70)
    res, snap, delta = w.step(RC.raw_of(in_modes(nxt, ALL, rng)))
    assert not snap.packed_addr and len(res.survivors) > 70_000
    assert delta.changes[0]["what"] == L.CH_ADDED and delta.changes[0]["addr"] == 0
    assert len(delta.changes) < 200


def test_refusals_leave_the_slot_and_reset_works(ctxs):
    ctx = ctxs[0]
    rng = np.random.default_rng(14)
    cur = [(nm, dict(SURVIVOR)) for nm, _ in RC.gen_entries(rng, 300, modes=(True, True))]
    w = Walker(ctxs)
    w.step(RC.raw_of(in_modes(cur, ("group",), rng)))
    descending = [cur[1], cur[0]] + cur[2:]
    with pytest.raises(L.KvgError) as e:
        ctx.scan_pci_raw_delta(RC.raw_of(descending))
    assert e.value.rc == L.KVG_EINVAL and "names" in str(e.value)
    duplicate = [cur[0], (cur[0][0], dict(SURVIVOR))] + cur[1:]
    with pytest.raises(L.KvgError):
        ctx.scan_pci_raw_delta(RC.raw_of(duplicate))
    with pytest.raises(kvgpu.ReferencePanic):
        ctx.scan_pci_raw_delta(RC.raw_of([(cur[0][0], dict(SURVIVOR, vendor=b"0"))]))
    prev_snap = w.prev[1]
    res, snap, delta = ctx.scan_pci_raw_delta(RC.raw_of([(n, e) for n, e in in_modes(cur, (), rng)]))
    assert delta.n_prev == len(w.prev[0]["names"]) and prev_snap.group_names is not None
    assert len(delta.changes) == 1 and delta.changes[0]["what"] == L.CH_GROUP   # the one "042" group is "3" again
    ctx.scan_pci_raw_delta_reset()
    res, snap, delta = ctx.scan_pci_raw_delta(RC.raw_of(cur))
    assert delta.n_prev == 0 and (delta.changes["what"] == L.CH_ADDED).all()
    assert len(delta.dev_dirty) == len(res.dev_keys) and len(delta.grp_gone) == 0


def test_isolation(ctxs):
    """other deltas, scans and health calls between two calls leave this slot alone, and this call theirs"""
    ctx = ctxs[0]
    rng = np.random.default_rng(15)
    cur = [(nm, dict(SURVIVOR, iommu_group=b"../g/%d" % rng.integers(0, 64))) for nm, _ in
           RC.gen_entries(rng, 500, modes=(True, True))]
    raw = RC.raw_of(in_modes(cur, ("name", "device"), rng))
    ctx.scan_pci_raw_delta_reset()
    ctx.scan_pci_raw_delta(raw)
    recs = O.gen_pci(0, 5000, O.nv_ids(util.pciids_text()), 16)
    ctx.scan_pci_delta_reset()
    ctx.scan_pci_delta(recs)
    mrecs, types = O.gen_mdev(0, 512), O.gen_type_names(16)
    ctx.scan_mdev_delta_reset()
    ctx.scan_mdev_delta(mrecs, types)
    ctx.health_rescan(recs)
    ctx.pci_group_check(recs[:64], recs["iommu_group"][:64])   # an Allocate re-check
    ctx.scan_pci_raw(RC.raw_of(cur[:10]))
    ctx.scan_pci(recs[:100])
    _, _, d = ctx.scan_pci_raw_delta(raw)
    assert d.n_prev > 0 and len(d.changes) == 0 and len(d.dev_dirty) == 0 and len(d.grp_dirty) == 0
    _, d = ctx.scan_pci_delta(recs)
    assert d.n_prev > 0 and len(d.changes) == 0
    _, d = ctx.scan_mdev_delta(mrecs, types)
    assert d.n_prev > 0 and len(d.changes) == 0
    assert len(ctx.health_rescan(recs).changed) == 0
