"""kvg_scan_mdev_raw_delta on the H100: over sequences of raw mdev snapshots (mdev_raw_cases.gen_entries with creates,
destroys, retypes, parent moves and NUMA moves), *res and *snap against kvg_scan_mdev_raw, every delta against a
string-level restatement keyed by entry name (UUID string, sanitised type label, decoded parent string), with names
and parents numeric on one side and index on the other in both directions and both in index mode, fully numeric
pairs byte for byte against kvg_scan_mdev_delta, launch counts, refusals, the reset, and isolation."""
import numpy as np
import pytest

import mdev_raw_cases as MC
import util
import kvgpu
from kvgpu import _lib as L
from oracle import oracle as O

pytestmark = pytest.mark.gpu
NO_INDEX = 0xFFFFFFFF


@pytest.fixture(scope="module")
def ctxs():
    cs = [kvgpu.Context(0), kvgpu.Context(0)]
    for c in cs:
        c.pciids_load(util.pciids_text())
    yield cs
    for c in cs:
        c.close()


def numeric(snap):
    return snap.uuid_ok and snap.parent_names is None


def side_of(res, snap):
    """every survivor's strings: name, sanitised label, parent string, and its handles"""
    s = res.survivors
    names = [kvgpu.format_uuid(u).encode() if snap.uuid_ok else snap.names[int(i)].encode("latin-1")
             for u, i in zip(s["uuid"], s["src"])]
    parents = [kvgpu.format_bdf(int(p)).encode() if snap.parent_names is None else
               snap.parent_names[int(p)].encode("latin-1") for p in s["parent"]]
    return dict(names=names, labels=[res.labels[int(t)] for t in s["type_key"]], parents=parents,
                numa=[int(x) for x in s["numa"]], surv=s, type_keys=list(res.type_keys), labels_all=res.labels,
                par_keys=[int(p) for p in res.par_keys],
                par_str={int(p): kvgpu.format_bdf(int(p)).encode() if snap.parent_names is None else
                         snap.parent_names[int(p)].encode("latin-1") for p in res.par_keys})


def empty_side():
    return dict(names=[], labels=[], parents=[], numa=[], surv=np.zeros(0, L.MDEV_SURV), type_keys=[],
                labels_all=[], par_keys=[], par_str={})


def expect(prev, now):
    """kvgpu.h kvg_scan_mdev_raw_delta restated on strings"""
    P = {n: i for i, n in enumerate(prev["names"])}
    N = {n: i for i, n in enumerate(now["names"])}
    rows = []
    for name in sorted(set(P) | set(N)):
        i, j = P.get(name), N.get(name)
        if i is None:
            what = L.CH_ADDED
        elif j is None:
            what = L.CH_REMOVED
        else:
            what = ((prev["labels"][i] != now["labels"][j]) * L.CH_TYPE |
                    (prev["parents"][i] != now["parents"][j]) * L.CH_PARENT |
                    (prev["numa"][i] != now["numa"][j]) * L.CH_NUMA)
        if not what:
            continue
        r = np.zeros(1, L.MDEV_CHANGE)[0]
        r["uuid"] = (now["surv"][j] if j is not None else prev["surv"][i])["uuid"]
        r["what"] = what
        for tag, side, k in (("prev", prev, i), ("now", now, j)):
            if k is not None:
                r[tag + "_parent"] = side["surv"][k]["parent"]
                r[tag + "_type"] = side["surv"][k]["type_key"]
                r[tag + "_numa"] = side["surv"][k]["numa"]
            r[tag + "_index"] = NO_INDEX if k is None else k
        rows.append(r)
    changes = np.array(rows, dtype=L.MDEV_CHANGE) if rows else np.zeros(0, L.MDEV_CHANGE)

    def members(side, col, key, with_numa):
        return [(n, m) if with_numa else n for n, c, m in zip(side["names"], side[col], side["numa"]) if c == key]

    type_dirty = [k for k, t in enumerate(now["type_keys"])
                  if members(now, "labels", now["labels_all"][int(t)], True) !=
                  members(prev, "labels", now["labels_all"][int(t)], True)]
    now_labels = {now["labels_all"][int(t)] for t in now["type_keys"]}
    type_gone = [prev["labels_all"][int(t)] for t in prev["type_keys"] if prev["labels_all"][int(t)] not in now_labels]
    par_dirty = [k for k, p in enumerate(now["par_keys"])
                 if members(now, "parents", now["par_str"][p], False) != members(prev, "parents", now["par_str"][p], False)]
    now_par = set(now["par_str"].values())
    par_gone = [p for p in prev["par_keys"] if prev["par_str"][p] not in now_par]
    return dict(changes=changes, type_dirty=np.array(type_dirty, np.uint32), type_gone=type_gone,
                par_dirty=np.array(par_dirty, np.uint32), par_gone=np.array(par_gone, np.uint32))


class Walker:
    def __init__(self, ctxs):
        self.ctx, self.ref = ctxs
        self.ctx.scan_mdev_raw_delta_reset()
        self.ref.scan_mdev_delta_reset()
        self.prev = None

    def step(self, raw, string_ref=True):
        want_res, want_snap = self.ctx.scan_mdev_raw(raw)
        c0 = self.ctx.launch_count
        res, snap, delta = self.ctx.scan_mdev_raw_delta(raw)
        c1 = self.ctx.launch_count
        self.ctx.scan_mdev_raw(raw)
        c2 = self.ctx.launch_count
        assert res.survivors.tobytes() == want_res.survivors.tobytes()
        assert snap.recs.tobytes() == want_snap.recs.tobytes() and snap.raw_types == want_snap.raw_types
        assert (snap.uuid_ok, snap.parent_names) == (want_snap.uuid_ok, want_snap.parent_names)
        both = numeric(snap) and (self.prev is None or numeric(self.prev[1]))
        assert c1 - c0 == c2 - c1 + (3 if both else 5), (c0, c1, c2, both)
        _, ref_delta = self.ref.scan_mdev_delta(snap.recs, snap.raw_types)
        if both:
            for f in ("changes", "type_dirty", "par_dirty", "par_gone"):
                assert getattr(delta, f).tobytes() == getattr(ref_delta, f).tobytes(), f
            assert delta.type_gone == ref_delta.type_gone
        side = side_of(res, snap)
        if string_ref:
            want = expect(self.prev[0] if self.prev else empty_side(), side)
            for f in ("changes", "type_dirty", "par_dirty", "par_gone"):
                assert np.array_equal(getattr(delta, f), want[f]), (f, getattr(delta, f)[:4], want[f][:4])
            assert delta.type_gone == want["type_gone"]
        self.prev = (side, snap)
        return res, snap, delta


def entry(rng, name, parent=None):
    p = parent or kvgpu.format_bdf(int(rng.integers(16)) << 8).encode()
    return (name, {"type": b"GRID T4-%dQ\n" % rng.integers(6), "link": MC.link_to(p, name),
                   "numa_node": b"%d\n" % rng.integers(0, 3)})


def mutate(rng, entries, k):
    out = [(n, dict(e)) for n, e in entries]
    for _ in range(k):
        i = int(rng.integers(len(out)))
        n, e = out[i]
        op = int(rng.integers(5))
        if op == 0:
            e["type"] = b"GRID T4-%dQ\n" % rng.integers(8)
        elif op == 1:
            e["link"] = MC.link_to(kvgpu.format_bdf(int(rng.integers(20)) << 8).encode(), n)
        elif op == 2:
            e["numa_node"] = b"%d\n" % rng.integers(0, 3)
        elif op == 3 and len(out) > 1:
            del out[i]
        else:
            nn = (n[:-1] + b"%x" % ((int(n[-1:], 16) + 1) % 16))
            if nn > n and (i + 1 == len(out) or nn < out[i + 1][0]):
                out.insert(i + 1, entry(rng, nn))
    return out


def in_modes(entries, modes, rng):
    """names: an entry named "zz-not-a-uuid" appended; parents: one parent written as a non-BDF directory"""
    out = [(n, dict(e)) for n, e in entries]
    if "parent" in modes:
        k = int(rng.integers(len(out)))
        out[k][1]["link"] = MC.link_to(b"gpu-a", out[k][0])
    if "name" in modes:
        out.append(entry(rng, b"zz-not-a-uuid"))
    return out


ALL = ("name", "parent")
SEQUENCE = [(), ("name",), (), ("parent",), (), ALL, ALL, (), ("parent",), ("name",)]


@pytest.mark.parametrize("n", [30, 3000])
def test_sequence_through_every_mode_pair(ctxs, n):
    rng = np.random.default_rng(n + 1)
    cur = [entry(rng, nm) for nm in MC.canonical_names(rng, n)]
    w = Walker(ctxs)
    for modes in SEQUENCE:
        cur = mutate(rng, cur, max(1, n // 100))
        w.step(MC.raw_of(in_modes(cur, modes, rng)))


def test_gen_entries_mixed_parents(ctxs):
    """gen_entries' own parents (empty and newline-wrapped ones among them), names canonical"""
    rng = np.random.default_rng(7)
    w = Walker(ctxs)
    for _ in range(3):
        ent = [(n, dict(e, numa_node=e["numa_node"] and b"1\n"))
               for n, e in MC.gen_entries(rng, 2000, parents="mixed")]
        w.step(MC.raw_of(ent))


def test_seventy_thousand_index_mode(ctxs):
    rng = np.random.default_rng(8)
    cur = [entry(rng, nm) for nm in MC.canonical_names(rng, 72_000)]
    w = Walker(ctxs)
    w.step(MC.raw_of(in_modes(cur, ALL, rng)))
    nxt = mutate(rng, cur, 70)
    res, snap, delta = w.step(MC.raw_of(in_modes(nxt, ALL, rng)))
    assert not snap.uuid_ok and snap.parent_names is not None and len(res.survivors) > 70_000
    assert len(delta.changes) < 200


def test_refusals_reset_and_isolation(ctxs):
    ctx = ctxs[0]
    rng = np.random.default_rng(9)
    cur = [entry(rng, nm) for nm in MC.canonical_names(rng, 300)]
    w = Walker(ctxs)
    raw = MC.raw_of(in_modes(cur, ("parent",), rng))
    w.step(raw)
    with pytest.raises(L.KvgError) as e:
        ctx.scan_mdev_raw_delta(MC.raw_of([cur[1], cur[0]] + cur[2:]))
    assert e.value.rc == L.KVG_EINVAL and "names" in str(e.value)
    with pytest.raises(kvgpu.ReferencePanic):
        ctx.scan_mdev_raw_delta(MC.raw_of([(cur[0][0], dict(cur[0][1], link=b"nolash"))]))
    # other calls between two calls: this slot unchanged, and theirs
    recs = O.gen_pci(0, 3000, O.nv_ids(util.pciids_text()), 16)
    ctx.scan_pci_delta_reset()
    ctx.scan_pci_delta(recs)
    mrecs, types = O.gen_mdev(0, 512), O.gen_type_names(16)
    ctx.scan_mdev_delta_reset()
    ctx.scan_mdev_delta(mrecs, types)
    ctx.scan_pci_raw_delta_reset()
    pci_raw = kvgpu.PciRaw(*_pci_raw_args())
    ctx.scan_pci_raw_delta(pci_raw)
    ctx.scan_mdev_raw(MC.raw_of(cur[:5]))
    _, _, d = ctx.scan_mdev_raw_delta(raw)
    assert d.n_prev == len(w.prev[0]["names"]) and len(d.changes) == 0 and len(d.par_dirty) == 0
    assert len(d.type_dirty) == 0
    assert len(ctx.scan_pci_delta(recs)[1].changes) == 0
    assert len(ctx.scan_mdev_delta(mrecs, types)[1].changes) == 0
    assert len(ctx.scan_pci_raw_delta(pci_raw)[2].changes) == 0
    ctx.scan_mdev_raw_delta_reset()
    res, _, d = ctx.scan_mdev_raw_delta(raw)
    assert d.n_prev == 0 and (d.changes["what"] == L.CH_ADDED).all() and len(d.par_dirty) == len(res.par_keys)


def _pci_raw_args():
    import raw_scan_cases as RC
    r = RC.raw_of([(kvgpu.format_bdf(k << 3).encode(), {"vendor": b"0x10de\n", "driver": b"../vfio-pci",
                                                         "iommu_group": b"../g/%d" % k, "numa_node": b"0\n",
                                                         "device": b"0x1db6\n"}) for k in range(1, 50)])
    return r.names, r.off, r.bytes, r.state
