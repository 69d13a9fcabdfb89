"""The sharded re-scan delta (k_delta_merge_shard -> k_delta_lists, kvg_dev_scan_pci_shard_fetch_delta), executed on
the CPU from its real kernel source under the warp emulator of tools/emu/, one call per rank, against the exact
restatement delta_ref.expect_pci_delta.  P ranks hold contiguous shards of the global survivor list (shard boundaries
move between steps, one shard is empty); rank r owns the keys with key % P == r, with all their members in Walk
order.  Per rank and step the local changes, the owned key lists and the patched map part are checked; over all
ranks merge_pci_shard_deltas must give exactly the delta of the whole snapshot."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import delta_ref

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

NONE = 0xFFFFFFFF
KINDS = ("hot_add", "hot_remove", "rebind", "regroup", "device", "numa")


class Rank:
    """One rank's library state: the tag words and the previous result (local list, both owned lists)."""

    def __init__(self, lib):
        self.lib = lib
        self.cap = 1 << 14
        self.flags = np.zeros(4 * self.cap, dtype=np.uint32)
        self.tag = 100
        self.prev = [np.zeros(0, kvgpu.PCI_SURV)] * 3

    def run(self, lists):
        """lists: [local, owned by device id, owned by group] now.  Returns the delta dict (or None on the ascent
        error; the previous result is then kept)."""
        prev = self.prev
        keys = [np.unique(lists[1]["device"]), np.unique(prev[1]["device"]),
                np.unique(lists[2]["iommu_group"]), np.unique(prev[2]["iommu_group"])]
        keys = [np.concatenate([k.astype(np.uint32), np.zeros(1, np.uint32)]) for k in keys]  # never empty
        kp = (C.c_void_p * 4)(*[k.ctypes.data for k in keys])
        nk = np.array([len(k) - 1 for k in keys], dtype=np.uint32)
        assert nk.max() <= self.cap
        pad = lambda a: np.ascontiguousarray(a) if len(a) else np.zeros(1, kvgpu.PCI_SURV)
        P, N = [pad(a) for a in prev], [pad(a) for a in lists]
        pp = (C.c_void_p * 3)(*[a.ctypes.data for a in P])
        npp = (C.c_void_p * 3)(*[a.ctypes.data for a in N])
        n_prev = np.array([len(a) for a in prev], dtype=np.uint32)
        n_now = np.array([len(a) for a in lists], dtype=np.uint32)
        ch = np.zeros(len(prev[0]) + len(lists[0]) + 1, dtype=kvgpu.PCI_CHANGE)
        out = [np.zeros(int(nk[0]) + 1, np.uint32), np.zeros(int(nk[1]) + 1, np.uint16),
               np.zeros(int(nk[2]) + 1, np.uint32), np.zeros(int(nk[3]) + 1, np.uint32)]
        counts = np.zeros(6, dtype=np.uint32)
        self.tag += 2
        assert self.lib.emu_shard_delta(pp, n_prev.ctypes.data, npp, n_now.ctypes.data, kp, nk.ctypes.data,
                                        self.flags.ctypes.data, self.cap, self.tag, ch.ctypes.data,
                                        *[x.ctypes.data for x in out], counts.ctypes.data) == 0
        if counts[1]:
            return None
        self.prev = [a.copy() for a in lists]
        return SimpleNamespace(n_prev=len(prev[0]), changes=ch[:counts[0]], dev_dirty=out[0][:counts[2]],
                               dev_gone=out[1][:counts[3]], grp_dirty=out[2][:counts[4]], grp_gone=out[3][:counts[5]])


@pytest.fixture(scope="module")
def lib():
    L = C.CDLL(emu_build.build_delta())
    L.emu_shard_delta.argtypes = [C.c_void_p] * 7 + [C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
    return L


def surv(addr, rng, n_dev=40, n_grp=300):
    s = np.zeros(len(addr), dtype=kvgpu.PCI_SURV)
    s["addr"] = addr
    s["iommu_group"] = rng.integers(0, n_grp, len(addr))
    s["device"] = rng.integers(0x1000, 0x1000 + n_dev, len(addr))
    s["numa"] = rng.integers(0, 4, len(addr))
    s["name_slot"] = kvgpu.KVG_NO_NAME
    return s


def step(cur, kind, rng):
    """One snapshot later, on the survivor list: about 1 % of the survivors hot-added, hot-removed, re-bound (no
    longer advertised), regrouped, re-identified or moved to another NUMA node."""
    nxt = cur.copy()
    k = max(1, len(nxt) // 100)
    pick = rng.choice(len(nxt), min(k, len(nxt)), replace=False)
    if kind == "hot_add":
        cand = np.setdiff1d(rng.choice(1 << 22, 4 * k, replace=False).astype(np.uint32), nxt["addr"])[:k]
        return np.sort(np.concatenate([nxt, surv(cand, rng, n_dev=48, n_grp=340)]), order="addr", kind="stable")
    if kind in ("hot_remove", "rebind"):
        return np.delete(nxt, pick)
    if kind == "regroup":
        nxt["iommu_group"][pick] = rng.integers(0, 340, len(pick))
    elif kind == "device":
        nxt["device"][pick] = rng.integers(0x1000, 0x1000 + 48, len(pick))
    else:
        nxt["numa"][pick] = (nxt["numa"][pick] + 1) % 4
    return nxt


def shard_bounds(n, P, rng, empty):
    """P contiguous shards of n survivors with random boundaries; shard `empty` (if any) holds nothing."""
    cuts = np.sort(rng.integers(0, n + 1, P - 1))
    b = np.concatenate([[0], cuts, [n]])
    if empty is not None and empty + 1 < P:
        b[empty + 1] = b[empty]
        b = np.maximum.accumulate(b)
    elif empty is not None:
        b[empty] = n
    return [(int(b[r]), int(b[r + 1])) for r in range(P)]


def owned(all_surv, P, r):
    return [all_surv[all_surv["device"] % P == r], all_surv[all_surv["iommu_group"] % P == r]]


def by_key(members, field):
    """A PciResult over `members` grouped by `field`, as the owned orderings of the sharded fetch build it."""
    keys = np.unique(members[field])
    perm = np.argsort(members[field], kind="stable").astype(np.uint32)
    off = np.searchsorted(members[field][perm], keys).astype(np.uint32)
    off = np.concatenate([off, [len(members)]]).astype(np.uint32)
    e32, e16, z32 = np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(1, np.uint32)
    if field == "device":
        return kvgpu.PciResult(0, members, keys.astype(np.uint16), off, perm,
                               np.full(len(keys), kvgpu.KVG_NO_NAME, np.uint32), e32, z32, e32, b"")
    return kvgpu.PciResult(0, members, e16, z32, e32, e32, keys.astype(np.uint32), off, perm, b"")


def shard_result(local, own):
    return kvgpu.PciShardResult(0, local, by_key(own[0], "device"), by_key(own[1], "iommu_group"))


def restricted(want, P, r, own):
    """The global key lists of expect_pci_delta restricted to the keys rank r owns, dirty keys re-indexed into the
    rank's owned keys."""
    now_dev, now_grp = np.unique(want["now_all"]["device"]), np.unique(want["now_all"]["iommu_group"])
    my_dev, my_grp = np.unique(own[0]["device"]), np.unique(own[1]["iommu_group"])
    dd = now_dev[want["dev_dirty"]]
    gd = now_grp[want["grp_dirty"]]
    dd, gd = dd[dd % P == r], gd[gd % P == r]
    return dict(dev_dirty=np.searchsorted(my_dev, dd).astype(np.uint32),
                dev_gone=want["dev_gone"][want["dev_gone"] % P == r],
                grp_dirty=np.searchsorted(my_grp, gd).astype(np.uint32),
                grp_gone=want["grp_gone"][want["grp_gone"] % P == r])


def run_sequence(lib, P, seed, n0=3000, steps=12):
    rng = np.random.default_rng(seed)
    ranks = [Rank(lib) for _ in range(P)]
    cur = surv(np.sort(rng.choice(1 << 22, n0, replace=False)).astype(np.uint32), rng)
    prev_all = cur[:0]
    parts_maps = [kvgpu.Maps() for _ in range(P)]
    crossed = 0
    prev_owner = {}
    for s in range(steps):
        if s:
            cur = step(cur, KINDS[(s - 1) % len(KINDS)], rng)
        empty = (s * 7) % P if P > 1 and s % 3 == 1 else None
        bounds = shard_bounds(len(cur), P, rng, empty)
        want = delta_ref.expect_pci_delta(prev_all, cur, kvgpu.PCI_CHANGE)
        want["now_all"] = cur
        summaries = []
        owner = {}
        for r in range(P):
            lo, hi = bounds[r]
            local, own = cur[lo:hi], owned(cur, P, r)
            for a in local["addr"]:
                owner[int(a)] = r
            prev_local = ranks[r].prev[0]
            got = ranks[r].run([local] + own)
            assert got is not None, "ascent error on ascending lists"
            loc = delta_ref.expect_pci_delta(prev_local, local, kvgpu.PCI_CHANGE)
            assert got.n_prev == len(prev_local)
            assert np.array_equal(got.changes, loc["changes"]), (P, s, r)
            exp = restricted(want, P, r, own)
            for f in ("dev_dirty", "dev_gone", "grp_dirty", "grp_gone"):
                assert np.array_equal(getattr(got, f), exp[f]), (P, s, r, f)
            res = shard_result(local, own)
            kvgpu.apply_pci_shard_delta(parts_maps[r], res, got)
            assert kvgpu.canonical_dump(parts_maps[r]) == kvgpu.canonical_dump(kvgpu.pci_maps_from_shard(res))
            summaries.append(kvgpu.shard_delta_part(res, got))
        crossed += sum(1 for a, r in owner.items() if a in prev_owner and prev_owner[a] != r)
        prev_owner = owner
        m = kvgpu.merge_pci_shard_deltas(summaries)
        assert m.n_prev == len(prev_all) and m.n_now == len(cur)
        assert m.changes.tobytes() == want["changes"].tobytes(), (P, s)
        assert np.array_equal(m.dev_dirty, np.unique(cur["device"])[want["dev_dirty"]].astype(np.uint16))
        assert np.array_equal(m.grp_dirty, np.unique(cur["iommu_group"])[want["grp_dirty"]])
        assert np.array_equal(m.dev_gone, want["dev_gone"]) and np.array_equal(m.grp_gone, want["grp_gone"])
        full = kvgpu.merge_parts(parts_maps)
        fresh = kvgpu.merge_parts([kvgpu.pci_maps_from_shard(shard_result(cur[lo:hi], owned(cur, P, r)))
                                   for r, (lo, hi) in enumerate(bounds)])
        assert kvgpu.canonical_dump(full) == kvgpu.canonical_dump(fresh)
        prev_all = cur
    return crossed


@pytest.mark.parametrize("P", [1, 2, 3, 8, 16])
def test_snapshot_sequence_per_rank_and_merged(lib, P):
    crossed = run_sequence(lib, P, seed=P)
    assert P == 1 or crossed > 0, "no address crossed a shard boundary"


def test_owned_lists_longer_than_one_merge_tile(lib):
    """Owned lists of several tiles (P = 2: each about half the survivors), local lists of a few."""
    run_sequence(lib, 2, seed=11, n0=9000, steps=7)


def test_first_call_reports_everything_added(lib):
    rng = np.random.default_rng(3)
    cur = surv(np.arange(0, 8000, 4, dtype=np.uint32), rng)
    rk = Rank(lib)
    own = owned(cur, 3, 1)
    got = rk.run([cur[500:1500]] + own)
    assert got.n_prev == 0 and (got.changes["what"] == delta_ref.CH_ADDED).all() and len(got.changes) == 1000
    assert np.array_equal(got.dev_dirty, np.arange(len(np.unique(own[0]["device"]))))
    assert np.array_equal(got.grp_dirty, np.arange(len(np.unique(own[1]["iommu_group"]))))
    assert len(got.dev_gone) == 0 and len(got.grp_gone) == 0
    again = rk.run([cur[500:1500]] + own)
    assert len(again.changes) == 0 and len(again.dev_dirty) == 0 and len(again.grp_dirty) == 0


@pytest.mark.parametrize("which", [0, 1, 2])
@pytest.mark.parametrize("where", [1, 1023, 1500])
def test_non_ascending_list_sets_the_error_word(lib, which, where):
    """A repeated or swapped address in the local list or either owned list is refused, and the previous result
    stays as it was."""
    rng = np.random.default_rng(6)
    cur = surv(np.arange(0, 4 * 4000, 4, dtype=np.uint32), rng)
    cur["device"], cur["iommu_group"] = 0x1000, 0                      # one key each: owned lists = cur
    rk = Rank(lib)
    assert rk.run([cur[:2000], cur, cur]) is not None
    kept = [a.copy() for a in rk.prev]
    for bad_kind in ("repeat", "swap"):
        lists = [cur[:2000].copy(), cur.copy(), cur.copy()]
        a = lists[which]["addr"]
        if bad_kind == "repeat":
            a[where] = a[where - 1]
        else:
            a[where], a[where - 1] = a[where - 1], a[where]
        assert rk.run(lists) is None, (which, where, bad_kind)
        assert all(np.array_equal(x, y) for x, y in zip(rk.prev, kept))
    nxt = step(cur, "numa", rng)
    got = rk.run([nxt[:2000], nxt, nxt])
    assert np.array_equal(got.changes, delta_ref.expect_pci_delta(cur[:2000], nxt[:2000], kvgpu.PCI_CHANGE)["changes"])


def test_merge_fuses_a_boundary_crossing_and_drops_an_unchanged_one():
    """Two addresses cross from rank 0 to rank 1: one unchanged (no entry), one regrouped (one GROUP entry with the
    global indices of both sides)."""
    rng = np.random.default_rng(9)
    a = surv(np.arange(10, 20, dtype=np.uint32), rng)
    b = a.copy()
    b["iommu_group"][6] += 1000
    old_parts, new_parts = [a[:7], a[7:]], [b[:5], b[5:]]
    want = delta_ref.expect_pci_delta(a, b, kvgpu.PCI_CHANGE)
    summ = []
    for r in range(2):
        d = delta_ref.expect_pci_delta(old_parts[r], new_parts[r], kvgpu.PCI_CHANGE)
        summ.append(kvgpu.PciShardDelta(len(old_parts[r]), len(new_parts[r]), d["changes"], np.zeros(0, np.uint16),
                                        np.zeros(0, np.uint16), np.zeros(0, np.uint32), np.zeros(0, np.uint32)))
    m = kvgpu.merge_pci_shard_deltas(summ)
    assert len(m.changes) == 1 and m.changes["what"][0] == delta_ref.CH_GROUP
    assert m.changes["prev_index"][0] == 6 and m.changes["now_index"][0] == 6
    assert m.changes.tobytes() == want["changes"].tobytes()
