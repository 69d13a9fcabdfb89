"""The sharded mdev re-scan delta (k_mdev_delta_types over whole dictionaries -> k_delta_merge_shard<MdevDeltaRec> ->
k_delta_lists, kvg_dev_scan_mdev_shard_fetch_delta), executed on the CPU from its real kernel source under the warp
emulator of tools/emu/, one call per rank, against the exact restatement mdev_delta_ref.expect_mdev_delta.  P ranks hold
contiguous shards of the global survivor list (shard boundaries move between steps, one shard is empty); rank r owns
the type ids with id % P == r and the parents with handle % P == r, with all their members in Walk order.  The
dictionary is reordered between some steps, so labels move between ranks.  Per rank and step the local changes, the
owned key lists and the patched map part are checked; over all ranks merge_mdev_shard_deltas must give exactly the
delta of the whole snapshot."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import mdev_delta_ref
from test_mdev_delta_emu import XMAP_SLOTS, Dictionary, EmuLabels, retype, surv, uuids
from test_shard_delta_emu import shard_bounds

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

KINDS = ("hot_add", "destroy", "retype", "reparent", "numa", "reorder")
# 20 labels, two of them under a second raw name (the label rule merges them)
RAW = [b"GRID T%02d\n" % k for k in range(20)] + [b"GRID  T03", b"GRID\tT11\n"]


def key16(s):
    return np.ascontiguousarray(s["uuid"]).view("V16").ravel()


class Rank:
    """One rank's library state: tag words, probe table and cross-map, and the previous result (local list, both owned
    lists, dictionary)."""

    def __init__(self, lib):
        self.lib = lib
        self.cap = 1 << 16
        self.flags = np.zeros(4 * self.cap, dtype=np.uint32)
        self.table = np.zeros(XMAP_SLOTS, dtype=np.uint64)
        self.xlate = np.zeros(1 << 16, dtype=np.uint32)
        self.tag = 100
        self.prev = [np.zeros(0, kvgpu.MDEV_SURV)] * 3
        self.dprev = Dictionary([])

    def run(self, lists, dnow):
        """lists: [local, owned by type id, owned by parent] now, dnow their dictionary.  Returns the delta (or None on
        the ascent error; the previous result is then kept)."""
        prev, dprev = self.prev, self.dprev
        keys = [np.unique(lists[1]["type_key"]), np.unique(prev[1]["type_key"]),
                np.unique(lists[2]["parent"]), np.unique(prev[2]["parent"])]
        keys = [np.concatenate([k.astype(np.uint32), np.zeros(1, np.uint32)]) for k in keys]   # never empty
        kp = (C.c_void_p * 4)(*[k.ctypes.data for k in keys])
        nk = np.array([len(k) - 1 for k in keys], dtype=np.uint32)
        canon = [np.concatenate([np.unique(d.canon).astype(np.uint32), np.zeros(1, np.uint32)]) for d in (dnow, dprev)]
        cp = (C.c_void_p * 2)(*[c.ctypes.data for c in canon])
        nc = np.array([len(c) - 1 for c in canon], dtype=np.uint32)
        lab = (EmuLabels * 2)(*[EmuLabels(d.bytes.ctypes.data, d.off.ctypes.data, d.len.ctypes.data,
                                          d.hash.ctypes.data) for d in (dnow, dprev)])
        pad = lambda a: np.ascontiguousarray(a) if len(a) else np.zeros(1, kvgpu.MDEV_SURV)
        P, N = [pad(a) for a in prev], [pad(a) for a in lists]
        pp = (C.c_void_p * 3)(*[a.ctypes.data for a in P])
        npp = (C.c_void_p * 3)(*[a.ctypes.data for a in N])
        n_prev = np.array([len(a) for a in prev], dtype=np.uint32)
        n_now = np.array([len(a) for a in lists], dtype=np.uint32)
        ch = np.zeros(len(prev[0]) + len(lists[0]) + 1, dtype=kvgpu.MDEV_CHANGE)
        out = [np.zeros(int(nk[k]) + 1, np.uint32) for k in range(4)]
        counts = np.zeros(6, dtype=np.uint32)
        self.tag += 2
        assert self.lib.emu_mdev_shard_delta(pp, n_prev.ctypes.data, npp, n_now.ctypes.data, kp, nk.ctypes.data, cp,
                                             nc.ctypes.data, lab, self.table.ctypes.data, self.xlate.ctypes.data,
                                             self.flags.ctypes.data, self.cap, self.tag, ch.ctypes.data,
                                             *[x.ctypes.data for x in out], counts.ctypes.data) == 0
        if counts[1]:
            return None
        self.prev, self.dprev = [a.copy() for a in lists], dnow
        return SimpleNamespace(n_prev=len(prev[0]), changes=ch[:counts[0]], type_dirty=out[0][:counts[2]],
                               type_gone=[dprev.labels[int(c)] for c in out[1][:counts[3]]],
                               par_dirty=out[2][:counts[4]], par_gone=out[3][:counts[5]])


@pytest.fixture(scope="module")
def lib():
    L = C.CDLL(emu_build.build_delta())
    L.emu_mdev_shard_delta.argtypes = [C.c_void_p] * 12 + [C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
    return L


def owned(all_surv, P, r):
    return [all_surv[all_surv["type_key"] % P == r], all_surv[all_surv["parent"] % P == r]]


def by_key(members, field, d):
    """An MdevResult over `members` grouped by `field`, as the owned orderings of the sharded fetch build it."""
    keys = np.unique(members[field])
    perm = np.argsort(members[field], kind="stable").astype(np.uint32)
    off = np.concatenate([np.searchsorted(members[field][perm], keys), [len(members)]]).astype(np.uint32)
    e32, e16, z32 = np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(1, np.uint32)
    names = ["name of " + lb.decode("latin-1") for lb in d.labels]
    if field == "type_key":
        return kvgpu.MdevResult(0, members, keys.astype(np.uint16), off, perm, d.labels, d.canon, names, e32, z32, e32)
    return kvgpu.MdevResult(0, members, e16, z32, e32, d.labels, d.canon, names, keys.astype(np.uint32), off, perm)


def shard_result(local, own, d):
    return kvgpu.MdevShardResult(0, local, by_key(own[0], "type_key", d), by_key(own[1], "parent", d))


def step(cur, d, raw, kind, rng):
    """One snapshot later, on the survivor list: about 1 % of the mdevs created, destroyed, retyped, moved to another
    parent or NUMA node, or the dictionary reordered (the same labels under other canonical ids)."""
    nxt = cur.copy()
    k = max(1, len(nxt) // 100)
    pick = rng.choice(len(nxt), min(k, len(nxt)), replace=False)
    if kind == "hot_add":
        add = surv(uuids(rng, 3 * k), d, rng)
        add = add[~np.isin(key16(add), key16(nxt))][:k]
        both = np.concatenate([nxt, add])
        return both[np.argsort(key16(both), kind="stable")], d, raw
    if kind == "destroy":
        return np.delete(nxt, pick), d, raw
    if kind == "retype":
        nxt["type_key"][pick] = d.canon[rng.integers(0, len(d.labels), len(pick))]
    elif kind == "reparent":
        nxt["parent"][pick] = rng.integers(0, 40, len(pick)) * 8 + 1
    elif kind == "numa":
        nxt["numa"][pick] = (nxt["numa"][pick] + 1) % 4
    else:
        raw = [raw[i] for i in rng.permutation(len(raw))]
        dn = Dictionary(raw)
        return retype(nxt, d, dn), dn, raw
    return nxt, d, raw


def check_rank(got, prev_lists, lists, dprev, dnow):
    """One rank's delta: local changes, and the four key lists of its owned lists."""
    exp = lambda a, b: mdev_delta_ref.expect_mdev_delta(a, b, dprev.labels, dnow.labels, kvgpu.MDEV_CHANGE)
    loc, by_type, by_par = exp(prev_lists[0], lists[0]), exp(prev_lists[1], lists[1]), exp(prev_lists[2], lists[2])
    assert got.n_prev == len(prev_lists[0])
    assert got.changes.tobytes() == loc["changes"].tobytes(), "local changes"
    assert np.array_equal(got.type_dirty, by_type["type_dirty"]) and got.type_gone == by_type["type_gone"], "types"
    assert np.array_equal(got.par_dirty, by_par["par_dirty"]) and np.array_equal(got.par_gone, by_par["par_gone"])


def check_merged(m, prev_all, cur, dprev, dnow):
    want = mdev_delta_ref.expect_mdev_delta(prev_all, cur, dprev.labels, dnow.labels, kvgpu.MDEV_CHANGE)
    assert m.n_prev == len(prev_all) and m.n_now == len(cur)
    assert m.changes.tobytes() == want["changes"].tobytes(), "merged changes"
    assert np.array_equal(m.type_keys, np.unique(cur["type_key"]))
    assert np.array_equal(m.type_dirty, np.unique(cur["type_key"])[want["type_dirty"]]), "merged type_dirty"
    assert m.type_gone == want["type_gone"], "merged type_gone"
    assert np.array_equal(m.par_dirty, np.unique(cur["parent"])[want["par_dirty"]])
    assert np.array_equal(m.par_gone, want["par_gone"])


def run_sequence(lib, P, seed, n0=3000, steps=13):
    rng = np.random.default_rng(seed)
    raw = list(RAW)
    d = Dictionary(raw)
    ranks = [Rank(lib) for _ in range(P)]
    cur = surv(uuids(rng, n0), d, rng)
    cur["parent"] += 1                                    # handles 8 k + 1: every rank owns some parents
    prev_all, dprev = cur[:0], Dictionary([])
    parts_maps = [kvgpu.Maps() for _ in range(P)]
    crossed = moved = 0
    prev_owner, prev_type_owner = {}, {}
    for s in range(steps):
        if s:
            cur, d, raw = step(cur, d, raw, KINDS[(s - 1) % len(KINDS)], rng)
        empty = (s * 7) % P if P > 1 and s % 3 == 1 else None
        bounds = shard_bounds(len(cur), P, rng, empty)
        summaries = []
        owner = {}
        for r in range(P):
            lo, hi = bounds[r]
            lists = [cur[lo:hi]] + owned(cur, P, r)
            for u in key16(lists[0]):
                owner[bytes(u)] = r
            prev_lists = list(ranks[r].prev)
            got = ranks[r].run(lists, d)
            assert got is not None, "ascent error on ascending lists"
            check_rank(got, prev_lists, lists, dprev, d)
            res = shard_result(lists[0], lists[1:], d)
            kvgpu.apply_mdev_shard_delta(parts_maps[r], res, got)
            assert kvgpu.canonical_dump(parts_maps[r]) == kvgpu.canonical_dump(kvgpu.mdev_maps_from_shard(res))
            summaries.append(kvgpu.mdev_shard_delta_part(res, got))
        crossed += sum(1 for u, r in owner.items() if u in prev_owner and prev_owner[u] != r)
        type_owner = {d.labels[int(c)]: int(c) % P for c in np.unique(cur["type_key"])}
        moved += sum(1 for lb, r in type_owner.items() if lb in prev_type_owner and prev_type_owner[lb] != r)
        prev_owner, prev_type_owner = owner, type_owner
        check_merged(kvgpu.merge_mdev_shard_deltas(summaries, dprev.labels, d.labels), prev_all, cur, dprev, d)
        full = kvgpu.merge_parts(parts_maps)
        fresh = kvgpu.merge_parts([kvgpu.mdev_maps_from_shard(shard_result(cur[lo:hi], owned(cur, P, r), d))
                                   for r, (lo, hi) in enumerate(bounds)])
        assert kvgpu.canonical_dump(full) == kvgpu.canonical_dump(fresh)
        prev_all, dprev = cur, d
    return crossed, moved


@pytest.mark.parametrize("P", [1, 2, 3, 8, 16])
def test_snapshot_sequence_per_rank_and_merged(lib, P):
    crossed, moved = run_sequence(lib, P, seed=P)
    assert P == 1 or crossed > 0, "no UUID crossed a shard boundary"
    assert P == 1 or moved > 0, "no label moved to another owner"


def test_owned_lists_longer_than_one_merge_tile(lib):
    """Owned lists of several tiles (P = 2: each about half the survivors), local lists of a few."""
    run_sequence(lib, 2, seed=11, n0=9000, steps=8)


def test_label_moves_owner_with_unchanged_members(lib):
    """The dictionary renumbers two labels across the two ranks and nothing else changes: each label is gone on its
    old owner and dirty on its new one, and absent from both merged lists."""
    rng = np.random.default_rng(12)
    raw0 = [b"alpha\n", b"beta\n", b"gamma\n", b"delta\n"]
    raw1 = [b"beta\n", b"alpha\n", b"gamma\n", b"delta\n"]        # alpha 0 -> 1 (rank 0 -> 1), beta 1 -> 0
    d0, d1 = Dictionary(raw0), Dictionary(raw1)
    a = surv(uuids(rng, 2000), d0, rng)
    b = retype(a, d0, d1)
    ranks = [Rank(lib), Rank(lib)]
    parts = []
    for r in range(2):
        lists = [a[r * 1000:(r + 1) * 1000]] + owned(a, 2, r)
        ranks[r].run(lists, d0)
    for r in range(2):
        lists = [b[r * 1000:(r + 1) * 1000]] + owned(b, 2, r)
        prev_lists = list(ranks[r].prev)
        got = ranks[r].run(lists, d1)
        check_rank(got, prev_lists, lists, d0, d1)
        assert len(got.changes) == 0 and len(got.par_dirty) == 0
        keys = np.unique(lists[1]["type_key"])
        dirty_labels = [d1.labels[int(c)] for c in keys[got.type_dirty]]
        old, new = (b"alpha", b"beta") if r == 0 else (b"beta", b"alpha")
        assert got.type_gone == [old] and dirty_labels == [new], (r, got.type_gone, dirty_labels)
        parts.append(kvgpu.mdev_shard_delta_part(shard_result(lists[0], lists[1:], d1), got))
    m = kvgpu.merge_mdev_shard_deltas(parts, d0.labels, d1.labels)
    assert len(m.changes) == 0 and len(m.type_dirty) == 0 and m.type_gone == []
    check_merged(m, a, b, d0, d1)


def test_first_call_reports_everything_added(lib):
    rng = np.random.default_rng(3)
    d = Dictionary(RAW)
    cur = surv(uuids(rng, 4000), d, rng)
    rk = Rank(lib)
    own = owned(cur, 3, 1)
    got = rk.run([cur[500:1500]] + own, d)
    assert got.n_prev == 0 and (got.changes["what"] == mdev_delta_ref.CH_ADDED).all() and len(got.changes) == 1000
    assert np.array_equal(got.type_dirty, np.arange(len(np.unique(own[0]["type_key"]))))
    assert np.array_equal(got.par_dirty, np.arange(len(np.unique(own[1]["parent"]))))
    assert got.type_gone == [] and len(got.par_gone) == 0
    again = rk.run([cur[500:1500]] + own, d)
    assert len(again.changes) == 0 and len(again.type_dirty) == 0 and len(again.par_dirty) == 0


@pytest.mark.parametrize("which", [0, 1, 2])
@pytest.mark.parametrize("where", [1, 1023, 1500])
def test_non_ascending_list_sets_the_error_word(lib, which, where):
    """A repeated or swapped UUID in the local list or either owned list is refused, and the previous result stays as
    it was."""
    rng = np.random.default_rng(6)
    d = Dictionary(RAW)
    cur = surv(uuids(rng, 4000), d, rng)
    cur["type_key"], cur["parent"] = 0, 0                        # one key each: owned lists = cur
    rk = Rank(lib)
    assert rk.run([cur[:2000], cur, cur], d) is not None
    kept = [a.copy() for a in rk.prev]
    for bad_kind in ("repeat", "swap"):
        lists = [cur[:2000].copy(), cur.copy(), cur.copy()]
        u = lists[which]["uuid"]
        if bad_kind == "repeat":
            u[where] = u[where - 1]
        else:
            u[[where - 1, where]] = u[[where, where - 1]]
        assert rk.run(lists, d) is None, (which, where, bad_kind)
        assert all(np.array_equal(x, y) for x, y in zip(rk.prev, kept))
    nxt = cur.copy()
    nxt["numa"][::50] ^= 1
    got = rk.run([nxt[:2000], nxt, nxt], d)
    check_rank(got, kept, [nxt[:2000], nxt, nxt], d, d)
