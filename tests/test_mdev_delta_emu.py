"""K7 for mdev scans (k_mdev_delta_types -> k_delta_merge<MdevDeltaRec> -> k_delta_lists), executed on the CPU from
the real kernel source under the warp emulator of tools/emu/, against the exact restatement
mdev_delta_ref.expect_mdev_delta: UUIDs that differ from a neighbour only in their low bytes (a compare in the wrong byte
order misplaces them), dictionaries reordered or merged by the label rule, relabels, parent and NUMA moves, a type
whose last mdev goes while its raw name stays, empty lists, merged lengths around one tile, and the ascent check."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import mdev_delta_ref

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

TILE = 1024          # DELTA_TILE: merged positions per CTA of k_delta_merge
XMAP_SLOTS = 1 << 17  # k_mdev_delta_types' table


def label_of(raw: bytes) -> bytes:
    """device_plugin.go:341-342: Trim(raw, "\\n"), then every run of RE2 \\s -> "_" (what k_mdev_labels computes)."""
    return re.sub(rb"[\t\n\f\r ]+", b"_", raw.strip(b"\n"))


def fnv1a(b: bytes) -> int:
    h = 1469598103934665603
    for c in b:
        h = ((h ^ c) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


class Dictionary:
    """A raw type dictionary as a scan sees it: label and canonical id (smallest raw index with the same label) of
    every raw entry."""

    def __init__(self, raw):
        self.labels = [label_of(r) for r in raw]
        first = {}
        self.canon = np.array([first.setdefault(lb, i) for i, lb in enumerate(self.labels)], np.uint16)
        self.off = np.zeros(len(raw) + 1, np.uint32)
        for i, lb in enumerate(self.labels):
            self.off[i + 1] = self.off[i] + len(lb)
        self.bytes = np.frombuffer(b"".join(self.labels) + b"\0" * 16, np.uint8).copy()
        self.len = np.array([len(lb) for lb in self.labels] + [0], np.uint32)
        self.hash = np.array([fnv1a(lb) for lb in self.labels] + [0], np.uint64)


class EmuLabels(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("off", C.c_void_p), ("len", C.c_void_p), ("hash", C.c_void_p)]


class Emu:
    """Runs the three mdev delta kernels like kvg_scan_mdev_delta: tag words, table and cross-map persist across
    calls, each call a new tag."""

    def __init__(self, lib):
        self.lib = lib
        self.cap = 1 << 16
        self.flags = np.zeros(4 * self.cap, dtype=np.uint32)
        self.table = np.zeros(XMAP_SLOTS, dtype=np.uint64)
        self.xlate = np.zeros(1 << 16, dtype=np.uint32)
        self.tag = 100

    def run(self, prev, now, dprev, dnow):
        keys = [np.unique(now["type_key"]).astype(np.uint32), np.unique(prev["type_key"]).astype(np.uint32),
                np.unique(now["parent"]).astype(np.uint32), np.unique(prev["parent"]).astype(np.uint32)]
        keys = [np.concatenate([k, np.zeros(1, np.uint32)]) for k in keys]      # never an empty buffer
        kp = (C.c_void_p * 4)(*[k.ctypes.data for k in keys])
        nk = np.array([len(k) - 1 for k in keys], dtype=np.uint32)
        lab = (EmuLabels * 2)(*[EmuLabels(d.bytes.ctypes.data, d.off.ctypes.data, d.len.ctypes.data,
                                          d.hash.ctypes.data) for d in (dnow, dprev)])
        P = np.ascontiguousarray(prev) if len(prev) else np.zeros(1, kvgpu.MDEV_SURV)
        N = np.ascontiguousarray(now) if len(now) else np.zeros(1, kvgpu.MDEV_SURV)
        ch = np.zeros(len(prev) + len(now) + 1, dtype=kvgpu.MDEV_CHANGE)
        lists = [np.zeros(int(nk[k]) + 1, np.uint32) for k in range(4)]
        counts = np.zeros(6, dtype=np.uint32)
        self.tag += 2
        assert self.lib.emu_mdev_delta(P.ctypes.data, len(prev), N.ctypes.data, len(now), kp, nk.ctypes.data, lab,
                                       self.table.ctypes.data, self.xlate.ctypes.data, self.flags.ctypes.data,
                                       self.cap, self.tag, ch.ctypes.data, *[x.ctypes.data for x in lists],
                                       counts.ctypes.data) == 0
        if counts[1]:
            return None
        return dict(changes=ch[:counts[0]], type_dirty=lists[0][:counts[2]],
                    type_gone=[dprev.labels[int(c)] for c in lists[1][:counts[3]]],
                    par_dirty=lists[2][:counts[4]], par_gone=lists[3][:counts[5]])


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_delta())
    L.emu_mdev_delta.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
    return Emu(L)


def uuids(rng, n):
    """n strictly ascending random UUIDs (big-endian bytes)."""
    v = np.unique(rng.integers(0, 1 << 62, 2 * n + 8, dtype=np.uint64))[:n]
    out = np.zeros((n, 16), np.uint8)
    out[:, :8] = v.astype(">u8").view(np.uint8).reshape(-1, 8)
    out[:, 8:] = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    return out


def surv(u, dic, rng, n_par=30):
    """Survivors with UUIDs u (ascending), raw types drawn from `dic`, parents and NUMA nodes at random."""
    s = np.zeros(len(u), dtype=kvgpu.MDEV_SURV)
    s["uuid"] = u
    s["type_key"] = dic.canon[rng.integers(0, len(dic.labels), len(u))]
    s["parent"] = rng.integers(0, n_par, len(u)) * 8
    s["numa"] = rng.integers(0, 4, len(u))
    s["src"] = np.arange(len(u))
    return s


def check(emu, prev, now, dprev, dnow):
    got = emu.run(prev, now, dprev, dnow)
    want = mdev_delta_ref.expect_mdev_delta(prev, now, dprev.labels, dnow.labels, kvgpu.MDEV_CHANGE)
    assert got is not None, "ascent error on an ascending list"
    for k in ("changes", "type_dirty", "par_dirty", "par_gone"):
        assert np.array_equal(got[k], want[k]), (k, len(prev), len(now))
    assert got["type_gone"] == want["type_gone"]
    return got


def retype(s, dold, dnew):
    """The same survivors described with another dictionary: each type_key becomes the new canonical id of its label
    (a label the new dictionary lacks becomes its entry 0: a relabel)."""
    r = s.copy()
    where = {lb: int(dnew.canon[i]) for i, lb in enumerate(dnew.labels)}
    r["type_key"] = [where.get(dold.labels[int(t)], 0) for t in s["type_key"]]
    return r


RAW = [b"GRID A100-1B\n", b"GRID A100-2Q\n", b"GRID A100-4C\n", b"NVIDIA H100-1-10C\n", b"NVIDIA H100-80C\n"]


def test_hot_added_uuids_between_neighbours(emu):
    """Record j copied with its last byte raised lies strictly between j and j + 1 only in big-endian byte order."""
    rng = np.random.default_rng(1)
    d = Dictionary(RAW)
    prev = surv(uuids(rng, 3000), d, rng)
    add = prev[::7].copy()
    add = add[add["uuid"][:, 15] < 255]
    add["uuid"][:, 15] += 1
    add["src"] = 0
    now = np.concatenate([prev, add])
    key = [bytes(u) for u in now["uuid"]]
    now = now[np.argsort(np.array(key, dtype="V16"), kind="stable")]
    assert len({bytes(u) for u in now["uuid"]}) == len(now)
    got = check(emu, prev, now, d, d)
    assert (got["changes"]["what"] == mdev_delta_ref.CH_ADDED).all() and len(got["changes"]) == len(add)


def test_reordered_dictionary_same_labels_is_no_change(emu):
    rng = np.random.default_rng(2)
    d0 = Dictionary(RAW)
    d1 = Dictionary([RAW[4], b"brand new\n", RAW[2], RAW[0], RAW[3], RAW[1]])    # every id renumbered
    prev = surv(uuids(rng, 2500), d0, rng)
    now = retype(prev, d0, d1)
    assert not np.array_equal(now["type_key"], prev["type_key"])
    got = check(emu, prev, now, d0, d1)
    assert len(got["changes"]) == 0 and len(got["type_dirty"]) == 0 and got["type_gone"] == []


def test_raw_names_with_one_label_are_one_type(emu):
    """An mdev moved between two raw names that sanitise to the same label has not changed."""
    rng = np.random.default_rng(3)
    d0 = Dictionary([b"GRID  A100-2Q\n", b"other\n"])
    d1 = Dictionary([b"other\n", b"GRID\tA100-2Q", b"GRID A100-2Q\n\n"])
    assert d1.canon[2] == 1
    prev = surv(uuids(rng, 500), d0, rng)
    now = retype(prev, d0, d1)
    got = check(emu, prev, now, d0, d1)
    assert len(got["changes"]) == 0 and len(got["type_dirty"]) == 0


def test_relabel_parent_move_and_numa_change(emu):
    rng = np.random.default_rng(4)
    d = Dictionary(RAW)
    prev = surv(uuids(rng, 4000), d, rng)
    i = 1234
    for field, bit, types, parents in (("type_key", mdev_delta_ref.CH_TYPE, True, False),
                                       ("parent", mdev_delta_ref.CH_PARENT, False, True),
                                       ("numa", mdev_delta_ref.CH_NUMA, True, False)):
        now = prev.copy()
        if field == "type_key":
            now["type_key"][i] = d.canon[(int(prev["type_key"][i]) + 1) % len(RAW)]
        elif field == "parent":
            now["parent"][i] = prev["parent"][i] + 8 if prev["parent"][i] < 200 else 0
        else:
            now["numa"][i] = (prev["numa"][i] + 1) % 4
        got = check(emu, prev, now, d, d)
        assert len(got["changes"]) == 1 and got["changes"][0]["what"] == bit
        assert (len(got["type_dirty"]) > 0) == types and (len(got["par_dirty"]) > 0) == parents


def test_type_whose_last_mdev_goes_is_gone(emu):
    """The raw name stays in the dictionary; without a survivor it is no key, so the label went."""
    rng = np.random.default_rng(5)
    d = Dictionary(RAW)
    prev = surv(uuids(rng, 2000), d, rng)
    gone = int(prev["type_key"][17])
    now = prev[prev["type_key"] != gone]
    got = check(emu, prev, now, d, d)
    assert got["type_gone"] == [d.labels[gone]]
    # and with the dictionary renumbered as well
    d1 = Dictionary(RAW[::-1])
    got = check(emu, prev, retype(now, d, d1), d, d1)
    assert got["type_gone"] == [d.labels[gone]]


def test_empty_previous_and_empty_new(emu):
    rng = np.random.default_rng(6)
    d = Dictionary(RAW)
    a = surv(uuids(rng, 1500), d, rng)
    empty = a[:0]
    got = check(emu, empty, a, Dictionary([]), d)
    assert (got["changes"]["what"] == mdev_delta_ref.CH_ADDED).all()
    assert len(got["type_dirty"]) == len(np.unique(a["type_key"])) and got["type_gone"] == []
    got = check(emu, a, empty, d, Dictionary([]))
    assert (got["changes"]["what"] == mdev_delta_ref.CH_REMOVED).all() and len(got["type_dirty"]) == 0
    assert sorted(got["type_gone"]) == sorted({d.labels[int(t)] for t in a["type_key"]})
    check(emu, empty, empty, d, d)


@pytest.mark.parametrize("m", [TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_merged_lengths_around_one_tile(emu, m):
    rng = np.random.default_rng(m)
    d0 = Dictionary(RAW)
    d1 = Dictionary(RAW[::-1] + [b"fresh type\n"])       # every id renumbered
    both = m // 3
    pool = uuids(rng, m - both)                          # exactly m merged positions
    side = rng.permutation(np.r_[np.zeros(m - 2 * both, np.int64), np.full(both, 2)])  # 0: one side only, 2: both
    prev_only = rng.integers(0, 2, len(pool)).astype(bool) & (side == 0)
    prev = surv(pool[(side == 2) | prev_only], d0, rng)
    now = retype(prev[side[(side == 2) | prev_only] == 2], d0, d1)
    now = np.concatenate([now, surv(pool[(side == 0) & ~prev_only], d1, rng)])
    now = now[np.argsort(np.array([bytes(u) for u in now["uuid"]], dtype="V16"), kind="stable")]
    assert len(prev) + len(now) == m
    flip = rng.choice(len(now), max(1, len(now) // 50), replace=False)
    now["numa"][flip] ^= 1
    check(emu, prev, now, d0, d1)


def test_sequence_of_steps_reuses_the_tag_words(emu):
    rng = np.random.default_rng(7)
    raws = [RAW, RAW[::-1], [b"x\n"] + RAW, RAW[2:] + RAW[:2], [b"GRID  A100-1B"] + RAW[1:]]
    dcur = Dictionary(raws[0])
    cur = surv(uuids(rng, 5000), dcur, rng)
    for step in range(10):
        dn = Dictionary(raws[(step + 1) % len(raws)])
        nxt = retype(cur, dcur, dn)
        k = max(1, len(nxt) // 100)
        op = step % 4
        if op == 0:
            add = surv(uuids(rng, 3 * k), dn, rng)
            add = add[~np.isin(np.array([bytes(u) for u in add["uuid"]], "V16"),
                               np.array([bytes(u) for u in nxt["uuid"]], "V16"))][:k]
            nxt = np.concatenate([nxt, add])
            nxt = nxt[np.argsort(np.array([bytes(u) for u in nxt["uuid"]], dtype="V16"), kind="stable")]
        elif op == 1:
            nxt = np.delete(nxt, rng.choice(len(nxt), k, replace=False))
        elif op == 2:
            nxt["type_key"][rng.choice(len(nxt), k, replace=False)] = dn.canon[rng.integers(0, len(dn.labels), k)]
        else:
            pick = rng.choice(len(nxt), k, replace=False)
            nxt["parent"][pick] = rng.integers(0, 40, k) * 8
            nxt["numa"][pick] ^= 1
        nxt["src"] = rng.integers(0, 1 << 20, len(nxt))    # never compared
        check(emu, cur, nxt, dcur, dn)
        cur, dcur = nxt, dn


@pytest.mark.parametrize("where", [1, TILE - 1, TILE, 2500])
def test_duplicate_and_swapped_uuids_set_the_error_flag(emu, where):
    rng = np.random.default_rng(8)
    d = Dictionary(RAW)
    prev = surv(uuids(rng, 3000), d, rng)
    now = surv(uuids(rng, 3000), d, rng)
    bad = now.copy()
    bad["uuid"][where] = bad["uuid"][where - 1]           # a repeated UUID
    assert emu.run(prev, bad, d, d) is None
    bad = now.copy()
    bad["uuid"][[where - 1, where]] = bad["uuid"][[where, where - 1]]   # two swapped
    assert emu.run(prev, bad, d, d) is None
