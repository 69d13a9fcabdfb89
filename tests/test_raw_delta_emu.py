"""kvg_scan_pci_raw_delta's kernels (k_raw_rekey, k_raw_xlate, then K7's k_delta_merge / k_delta_lists) executed on
the CPU from their real source under the warp emulator of tools/emu/, against the string-level restatement
raw_delta_ref.expect: lengths around one merge tile, an equal pair split across two CTAs, names that differ in the
last byte or extend another, a hot-add at the front of an index-mode Walk, a new group string first, "042" against
"42", every column moving between numeric and index mode in both directions, an empty side, and the ascent check."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import delta_ref
import raw_delta_ref

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

TILE = 1024            # DELTA_TILE: merged positions per CTA of k_delta_merge
XLATE_GROUP = 65536    # RAW_XLATE_GROUP
NUM_ADDR, NUM_DEVICE, NUM_GROUP = 1, 2, 4
ALL = NUM_ADDR | NUM_DEVICE | NUM_GROUP


class Side(C.Structure):  # kvg_delta.cuh RawDeltaSide
    _fields_ = [("surv", C.c_void_p), ("n", C.c_uint32), ("off", C.c_void_p), ("bytes", C.c_void_p),
                ("tab", C.c_void_p * 2), ("keys", C.c_void_p * 2), ("n_keys", C.c_uint32 * 2),
                ("numeric", C.c_uint32)]


def make_side(rows, rng, index=(), dummies=0.0):
    """One snapshot of survivors rows = [(name, group, device, numa)] in Walk order, with non-surviving entries mixed
    in at rate `dummies`.  A column is numeric when every string of it is canonical and not listed in `index`
    ('addr', 'group', 'device'), as the raw decode chooses.  -> (side for the restatement, arrays for the emulator)"""
    names = [r[0] for r in rows]
    canon_addr = all(n == kvgpu.format_bdf(kvgpu.parse_bdf(n.decode("latin-1")) or 0).encode()
                     if kvgpu.parse_bdf(n.decode("latin-1")) is not None else False for n in names) and \
        all(a < b for a, b in zip(names, names[1:]))
    canon_grp = all(g.isdigit() and (g == b"0" or g[:1] != b"0") and int(g) < 1 << 32 for _, g, _, _ in rows)
    canon_dev = all(len(d) == 4 and all(c in b"0123456789abcdef" for c in d) for _, _, d, _ in rows)
    numeric = (NUM_ADDR * (canon_addr and "addr" not in index) | NUM_GROUP * (canon_grp and "group" not in index) |
               NUM_DEVICE * (canon_dev and "device" not in index))
    walk = []   # (name, survivor index or None)
    for i, n in enumerate(names):
        while rng.random() < dummies:
            walk.append((b"dummy", None))
        walk.append((n, i))
    blob, off = bytearray(), np.zeros(len(walk) * 6 + 1, np.uint32)
    where = {}
    for w, (n, i) in enumerate(walk):
        off[w * 6] = len(blob)
        blob += n
        off[w * 6 + 1: w * 6 + 7] = len(blob)
        if i is not None:
            where[i] = w
    hnd, tab = {}, {}
    for col, k in (("group", 1), ("device", 2)):
        h, spans = {}, []
        for r in rows:
            if r[k] not in h:
                h[r[k]] = len(spans)
                spans.append((len(blob), len(blob) + len(r[k])))
                blob += r[k]
        hnd[col], tab[col] = h, np.array(spans + [(0, 0)], np.uint32).reshape(-1, 2)
    s = np.zeros(len(rows), dtype=kvgpu.PCI_SURV)
    s["addr"] = [kvgpu.parse_bdf(n.decode()) if numeric & NUM_ADDR else where[i] for i, n in enumerate(names)]
    s["iommu_group"] = [int(g) if numeric & NUM_GROUP else hnd["group"][g] for _, g, _, _ in rows]
    s["device"] = [int(d, 16) if numeric & NUM_DEVICE else hnd["device"][d] for _, _, d, _ in rows]
    s["numa"] = [r[3] for r in rows]
    s["name_slot"] = rng.integers(0, 1 << 20, len(rows))
    ref = dict(names=names, groups=[r[1] for r in rows], devices=[r[2] for r in rows],
               numa=s["numa"].astype(np.uint16), addr=s["addr"].astype(np.uint32),
               grp=s["iommu_group"].astype(np.uint32), dev=s["device"].astype(np.uint32),
               dev_keys=np.unique(s["device"]).astype(np.uint32), grp_keys=np.unique(s["iommu_group"]).astype(np.uint32))
    emu = dict(surv=s if len(s) else np.zeros(1, kvgpu.PCI_SURV), off=off,
               bytes=np.frombuffer(bytes(blob) + b"\0", np.uint8), numeric=numeric,
               tab=[tab["device"], tab["group"]], keys=[np.concatenate([ref["dev_keys"], [0]]).astype(np.uint32),
                                                        np.concatenate([ref["grp_keys"], [0]]).astype(np.uint32)])
    return ref, emu


class Emu:
    """Runs the raw delta's kernels like kvg_scan_pci_raw_delta: the tag words and the key tables persist across
    calls, each call a new tag."""

    def __init__(self, lib):
        self.lib = lib
        self.cap = 1 << 17
        self.flags = np.zeros(4 * self.cap, dtype=np.uint32)
        self.table = np.zeros(1 << 19, dtype=np.uint64)
        self.tag = 100

    def run(self, prev, now):
        (pr, pe), (nr, ne) = prev, now
        sides = (Side * 2)()
        for k, (r, e) in enumerate(((pr, pe), (nr, ne))):
            sides[k] = Side(e["surv"].ctypes.data, len(r["names"]), e["off"].ctypes.data, e["bytes"].ctypes.data,
                            (C.c_void_p * 2)(*[t.ctypes.data for t in e["tab"]]),
                            (C.c_void_p * 2)(*[t.ctypes.data for t in e["keys"]]),
                            (C.c_uint32 * 2)(len(r["dev_keys"]), len(r["grp_keys"])), e["numeric"])
        n_prev, n_now = len(pr["names"]), len(nr["names"])
        xlate = np.full(XLATE_GROUP + len(pr["grp_keys"]) + 1, 0xDEADBEEF, np.uint32)
        rekeyed = np.zeros(4 * (n_prev + n_now + 1), np.uint32)
        ch = np.zeros(n_prev + n_now + 1, dtype=kvgpu.PCI_CHANGE)
        lists = [np.zeros(len(nr["dev_keys"]) + 1, np.uint32), np.zeros(len(pr["dev_keys"]) + 1, np.uint16),
                 np.zeros(len(nr["grp_keys"]) + 1, np.uint32), np.zeros(len(pr["grp_keys"]) + 1, np.uint32)]
        counts = np.zeros(6, np.uint32)
        launches = np.zeros(1, np.uint32)
        self.tag += 2
        assert self.lib.emu_pci_raw_delta(sides, self.table.ctypes.data, xlate.ctypes.data, rekeyed.ctypes.data,
                                          self.flags.ctypes.data, self.cap, self.tag, ch.ctypes.data,
                                          *[x.ctypes.data for x in lists], counts.ctypes.data,
                                          launches.ctypes.data) == 0
        self.launches = int(launches[0])
        if counts[1]:
            return None
        return dict(changes=ch[:counts[0]], dev_dirty=lists[0][:counts[2]], dev_gone=lists[1][:counts[3]],
                    grp_dirty=lists[2][:counts[4]], grp_gone=lists[3][:counts[5]])


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_delta())
    L.emu_pci_raw_delta.argtypes = [C.c_void_p] * 5 + [C.c_uint32, C.c_uint32] + [C.c_void_p] * 7
    return Emu(L)


def check(emu, prev, now):
    got = emu.run(prev, now)
    want = raw_delta_ref.expect(prev[0], now[0])
    assert got is not None, "ascent error on ascending names"
    for k in ("changes", "dev_dirty", "dev_gone", "grp_dirty", "grp_gone"):
        assert np.array_equal(got[k], want[k]), (k, got[k][:8], want[k][:8])
    both_numeric = prev[1]["numeric"] == ALL and now[1]["numeric"] == ALL
    assert emu.launches == (2 if both_numeric else 4)
    return got


def bdf(k):
    return kvgpu.format_bdf(((k >> 8) << 16) | (k & 0xFF)).encode()


def rows_of(rng, keys, n_grp=300, n_dev=40, grp_fmt=b"%d", dev_fmt=b"%04x"):
    return [(bdf(int(k)), grp_fmt % rng.integers(0, n_grp), dev_fmt % (0x1000 + rng.integers(0, n_dev)),
             int(rng.integers(0, 4))) for k in keys]


def mutate(rng, rows, k, n_grp=300, n_dev=40):
    """k random regroups, re-ids, NUMA moves, removals and hot-adds"""
    out = list(rows)
    for _ in range(k):
        i = int(rng.integers(len(out)))
        n, g, d, m = out[i]
        op = rng.integers(5)
        if op == 0:
            out[i] = (n, b"%d" % rng.integers(0, n_grp + 10), d, m)
        elif op == 1:
            out[i] = (n, g, b"%04x" % (0x1000 + rng.integers(0, n_dev + 3)), m)
        elif op == 2:
            out[i] = (n, g, d, m ^ 1)
        elif op == 3 and len(out) > 1:
            del out[i]
        else:
            out.insert(i, (n[:-1] + b"%x" % ((int(n[-1:], 16) + 1) % 8), g, d, m))
            if i + 1 < len(out) and out[i][0] >= out[i + 1][0] or i > 0 and out[i - 1][0] >= out[i][0]:
                del out[i]
    return out


MODES = [(), ("addr",), ("group",), ("device",), ("addr", "group", "device")]


@pytest.mark.parametrize("n_prev,n_now", [(0, 0), (0, 1), (1, 0), (TILE - 1, 0), (0, TILE + 1), (512, 511),
                                          (512, 512), (513, 512), (TILE - 1, TILE + 1), (1500, 1400)])
@pytest.mark.parametrize("modes", [((), ()), (("addr", "group", "device"), ("addr", "group", "device")),
                                   ((), ("addr", "group", "device"))])
def test_lengths_around_one_tile(emu, n_prev, n_now, modes):
    """merged lengths 1023, 1024 and 1025 (shared names count twice) and others, in three mode pairs"""
    rng = np.random.default_rng(n_prev * 7 + n_now)
    pool = np.sort(rng.choice(1 << 20, n_prev + n_now + 10, replace=False))
    a = rows_of(rng, np.sort(rng.choice(pool, n_prev, replace=False)))
    b = rows_of(rng, np.sort(rng.choice(pool, n_now, replace=False)))
    shared = {r[0]: r for r in a}
    b = [shared.get(r[0], r) for r in b]
    check(emu, make_side(a, rng, modes[0], 0.2), make_side(b, rng, modes[1], 0.2))


@pytest.mark.parametrize("what", ["group", "device", "numa", "same"])
@pytest.mark.parametrize("modes", [((), ()), (("addr",), ("addr", "group", "device"))])
def test_equal_pair_split_across_two_ctas(emu, what, modes):
    """one new-only name in front shifts every pair by one: pair 511 straddles the diagonal of CTAs 0 and 1"""
    rng = np.random.default_rng(2)
    prev = rows_of(rng, np.arange(10, 10 + 2 * 1500, 2))
    now = [(bdf(1), b"5", b"1001", 0)] + list(prev)
    k = 512
    n, g, d, m = now[k]
    now[k] = {"group": (n, b"99999", d, m), "device": (n, g, b"2fff", m), "numa": (n, g, d, m + 1),
              "same": now[k]}[what]
    got = check(emu, make_side(prev, rng, modes[0]), make_side(now, rng, modes[1]))
    if what != "same":
        assert len(got["changes"]) == 2
        assert got["changes"][1]["now_index"] == k and got["changes"][1]["prev_index"] == 511


@pytest.mark.parametrize("modes", MODES)
def test_names_differing_in_the_last_byte_and_prefixes(emu, modes):
    rows = [(b"0000:00:01.0", b"1", b"1db6", 0), (b"0000:00:01.0 ", b"1", b"1db6", 0), (b"0000:00:01.1", b"2", b"1db6", 1),
            (b"0000:00:01.2", b"3", b"20b0", 0)]
    rng = np.random.default_rng(3)
    for prev, now in ((rows, rows[1:]), (rows[1:], rows), ([rows[0], rows[2]], [rows[1], rows[3]]), (rows, rows)):
        got = check(emu, make_side(prev, rng, modes, 0.3), make_side(now, rng, modes, 0.3))
        if prev is now:
            assert len(got["changes"]) == 0 and len(got["dev_dirty"]) == 0 and len(got["grp_dirty"]) == 0


def test_hot_add_at_the_front_of_an_index_mode_walk(emu):
    """every Walk index shifts by one, and only the new entry changes"""
    rng = np.random.default_rng(4)
    prev = rows_of(rng, np.arange(100, 3100), n_grp=400)
    now = [(b"0000:00:00.0", b"77777", b"1fff", 0)] + prev
    got = check(emu, make_side(prev, rng, ("addr", "group", "device")), make_side(now, rng, ("addr", "group", "device")))
    assert len(got["changes"]) == 1 and got["changes"][0]["what"] == delta_ref.CH_ADDED
    assert got["changes"][0]["addr"] == 0 and len(got["dev_dirty"]) == 1 and len(got["grp_dirty"]) == 1
    assert len(got["dev_gone"]) == 0 and len(got["grp_gone"]) == 0


def test_new_group_string_first_in_the_walk(emu):
    """a new group first renumbers every group handle; no other entry gets KVG_CH_GROUP"""
    rng = np.random.default_rng(5)
    prev = rows_of(rng, np.arange(100, 2100), n_grp=200)
    now = list(prev)
    n, g, d, m = now[0]
    now[0] = (n, b"g-new", d, m)
    got = check(emu, make_side(prev, rng, ("group",)), make_side(now, rng))
    assert len(got["changes"]) == 1 and got["changes"][0]["what"] == delta_ref.CH_GROUP
    assert len(got["dev_dirty"]) == 0


def test_042_is_not_42(emu):
    rng = np.random.default_rng(6)
    prev = [(bdf(1), b"42", b"1db6", 0), (bdf(2), b"7", b"1db6", 0)]
    now = [(bdf(1), b"042", b"1db6", 0), (bdf(2), b"7", b"1DB6", 0)]
    got = check(emu, make_side(prev, rng), make_side(now, rng))
    assert list(got["changes"]["what"]) == [delta_ref.CH_GROUP, delta_ref.CH_DEVICE]
    assert list(got["grp_gone"]) == [42] and list(got["dev_gone"]) == []


@pytest.mark.parametrize("col", ["addr", "group", "device"])
@pytest.mark.parametrize("direction", ["to_index", "to_numeric"])
def test_each_column_between_modes(emu, col, direction):
    """one column changes mode between the two snapshots while a sequence of edits runs, both directions"""
    rng = np.random.default_rng(hash((col, direction)) & 0xFFFF)
    cur = rows_of(rng, np.sort(rng.choice(1 << 16, 3000, replace=False)))
    for step in range(4):
        nxt = mutate(rng, cur, 12)
        a, b = ((), (col,)) if (direction == "to_index") == (step % 2 == 0) else ((col,), ())
        check(emu, make_side(cur, rng, a, 0.1), make_side(nxt, rng, b, 0.1))
        cur = nxt


@pytest.mark.parametrize("modes", MODES)
def test_sequence_of_edits_in_one_mode(emu, modes):
    rng = np.random.default_rng(len(modes) * 11 + 1)
    cur = rows_of(rng, np.sort(rng.choice(1 << 16, 4000, replace=False)))
    for _ in range(5):
        nxt = mutate(rng, cur, 20)
        check(emu, make_side(cur, rng, modes, 0.1), make_side(nxt, rng, modes, 0.1))
        cur = nxt


@pytest.mark.parametrize("modes", MODES)
def test_one_side_empty(emu, modes):
    rng = np.random.default_rng(7)
    rows = rows_of(rng, np.arange(5, 2005))
    got = check(emu, make_side(rows, rng, modes), make_side([], rng, modes))
    assert (got["changes"]["what"] == delta_ref.CH_REMOVED).all() and len(got["dev_dirty"]) == 0
    got = check(emu, make_side([], rng, modes), make_side(rows, rng, modes))
    assert (got["changes"]["what"] == delta_ref.CH_ADDED).all() and len(got["dev_gone"]) == 0


@pytest.mark.parametrize("where", [1, TILE - 1, TILE, 1500])
@pytest.mark.parametrize("prev_empty", [False, True])
def test_duplicate_and_descending_names_are_refused(emu, where, prev_empty):
    rng = np.random.default_rng(8)
    prev = [] if prev_empty else rows_of(rng, np.arange(0, 6000, 2))
    now = rows_of(rng, np.arange(1, 6000, 2))
    dup = list(now)
    dup[where] = (dup[where - 1][0],) + dup[where][1:]
    assert emu.run(make_side(prev, rng, ("addr",)), make_side(dup, rng, ("addr",))) is None
    swapped = list(now)
    swapped[where], swapped[where - 1] = swapped[where - 1], swapped[where]
    assert emu.run(make_side(prev, rng, ("addr",)), make_side(swapped, rng, ("addr",))) is None
