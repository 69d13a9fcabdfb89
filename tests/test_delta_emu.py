"""K7, the re-scan delta (k_delta_merge -> k_delta_lists), executed on the CPU from its real kernel source under the
warp emulator of tools/emu/, against the exact restatement delta_ref.expect_pci_delta: list lengths around one merge
tile, everything removed / added, interleaved lists, an equal pair split across two CTAs, each kind of change,
keys that go while others of the same map turn dirty, tag words reused across calls, and the ascent check."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import delta_ref

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

TILE = 1024  # DELTA_TILE: merged positions per CTA of k_delta_merge


class Emu:
    """Runs the two delta kernels like kvg_scan_pci_delta: the tag words persist across calls, each call a new tag."""

    def __init__(self, lib):
        self.lib = lib
        self.cap = 1 << 16
        self.flags = np.zeros(4 * self.cap, dtype=np.uint32)
        self.tag = 100

    def run(self, prev, now):
        keys = [np.unique(now["device"]).astype(np.uint32), np.unique(prev["device"]).astype(np.uint32),
                np.unique(now["iommu_group"]).astype(np.uint32), np.unique(prev["iommu_group"]).astype(np.uint32)]
        assert max(len(k) for k in keys) <= self.cap
        keys = [np.concatenate([k, np.zeros(1, np.uint32)]) for k in keys]      # never an empty buffer
        kp = (C.c_void_p * 4)(*[k.ctypes.data for k in keys])
        nk = np.array([len(k) - 1 for k in keys], dtype=np.uint32)
        P = np.ascontiguousarray(prev) if len(prev) else np.zeros(1, kvgpu.PCI_SURV)
        N = np.ascontiguousarray(now) if len(now) else np.zeros(1, kvgpu.PCI_SURV)
        ch = np.zeros(len(prev) + len(now) + 1, dtype=kvgpu.PCI_CHANGE)
        lists = [np.zeros(int(nk[0]) + 1, np.uint32), np.zeros(int(nk[1]) + 1, np.uint16),
                 np.zeros(int(nk[2]) + 1, np.uint32), np.zeros(int(nk[3]) + 1, np.uint32)]
        counts = np.zeros(6, dtype=np.uint32)
        self.tag += 2
        assert self.lib.emu_delta(P.ctypes.data, len(prev), N.ctypes.data, len(now), kp, nk.ctypes.data,
                                  self.flags.ctypes.data, self.cap, self.tag, ch.ctypes.data,
                                  *[x.ctypes.data for x in lists], counts.ctypes.data) == 0
        if counts[1]:
            return None
        return dict(changes=ch[:counts[0]], dev_dirty=lists[0][:counts[2]], dev_gone=lists[1][:counts[3]],
                    grp_dirty=lists[2][:counts[4]], grp_gone=lists[3][:counts[5]])


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_delta())
    L.emu_delta.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                            C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
    return Emu(L)


def surv(addr, rng, n_dev=40, n_grp=200):
    s = np.zeros(len(addr), dtype=kvgpu.PCI_SURV)
    s["addr"] = addr
    s["iommu_group"] = rng.integers(0, n_grp, len(addr))
    s["device"] = rng.integers(0x1000, 0x1000 + n_dev, len(addr))
    s["numa"] = rng.integers(0, 4, len(addr))
    s["name_slot"] = rng.integers(0, 1 << 20, len(addr))
    return s


def check(emu, prev, now):
    got = emu.run(prev, now)
    want = delta_ref.expect_pci_delta(prev, now, kvgpu.PCI_CHANGE)
    assert got is not None, "ascent error on an ascending list"
    for k in ("changes", "dev_dirty", "dev_gone", "grp_dirty", "grp_gone"):
        assert np.array_equal(got[k], want[k]), (k, len(prev), len(now))
    return got


def sorted_addrs(rng, n, hi=1 << 28):
    return np.sort(rng.choice(hi, n, replace=False)).astype(np.uint32)


@pytest.mark.parametrize("n_prev,n_now", [(0, 0), (0, 1), (1, 0), (1, 1), (TILE - 1, 0), (0, TILE + 1),
                                          (TILE - 1, TILE + 1), (TILE + 1, TILE - 1), (3000, 2500)])
def test_lengths_around_one_tile(emu, n_prev, n_now):
    rng = np.random.default_rng(n_prev * 7 + n_now)
    pool = sorted_addrs(rng, n_prev + n_now + 10)
    prev = surv(np.sort(rng.choice(pool, n_prev, replace=False)), rng)
    now = surv(np.sort(rng.choice(pool, n_now, replace=False)), rng)
    now[np.isin(now["addr"], prev["addr"])] = prev[np.isin(prev["addr"], now["addr"])]  # shared addresses: same device
    check(emu, prev, now)


def test_all_removed_all_added_interleaved(emu):
    rng = np.random.default_rng(1)
    a = surv(np.arange(0, 5000, 2, dtype=np.uint32), rng)
    b = surv(np.arange(1, 5000, 2, dtype=np.uint32), rng)
    empty = a[:0]
    got = check(emu, a, empty)
    assert (got["changes"]["what"] == delta_ref.CH_REMOVED).all() and len(got["dev_dirty"]) == 0
    assert np.array_equal(got["dev_gone"], np.unique(a["device"]))
    got = check(emu, empty, b)
    assert (got["changes"]["what"] == delta_ref.CH_ADDED).all() and len(got["dev_gone"]) == 0
    assert len(got["dev_dirty"]) == len(np.unique(b["device"])) and len(got["grp_dirty"]) == len(np.unique(b["iommu_group"]))
    got = check(emu, a, b)                     # nothing shared: every address once
    assert len(got["changes"]) == len(a) + len(b)
    check(emu, a, a)                           # nothing changed
    assert len(emu.run(a, a)["changes"]) == 0


@pytest.mark.parametrize("what", ["group", "device", "numa", "same"])
def test_equal_pair_split_across_two_ctas(emu, what):
    """One new-only address in front shifts every pair by one: pair k sits at merged positions 2k+1, 2k+2, so
    pair 511 straddles the diagonal between CTA 0 and CTA 1."""
    rng = np.random.default_rng(2)
    prev = surv(np.arange(10, 10 + 2 * 1500, 2, dtype=np.uint32), rng)
    now = np.concatenate([surv(np.array([1], np.uint32), rng), prev.copy()])
    k = 511 + 1
    if what == "group":
        now["iommu_group"][k] += 1000
    elif what == "device":
        now["device"][k] ^= 0x4000
    elif what == "numa":
        now["numa"][k] += 1
    got = check(emu, prev, now)
    assert got["changes"]["addr"][0] == 1
    if what != "same":
        assert len(got["changes"]) == 2 and got["changes"][1]["addr"] == prev["addr"][511]
        assert got["changes"][1]["now_index"] == k and got["changes"][1]["prev_index"] == 511


def test_each_kind_of_change_dirties_its_maps(emu):
    rng = np.random.default_rng(3)
    prev = surv(sorted_addrs(rng, 4000), rng, n_dev=30, n_grp=500)
    i = 1234
    for field, bit, dev_dirty, grp_dirty in (("iommu_group", delta_ref.CH_GROUP, 0, 2), ("device", delta_ref.CH_DEVICE, 2, 0),
                                             ("numa", delta_ref.CH_NUMA, 1, 1)):
        now = prev.copy()
        now[field][i] = prev[field][i] + 1 if field != "iommu_group" else 100_000   # a new group
        if field == "device":
            now["device"][i] = prev["device"][(i + 1) % len(prev)] if prev["device"][(i + 1) % len(prev)] != prev["device"][i] \
                else prev["device"][i] + 1
        got = check(emu, prev, now)
        assert len(got["changes"]) == 1 and got["changes"][0]["what"] == bit
        assert len(got["dev_dirty"]) + len(got["dev_gone"]) <= dev_dirty
        assert len(got["grp_dirty"]) + len(got["grp_gone"]) <= grp_dirty
        assert (len(got["dev_dirty"]) > 0) == (dev_dirty > 0) and (len(got["grp_dirty"]) > 0) == (grp_dirty > 0)


def test_key_gone_while_another_turns_dirty(emu):
    rng = np.random.default_rng(4)
    prev = surv(sorted_addrs(rng, 3000), rng, n_dev=20, n_grp=300)
    now = prev.copy()
    gone_dev = prev["device"][100]
    keep = prev["device"] != gone_dev                     # every member of one device id leaves
    now = now[keep]
    now["device"][5] = 0x7777                             # another one moves to a brand-new id
    grp = now["iommu_group"][7]
    now = now[now["iommu_group"] != grp]                  # a whole group leaves too
    got = check(emu, prev, now)
    assert gone_dev in got["dev_gone"] and 0x7777 in np.unique(now["device"])[got["dev_dirty"]]
    assert grp in got["grp_gone"] and len(got["grp_dirty"]) > 0


def test_sequence_of_steps_reuses_the_tag_words(emu):
    """Random hot-add / hot-remove / regroup / re-id / NUMA steps, each diffed against the one before, with the
    tag words of earlier calls left in place (they must read as unmarked)."""
    rng = np.random.default_rng(5)
    cur = surv(sorted_addrs(rng, 6000), rng, n_dev=50, n_grp=2000)
    for step in range(12):
        nxt = cur.copy()
        k = max(1, len(nxt) // 200)
        op = step % 5
        if op == 0:
            add = surv(np.setdiff1d(sorted_addrs(rng, 4 * k), nxt["addr"])[:k], rng, n_dev=60, n_grp=2200)
            nxt = np.sort(np.concatenate([nxt, add]), order="addr")
        elif op == 1:
            nxt = np.delete(nxt, rng.choice(len(nxt), k, replace=False))
        elif op == 2:
            nxt["iommu_group"][rng.choice(len(nxt), k, replace=False)] = rng.integers(0, 2500, k)
        elif op == 3:
            nxt["device"][rng.choice(len(nxt), k, replace=False)] = rng.integers(0x1000, 0x1040, k)
        else:
            nxt["numa"][rng.choice(len(nxt), k, replace=False)] ^= 1
        nxt["name_slot"] = rng.integers(0, 1 << 20, len(nxt))    # never compared
        check(emu, cur, nxt)
        cur = nxt


@pytest.mark.parametrize("where", [1, TILE - 1, TILE, 2500])
def test_non_ascending_new_list_sets_the_error_flag(emu, where):
    rng = np.random.default_rng(6)
    prev = surv(np.arange(0, 6000, 2, dtype=np.uint32), rng)
    now = surv(np.arange(1, 6000, 2, dtype=np.uint32), rng)
    now["addr"][where] = now["addr"][where - 1]           # a repeated address
    assert emu.run(prev, now) is None
    now = surv(np.arange(1, 6000, 2, dtype=np.uint32), rng)
    now["addr"][where], now["addr"][where - 1] = now["addr"][where - 1], now["addr"][where]   # two swapped
    assert emu.run(prev, now) is None
