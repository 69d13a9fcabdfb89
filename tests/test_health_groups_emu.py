"""K6 for passthrough GPUs by IOMMU group (kvg_health_rescan_groups), both kernel forms executed on the CPU from their
real source under the warp emulator of tools/emu/, against the numpy state machine of tests/health_groups_ref.py:
k_health_small<GroupHealthRule> (one CTA, 12 rows of 1024 records per TMA round, the group set behind the stage)
and k_compact<HealthOp<GroupHealthRule>, 256, 8> (look-back over 2048-record tiles), on the same state bytes.  Also the
two properties the call promises: with a node for every group it reports what kvg_health_rescan's kernels
(PciHealthRule) report (P1), and with every record alive all devices of a group flip together (P2)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import health_groups_ref as H

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

ROUND = 12 * 1024       # records per TMA round of k_health_small<GroupHealthRule>
SMALL_MAX = 32 * 1024
TILE = 2048             # records per look-back tile
CAP = 4096              # KVG_HEALTH_MAX_GROUPS


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_classify())
    for f in (L.emu_health_groups_small, L.emu_health_groups_compact):
        f.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    for f in (L.emu_health_small, L.emu_health_rescan):
        f.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _sorted_set(nodes):
    g = np.unique(np.asarray(nodes, dtype=np.uint32))
    return g, (g if len(g) else np.zeros(1, dtype=np.uint32))


class Kernel:
    """One kernel form with its own state bytes, checked against the reference after every tick."""

    def __init__(self, emu, form, n):
        self.emu, self.form, self.n = emu, form, n
        self.state = np.zeros(n + 1, dtype=np.uint8)
        self.ref = H.HealthGroupsRef()

    def tick(self, recs, nodes):
        n = self.n
        g, gbuf = _sorted_set(nodes)                 # what the host hands the kernels: sorted, deduplicated
        changed = np.zeros(n + 1, dtype=np.uint32)
        hdr = np.zeros(3, dtype=np.uint32)
        buf = np.ascontiguousarray(recs)
        fn = self.emu.emu_health_groups_small if self.form == "small" else self.emu.emu_health_groups_compact
        assert fn(buf.ctypes.data, n, gbuf.ctypes.data, len(g), self.state.ctypes.data, changed.ctypes.data,
                  hdr.ctypes.data) == 0
        if self.form == "small":
            n_alive, n_changed = int(hdr[0]), int(hdr[1])
            assert int(hdr[2]) == 5
        else:
            n_changed, n_alive = int(hdr[0]), int(hdr[1])
        want = self.ref.rescan(recs, nodes)          # the raw set, duplicates and order included
        assert n_alive == want.n_alive and n_changed == len(want.changed), (self.form, n)
        assert np.array_equal(changed[:n_changed], want.changed), (self.form, n)
        assert np.array_equal(self.state[:n], self.ref.state_bytes()), (self.form, n)
        return changed[:n_changed].copy(), n_alive


class PlainHealth:
    """kvg_health_rescan's kernels (k_health_small<PciHealthRule> / k_compact<HealthOp<PciHealthRule>>) on their own
    state."""

    def __init__(self, emu, form, n):
        self.emu, self.form, self.n = emu, form, n
        self.state = np.zeros(n + 1, dtype=np.uint8)

    def tick(self, recs):
        n = self.n
        changed = np.zeros(n + 1, dtype=np.uint32)
        hdr = np.zeros(3, dtype=np.uint32)
        buf = np.ascontiguousarray(recs)
        if self.form == "small":
            assert self.emu.emu_health_small(buf.ctypes.data, n, self.state.ctypes.data, changed.ctypes.data,
                                             hdr.ctypes.data) == 0
            n_alive, n_changed = int(hdr[0]), int(hdr[1])
        else:
            self.emu.emu_health_rescan(buf.ctypes.data, n, self.state.ctypes.data, changed.ctypes.data, hdr.ctypes.data)
            n_changed, n_alive = int(hdr[0]), int(hdr[1])
        return changed[:n_changed].copy(), n_alive


def _edges(n):
    pts = [0, n - 1]
    for b in (32, 1024, ROUND, 2 * ROUND, TILE, 2 * TILE, SMALL_MAX):
        pts += [b - 1, b, b + 1]
    return np.unique(np.array([p for p in pts if 0 <= p < n], dtype=np.int64))


def _per_group(n):
    return max(4, -(-n // CAP))                      # 4 functions per group, fewer groups than the cap


def _drive(k, n, seed):
    rng = np.random.default_rng(seed)
    recs = H.make_recs(n, rng, _per_group(n))
    groups = np.unique(recs["iommu_group"])
    unused = np.setdiff1d(np.arange(1, 2 * CAP + len(groups) + 2, dtype=np.uint32), groups)
    k.tick(recs, groups)                                              # arming: every group has a node
    edges = _edges(n)
    gone = rng.choice(groups, max(1, len(groups) // 5), replace=False)
    node_sets = [
        [],                                                           # no node at all: nothing is healthy
        [int(groups[-1])],                                            # a set of one
        list(np.setdiff1d(groups, gone)[::-1]) + [int(groups[0])] * 3 + [0, 0xDEADBEEF, 0xFFFFFFFF],
        # ^ some nodes vanished; descending, duplicates, handles no record carries (0 = no group)
        np.concatenate([groups, unused[:CAP - len(groups)]]),        # exactly KVG_HEALTH_MAX_GROUPS handles
        groups,                                                       # every node back
    ]
    for t, nodes in enumerate(node_sets):
        f = np.concatenate([edges, rng.integers(0, n, 8)])
        if t % 2:
            H.revive(recs, f)
        else:
            H.kill(recs, f[::2], rng)
        k.tick(recs, nodes)


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, ROUND, ROUND + 1, 10_000, SMALL_MAX])
def test_small_form_matches_the_state_machine(emu, n):
    _drive(Kernel(emu, "small", n), n, 70 + n % 97)


@pytest.mark.parametrize("n", [1, TILE - 1, TILE, TILE + 1, 2 * TILE + 1, 50_000])
def test_compact_form_matches_the_state_machine(emu, n):
    _drive(Kernel(emu, "compact", n), n, 80 + n % 89)


@pytest.mark.parametrize("form", ["small", "compact"])
def test_every_node_present_is_kvg_health_rescan(emu, form):
    """P1: with a node for every group, the transition lists, counters and state bytes are those of the plain health
    kernels on the same sequence of snapshots."""
    n = 5000
    rng = np.random.default_rng(11)
    recs = H.make_recs(n, rng, 3, alive_frac=0.6)
    k, plain = Kernel(emu, form, n), PlainHealth(emu, form, n)
    for t in range(5):
        if t:
            f = rng.integers(0, n, 40)
            H.kill(recs, f[:20], rng)
            H.revive(recs, f[20:])
            recs["iommu_group"][rng.integers(0, n, 4)] = rng.integers(1, 3000, 4)   # regrouped, still with a node
        got = k.tick(recs, np.unique(recs["iommu_group"]))
        want = plain.tick(recs)
        assert np.array_equal(got[0], want[0]) and got[1] == want[1], (form, t)
        assert np.array_equal(k.state[:n], plain.state[:n]), (form, t)


@pytest.mark.parametrize("form", ["small", "compact"])
def test_a_group_flips_as_a_whole(emu, form):
    """P2, the reference's Create / Remove / Rename of /dev/vfio/<group> (generic_device_plugin.go:611-690): with every
    record alive, the devices of a group go unhealthy together when its node vanishes and healthy when it returns."""
    n = 3000
    rng = np.random.default_rng(12)
    recs = H.make_recs(n, rng, 4, alive_frac=1.0)
    groups = np.unique(recs["iommu_group"])
    k = Kernel(emu, form, n)
    changed, alive = k.tick(recs, groups)
    assert alive == n and len(changed) == n
    members = {int(g): np.nonzero(recs["iommu_group"] == g)[0] for g in groups}
    a, b = int(groups[17]), int(groups[500])
    changed, alive = k.tick(recs, np.setdiff1d(groups, [a]))
    assert list(changed) == [int(i) << 1 for i in members[a]] and alive == n - 4
    assert len(k.tick(recs, np.setdiff1d(groups, [a]))[0]) == 0                 # still gone: nothing new
    changed, _ = k.tick(recs, np.setdiff1d(groups, [b]))                       # a returns as b goes
    assert list(changed) == sorted([(int(i) << 1) | 1 for i in members[a]] + [int(i) << 1 for i in members[b]])
    changed, alive = k.tick(recs, groups)
    assert list(changed) == [(int(i) << 1) | 1 for i in members[b]] and alive == n


def test_both_forms_share_one_state(emu):
    """The host runs the look-back form for a timed tick between untimed ones: the state bytes are one format."""
    n = 10_000
    rng = np.random.default_rng(2)
    recs = H.make_recs(n, rng)
    groups = np.unique(recs["iommu_group"])
    a = Kernel(emu, "small", n)
    a.tick(recs, groups)
    for t in range(4):
        H.kill(recs, rng.integers(0, n, 16), rng)
        a.form = "compact" if t % 2 else "small"
        a.tick(recs, np.setdiff1d(groups, groups[t * 7:t * 7 + 3]))
