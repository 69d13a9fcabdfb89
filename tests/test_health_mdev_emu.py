"""K6 for vGPUs (kvg_health_rescan_mdev), both kernel forms executed on the CPU from their real source under the warp
emulator of tools/emu/, against the numpy state machine of tests/health_mdev_ref.py: k_health_small<MdevHealthRule>
(one CTA, 6 rows of 1024 records per TMA round) and k_compact<HealthOp<MdevHealthRule>, 256, 8> (look-back over
2048-record tiles), on the same state bytes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import health_mdev_ref as H
from oracle import oracle as O

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

ROUND = 6 * 1024        # records per TMA round of k_health_small<MdevHealthRule>
SMALL_MAX = 32 * 1024
TILE = 2048             # records per look-back tile
N_TYPES = 200           # gen_mdev draws type indices 0..255: some records are out of the dictionary


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_classify())
    for f in (L.emu_health_mdev_small, L.emu_health_mdev_compact):
        f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


class Kernel:
    """One kernel form with its own state bytes, checked against the reference after every tick."""

    def __init__(self, emu, form, n):
        self.emu, self.form, self.n = emu, form, n
        self.state = np.zeros(n + 1, dtype=np.uint8)
        self.ref = H.HealthMdevRef()

    def tick(self, recs, xids, n_types=N_TYPES):
        n = self.n
        x = np.unique(np.asarray(xids, dtype=np.uint32))
        xbuf = x if len(x) else np.zeros(1, dtype=np.uint32)
        changed = np.zeros(n + 1, dtype=np.uint32)
        hdr = np.zeros(3, dtype=np.uint32)
        buf = np.ascontiguousarray(recs)
        fn = self.emu.emu_health_mdev_small if self.form == "small" else self.emu.emu_health_mdev_compact
        assert fn(buf.ctypes.data, n, n_types, xbuf.ctypes.data, len(x), self.state.ctypes.data, changed.ctypes.data,
                  hdr.ctypes.data) == 0
        if self.form == "small":
            n_alive, n_changed = int(hdr[0]), int(hdr[1])
            assert int(hdr[2]) == 9
        else:
            n_changed, n_alive = int(hdr[0]), int(hdr[1])
        # the host passes X once, duplicates and order included: the reference sees it raw
        want = self.ref.rescan(recs, n_types, xids)
        assert n_alive == want.n_alive and n_changed == len(want.changed), (self.form, n)
        assert np.array_equal(changed[:n_changed], want.changed), (self.form, n)
        assert np.array_equal(self.state[:n], self.ref.state_bytes()), (self.form, n)
        return want


def _edges(n):
    pts = [0, n - 1]
    for b in (32, 1024, ROUND, 2 * ROUND, TILE, 2 * TILE, SMALL_MAX):
        pts += [b - 1, b, b + 1]
    return np.unique(np.array([p for p in pts if 0 <= p < n], dtype=np.int64))


def _drive(k, n, seed):
    rng = np.random.default_rng(seed)
    recs = O.gen_mdev(seed, n)
    parents = np.unique(recs["parent"])
    k.tick(recs, [])                                            # arming: everything present is a transition
    edges = _edges(n)
    xid_lists = [
        [],
        [int(parents[0]), int(parents[0]), 0xdeadbeef, 0],      # duplicates, a handle no record has, handle 0
        [int(parents[-1])],                                     # one parent
        list(map(int, parents[::-1][:1024])),                   # every parent (up to KVG_HEALTH_MAX_XID), descending
        [],
    ]
    for t, xids in enumerate(xid_lists):
        f = np.concatenate([edges, rng.integers(0, n, 8)])
        recs["flags"][f] ^= rng.integers(0, 4, len(f)).astype(np.uint8)      # type / parent read errors flip
        if t == 3:
            recs["type_idx"][f[::2]] = rng.integers(0, 256, len(f[::2]))
        k.tick(recs, xids)


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, ROUND, ROUND + 1, 10_000, SMALL_MAX])
def test_small_form_matches_the_state_machine(emu, n):
    _drive(Kernel(emu, "small", n), n, 40 + n % 97)


@pytest.mark.parametrize("n", [1, 1025, 10_000, 50_000])
def test_compact_form_matches_the_state_machine(emu, n):
    _drive(Kernel(emu, "compact", n), n, 60 + n % 89)


@pytest.mark.parametrize("form", ["small", "compact"])
def test_xid_mark_is_sticky_until_the_vgpu_returns(emu, form):
    """The reference's sequence (generic_vgpu_device_plugin.go:330-351): an XID marks, the mark outlives later ticks,
    a removal while marked sends nothing, a Create sends healthy, and a Create on the tick of an XID sends nothing."""
    n = 3000
    k = Kernel(emu, form, n)
    recs = O.gen_mdev(3, n)
    recs["flags"] = 0
    recs["type_idx"] %= N_TYPES
    v = 1234
    par = int(recs["parent"][v])
    siblings = np.nonzero(recs["parent"] == par)[0]
    k.tick(recs, [])
    d = k.tick(recs, [par])                                             # 1. XID -> unhealthy
    assert list(d.changed) == [int(i) << 1 for i in siblings]
    assert len(k.tick(recs, []).changed) == 0                           # 2. no XID: still unhealthy
    recs["flags"][v] = 1                                                # 3. removed: no transition
    assert len(k.tick(recs, []).changed) == 0
    recs["flags"][v] = 0                                                # 4. back: healthy
    assert list(k.tick(recs, []).changed) == [(v << 1) | 1]
    recs["flags"][v] = 2
    d = k.tick(recs, [])
    assert list(d.changed) == [v << 1]
    recs["flags"][v] = 0                                                # 5. back on the tick of an XID: nothing
    assert len(k.tick(recs, [par]).changed) == 0                        # (its siblings are still marked)


def test_both_forms_share_one_state(emu):
    """The host runs the look-back form for a timed tick between untimed ones: the state bytes are one format."""
    n = 10_000
    recs = O.gen_mdev(8, n)
    a = Kernel(emu, "small", n)
    a.tick(recs, [])
    rng = np.random.default_rng(2)
    parents = np.unique(recs["parent"])
    for t in range(4):
        recs["flags"][rng.integers(0, n, 16)] ^= 1
        a.form = "compact" if t % 2 else "small"
        a.tick(recs, [int(parents[t * 7])])
