"""The keyed health re-scans (kvg_health_rescan_mdev_keyed / _groups_keyed), both kernel forms of both kinds executed
on the CPU from their real source under the warp emulator of tools/emu/: k_health_small<Keyed<Rule>> and
k_compact<HealthOp<Keyed<Rule>>, 256, 8>, against the dict-keyed state machine of tests/health_keyed_ref.py.  The
harness keeps the two slots as the host driver does: a call writes this call's keys and bytes, which become the
previous list only when the call is not refused."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import health_groups_ref as HG
import health_keyed_ref as HK
from oracle import oracle as O

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

SMALL_MAX = 32 * 1024
N_TYPES = 200           # gen_mdev draws type indices 0..255: some records are out of the dictionary
vp, u32 = C.c_void_p, C.c_uint32


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_classify())
    for f in (L.emu_health_mdev_keyed_small, L.emu_health_mdev_keyed_compact):
        f.argtypes = [vp, u32, u32, vp, u32, vp, vp, u32, vp, vp, vp, vp]
    for f in (L.emu_health_groups_keyed_small, L.emu_health_groups_keyed_compact):
        f.argtypes = [vp, u32, vp, u32, vp, vp, u32, vp, vp, vp, vp]
    for f in (L.emu_health_mdev_small, L.emu_health_mdev_compact):
        f.argtypes = [vp, u32, u32, vp, u32, vp, vp, vp]
    for f in (L.emu_health_groups_small, L.emu_health_groups_compact):
        f.argtypes = [vp, u32, vp, u32, vp, vp, vp]
    return L


def _set(xs):
    x = np.unique(np.asarray(list(xs), dtype=np.uint32))
    return x, (x if len(x) else np.zeros(1, dtype=np.uint32))


class Keyed:
    """One kind's keyed state as the host keeps it (the previous list), run through either kernel form and checked
    against the reference after every call."""

    def __init__(self, emu, kind):
        self.emu, self.kind = emu, kind
        self.kw = 16 if kind == "mdev" else 4          # key bytes
        self.prev_key = np.zeros(self.kw, dtype=np.uint8)
        self.prev_state = np.zeros(1, dtype=np.uint8)
        self.n_prev = 0
        self.ref = HK.KeyedMdevRef() if kind == "mdev" else HK.KeyedGroupsRef()

    def raw(self, recs, xs, form):
        """One kernel call: -> (refused, n_alive, changed)."""
        n = len(recs)
        x, xbuf = _set(xs)
        key_out = np.zeros((n + 1) * self.kw, dtype=np.uint8)
        state_out = np.zeros(n + 1, dtype=np.uint8)
        changed = np.zeros(n + 1, dtype=np.uint32)
        hdr = np.zeros(4, dtype=np.uint32)
        buf = np.ascontiguousarray(recs)
        k = self.emu
        fn = {("mdev", "small"): k.emu_health_mdev_keyed_small, ("mdev", "compact"): k.emu_health_mdev_keyed_compact,
              ("groups", "small"): k.emu_health_groups_keyed_small,
              ("groups", "compact"): k.emu_health_groups_keyed_compact}[(self.kind, form)]
        head = [buf.ctypes.data, n] + ([N_TYPES] if self.kind == "mdev" else [])
        assert fn(*head, xbuf.ctypes.data, len(x), self.prev_key.ctypes.data, self.prev_state.ctypes.data, self.n_prev,
                  key_out.ctypes.data, state_out.ctypes.data, changed.ctypes.data, hdr.ctypes.data) == 0
        if form == "small":
            n_alive, n_changed, err = int(hdr[0]), int(hdr[1]), int(hdr[3])
        else:
            n_changed, n_alive, err = int(hdr[0]), int(hdr[1]), int(hdr[2])
        if not err:  # adopt this call's slot
            self.prev_key, self.prev_state, self.n_prev = key_out, state_out, n
        return bool(err), n_alive, changed[:n_changed].copy()

    def keys(self, recs):
        return HK.mdev_keys(recs) if self.kind == "mdev" else HK.group_keys(recs)

    def tick(self, recs, xs, form):
        refused, n_alive, changed = self.raw(recs, xs, form)
        assert not refused
        want = self.ref.rescan(recs, N_TYPES, xs) if self.kind == "mdev" else self.ref.rescan(recs, xs)
        assert n_alive == want.n_alive, (self.kind, form, len(recs))
        assert np.array_equal(changed, want.changed), (self.kind, form, len(recs))
        # the kept list is this call's keys, ascending, with the reference's state bytes
        got_keys = self.prev_key[:self.n_prev * self.kw].reshape(-1, self.kw)
        want_keys = (np.array([list(k) for k in self.keys(recs)], dtype=np.uint8).reshape(-1, 16)
                     if self.kind == "mdev" else np.ascontiguousarray(recs["addr"], dtype="<u4").view(np.uint8).reshape(-1, 4))
        assert np.array_equal(got_keys, want_keys)
        assert np.array_equal(self.prev_state[:self.n_prev], self.ref.state_bytes(self.keys(recs)))
        return changed


def _universe(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "mdev":
        return O.gen_mdev(seed, n), rng
    return HG.make_recs(n, rng, per_group=4), rng


def _mutate(kind, u, idx, rng):
    if kind == "mdev":
        u["flags"][idx] ^= rng.integers(0, 4, len(idx)).astype(np.uint8)
    else:
        dead = idx[rng.random(len(idx)) < 0.5]
        HG.kill(u, dead, rng)
        HG.revive(u, np.setdiff1d(idx, dead))


def _sets(kind, u, rng):
    if kind == "mdev":
        parents = np.unique(u["parent"])
        return [[], [int(parents[0]), int(parents[0]), 0xdeadbeef], [], [int(p) for p in rng.choice(parents, 3)], []]
    groups = np.unique(u["iommu_group"])
    every = [int(g) for g in groups[:4096]]
    return [every, every[::2], every, [int(g) for g in rng.choice(groups, min(len(groups), 50))], every]


def _edit(sel, n_universe, t, rng):
    """The list edits of the random sequences: insert at 0, drop the last, replace the middle, unchanged."""
    sel = list(sel)
    free = sorted(set(range(n_universe)) - set(sel))
    e = t % 4
    if e == 0 and free and free[0] < sel[0]:
        sel.insert(0, max(f for f in free if f < sel[0]))
    elif e == 1 and len(sel) > 1:
        sel.pop()
    elif e == 2 and len(sel) > 2:
        mid = len(sel) // 2
        lo, hi = sel[mid - 1], sel[mid + 1]
        cands = [f for f in free if lo < f < hi]
        sel.pop(mid)
        if cands:
            sel.insert(mid, int(rng.choice(cands)))
    return np.array(sel, dtype=np.int64)


def _drive(emu, kind, n, forms, seed, ticks=10):
    u, rng = _universe(kind, n + 64, seed)
    k = Keyed(emu, kind)
    sel = np.arange(40, 40 + n)
    sets = _sets(kind, u, rng)
    for t in range(ticks):
        _mutate(kind, u, rng.integers(0, len(u), 12 + n // 200), rng)
        if t:
            sel = _edit(sel, len(u), t, rng)
        k.tick(u[sel], sets[t % len(sets)], forms[t % len(forms)])


@pytest.mark.parametrize("kind", ["mdev", "groups"])
@pytest.mark.parametrize("n", [1, 1023, 6 * 1024 + 1, 12 * 1024 + 1, 10_000, SMALL_MAX - 2])
def test_small_form_matches_the_keyed_state_machine(emu, kind, n):
    _drive(emu, kind, n, ["small"], 70 + n % 53)


@pytest.mark.parametrize("kind", ["mdev", "groups"])
@pytest.mark.parametrize("n", [1, 2047, 2049, 10_000, 40_000])
def test_compact_form_matches_the_keyed_state_machine(emu, kind, n):
    _drive(emu, kind, n, ["compact"], 80 + n % 59, ticks=6)


@pytest.mark.parametrize("kind", ["mdev", "groups"])
def test_small_and_compact_forms_continue_one_state(emu, kind):
    """The host runs the look-back form for a timed tick between untimed ones: one list, two forms."""
    _drive(emu, kind, 5000, ["small", "compact"], 5, ticks=8)


def _index(emu, kind, form, recs, xs, state):
    n = len(recs)
    x, xbuf = _set(xs)
    changed = np.zeros(n + 1, dtype=np.uint32)
    hdr = np.zeros(3, dtype=np.uint32)
    buf = np.ascontiguousarray(recs)
    if kind == "mdev":
        fn = emu.emu_health_mdev_small if form == "small" else emu.emu_health_mdev_compact
        assert fn(buf.ctypes.data, n, N_TYPES, xbuf.ctypes.data, len(x), state.ctypes.data, changed.ctypes.data,
                  hdr.ctypes.data) == 0
    else:
        fn = emu.emu_health_groups_small if form == "small" else emu.emu_health_groups_compact
        assert fn(buf.ctypes.data, n, xbuf.ctypes.data, len(x), state.ctypes.data, changed.ctypes.data,
                  hdr.ctypes.data) == 0
    n_alive, n_changed = (hdr[0], hdr[1]) if form == "small" else (hdr[1], hdr[0])
    return int(n_alive), changed[:int(n_changed)].copy()


@pytest.mark.parametrize("form", ["small", "compact"])
@pytest.mark.parametrize("kind", ["mdev", "groups"])
def test_k1_same_key_list_gives_the_index_keyed_delta(emu, kind, form):
    """K1: with the same key list on every call, each delta equals the index-keyed call's, from fresh states."""
    n = 7000
    u, rng = _universe(kind, n, 11)
    k = Keyed(emu, kind)
    state = np.zeros(n + 1, dtype=np.uint8)
    for t, xs in enumerate(_sets(kind, u, rng)):
        _mutate(kind, u, rng.integers(0, n, 40), rng)
        refused, alive, changed = k.raw(u, xs, form)
        assert not refused
        alive_i, changed_i = _index(emu, kind, form, u, xs, state)
        assert alive == alive_i and np.array_equal(changed, changed_i), t
        assert np.array_equal(k.prev_state[:n], state[:n])


@pytest.mark.parametrize("kind", ["mdev", "groups"])
def test_k2_other_keys_never_change_a_staying_key(emu, kind):
    """K2: adding or removing other keys changes neither the delta entry nor the state of a key that stays."""
    u, rng = _universe(kind, 4000, 12)
    core = np.arange(0, 4000, 3)
    a, b = Keyed(emu, kind), Keyed(emu, kind)
    sets = _sets(kind, u, rng)
    for t in range(8):
        _mutate(kind, u, rng.integers(0, 4000, 60), rng)
        others = np.setdiff1d(rng.choice(4000, 800, replace=False), core)
        sel_b = np.union1d(core, others)
        xs = sets[t % len(sets)]
        _, _, ca = a.raw(u[core], xs, "small" if t % 2 else "compact")
        _, _, cb = b.raw(u[sel_b], xs, "compact" if t % 2 else "small")
        pos = {int(s): i for i, s in enumerate(sel_b)}
        in_b = {int(sel_b[w >> 1]): int(w & 1) for w in cb}
        want = {int(core[w >> 1]): int(w & 1) for w in ca}
        assert {s: v for s, v in in_b.items() if s in set(core.tolist())} == want
        assert np.array_equal(a.prev_state[:len(core)], b.prev_state[[pos[int(s)] for s in core]])


def test_xid_marks_survive_unrelated_list_edits(emu):
    """An XID marks the vGPUs of one GPU; a vGPU added on another GPU, or one dropped, does not clear the marks.  Only
    a vanish and return of a marked vGPU clears its own mark."""
    u, _ = _universe("mdev", 3000, 3)
    u["flags"] = 0
    u["type_idx"] %= N_TYPES
    k = Keyed(emu, "mdev")
    sel = np.arange(100, 2900)
    par = int(u["parent"][1234])
    marked = sel[u["parent"][sel] == par]
    k.tick(u[sel], [], "small")
    ch = k.tick(u[sel], [par], "small")
    assert sorted(int(w >> 1) for w in ch) == [int(np.nonzero(sel == m)[0][0]) for m in marked]
    for form, new_sel in (("small", np.concatenate([[50], sel])), ("compact", sel[:-5]),
                          ("small", np.concatenate([[7, 8], sel[1:]]))):
        sel = new_sel
        ch = k.tick(u[sel], [], form)
        added = set(int(w >> 1) for w in ch)
        assert all(w & 1 for w in ch)              # only new keys, which come in healthy
        assert all(int(sel[i]) not in set(marked.tolist()) for i in added)
    v = int(marked[3])
    u["flags"][v] = 1
    assert len(k.tick(u[sel], [], "small")) == 0       # a marked vGPU vanishes: no transition
    u["flags"][v] = 0
    ch = k.tick(u[sel], [], "compact")                 # it returns: healthy again, its siblings stay marked
    assert list(ch) == [(int(np.nonzero(sel == v)[0][0]) << 1) | 1]


@pytest.mark.parametrize("form", ["small", "compact"])
@pytest.mark.parametrize("kind", ["mdev", "groups"])
@pytest.mark.parametrize("bad", ["descending", "duplicate", "first_pair", "round_edge"])
def test_unsorted_or_duplicate_keys_are_refused_and_keep_the_list(emu, kind, form, bad):
    n = 13_000
    u, rng = _universe(kind, n, 21)
    k = Keyed(emu, kind)
    xs = _sets(kind, u, rng)[0]
    k.tick(u, xs, form)
    _mutate(kind, u, rng.integers(0, n, 100), rng)
    at = {"descending": 5000, "duplicate": 777, "first_pair": 0,
          "round_edge": (6 if kind == "mdev" else 12) * 1024 - 1}[bad]
    sel = np.arange(n)
    sel[at], sel[at + 1] = (sel[at + 1], sel[at]) if bad != "duplicate" else (sel[at], sel[at])
    prev = (k.prev_key.copy(), k.prev_state.copy(), k.n_prev)
    refused, _, _ = k.raw(u[sel], xs, form)
    assert refused
    assert np.array_equal(k.prev_key, prev[0]) and np.array_equal(k.prev_state, prev[1]) and k.n_prev == prev[2]
    k.tick(u, xs, form)                                # the next valid call sees the state unchanged


@pytest.mark.parametrize("kind", ["mdev", "groups"])
def test_n_zero_resets(emu, kind):
    u, rng = _universe(kind, 3000, 31)
    k = Keyed(emu, kind)
    xs = _sets(kind, u, rng)[0]
    k.tick(u, xs, "small")
    k.tick(u[:0], xs, "compact")
    assert k.n_prev == 0
    ch = k.tick(u, xs, "small")                        # after the reset: every healthy record is new
    want = HK.KeyedMdevRef() if kind == "mdev" else HK.KeyedGroupsRef()
    d = want.rescan(u, N_TYPES, xs) if kind == "mdev" else want.rescan(u, xs)
    assert np.array_equal(ch, d.changed) and all(w & 1 for w in ch)
