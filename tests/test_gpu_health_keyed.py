"""kvg_health_rescan_mdev_keyed and kvg_health_rescan_groups_keyed on the H100 against the dict-keyed state machine of
tests/health_keyed_ref.py, on both sides of every threshold the host uses to pick a kernel (k_health_small<Keyed<Rule>>
up to 32,768 records with kernel timing off, the look-back form above it or with timing on), with pinned snapshots read
in place and pageable ones staged.  Each tick may edit the list (a key inserted at the front, the last dropped, one in
the middle replaced), change records, raise XIDs and remove or restore group nodes.  Also: K1 (a fixed key list gives
the index-keyed call's deltas byte for byte), refusals that keep the list, isolation from the index-keyed states, the
scans and the deltas, and one launch per small-form tick."""
import ctypes as C

import numpy as np
import pytest

import health_groups_ref as HG
import health_keyed_ref as HK
import health_mdev_ref as HM
from oracle import oracle as O

pytestmark = pytest.mark.gpu

SMALL_MAX = 32 * 1024
SIZES = [1, 1000, SMALL_MAX, SMALL_MAX + 1, 65_536, 200_000]
N_TYPES = 200
KINDS = ["mdev", "groups"]


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


def _universe(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "mdev":
        return O.gen_mdev(seed, n), rng
    return HG.make_recs(n, rng, per_group=max(4, -(-n // 4000))), rng


def _events(kind, u, t, rng):
    """The tick's set: XID parents (mdev, a one-shot list), or the groups whose node exists (a standing set with a
    few nodes missing, different ones each tick)."""
    if kind == "mdev":
        parents = np.unique(u["parent"])
        return [int(p) for p in rng.choice(parents, t % 3)] + ([0xfffffff0] if t % 5 == 1 else [])
    groups = np.unique(u["iommu_group"])
    gone = rng.choice(groups, min(len(groups) - 1, 1 + t % 4), replace=False)
    return [int(g) for g in np.setdiff1d(groups, gone)]


def _mutate(kind, u, rng, k):
    idx = rng.integers(0, len(u), k)
    if kind == "mdev":
        u["flags"][idx] ^= rng.integers(0, 4, len(idx)).astype(np.uint8)
    else:
        dead = idx[rng.random(len(idx)) < 0.5]
        HG.kill(u, dead, rng)
        HG.revive(u, np.setdiff1d(idx, dead))


def _edit(sel, n_universe, t, rng):
    e = t % 4
    if e == 0 and sel[0] > 0:
        return np.concatenate([[sel[0] - 1], sel])                       # insert at the front
    if e == 1 and len(sel) > 1:
        return sel[:-1]                                                  # drop the last
    if e == 2 and len(sel) > 2:
        mid = len(sel) // 2
        lo, hi = sel[mid - 1], sel[mid + 1]
        out = np.delete(sel, mid)
        if hi - lo > 2:                                                  # replace the middle by another key
            out = np.insert(out, mid, lo + 1 if sel[mid] != lo + 1 else hi - 1)
        return out
    return sel


class Caller:
    def __init__(self, kv, ctx, kind, pinned, cap):
        self.kv, self.ctx, self.kind = kv, ctx, kind
        self.dtype = kv.MDEV_REC if kind == "mdev" else kv.PCI_REC
        self.buf = None
        if pinned:
            import torch
            self.t = torch.empty(cap * self.dtype.itemsize, dtype=torch.uint8, pin_memory=True)
            self.buf = self.t.numpy().view(self.dtype)

    def place(self, recs):
        if self.buf is None:
            return np.ascontiguousarray(recs)
        out = self.buf[:len(recs)]
        out[:] = recs
        return out

    def keyed(self, recs, xs):
        if self.kind == "mdev":
            return self.ctx.health_rescan_mdev_keyed(self.place(recs), N_TYPES, xs)
        return self.ctx.health_rescan_groups_keyed(self.place(recs), xs)

    def index(self, recs, xs):
        if self.kind == "mdev":
            return self.ctx.health_rescan_mdev(self.place(recs), N_TYPES, xs)
        return self.ctx.health_rescan_groups(self.place(recs), xs)


def _ref(kind):
    return HK.KeyedMdevRef() if kind == "mdev" else HK.KeyedGroupsRef()


def _want(ref, kind, recs, xs):
    return ref.rescan(recs, N_TYPES, xs) if kind == "mdev" else ref.rescan(recs, xs)


def _check(d, want, what):
    assert d.n_records == want.n_records and d.n_alive == want.n_alive, what
    assert np.array_equal(d.changed, want.changed), (what, len(d.changed), len(want.changed))


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", KINDS)
def test_keyed_sequences_match_the_state_machine(kv, kind, n, pinned):
    u, rng = _universe(kind, n + 64, 7 + n % 101 + pinned)
    with kv.Context(0) as ctx:
        c = Caller(kv, ctx, kind, pinned, n + 64)
        ref = _ref(kind)
        sel = np.arange(32, 32 + n)
        label = "health_%s_keyed_compact" % kind
        for t in range(50):
            if t:
                _mutate(kind, u, rng, 8 + n // 500)
                sel = _edit(sel, len(u), t, rng)
            xs = _events(kind, u, t, rng)
            timed = t % 7 == 3                                          # the look-back form at every size
            if timed:
                ctx.set_kernel_timing(True)
            d = c.keyed(u[sel], xs)
            if timed:
                labels = {name for name, _ in ctx.kernel_times(1 << 16)}
                ctx.set_kernel_timing(False)
                assert label in labels and "health_%s_keyed_small" % kind not in labels, sorted(labels)
            _check(d, _want(ref, kind, u[sel], xs), (kind, n, pinned, t))


@pytest.mark.parametrize("n", [1000, SMALL_MAX, SMALL_MAX + 1, 200_000])
@pytest.mark.parametrize("kind", KINDS)
def test_k1_fixed_key_list_gives_the_index_keyed_deltas(kv, kind, n):
    u, rng = _universe(kind, n, 3 + n % 7)
    with kv.Context(0) as ctx:
        c = Caller(kv, ctx, kind, False, n)
        for t in range(6):
            if t:
                _mutate(kind, u, rng, 20 + n // 300)
            xs = _events(kind, u, t, rng)
            a, b = c.keyed(u, xs), c.index(u, xs)
            assert (a.n_records, a.n_alive) == (b.n_records, b.n_alive), t
            assert a.changed.tobytes() == b.changed.tobytes(), t


@pytest.mark.parametrize("n", [5000, 50_000])
@pytest.mark.parametrize("kind", KINDS)
def test_refusals_keep_the_list(kv, kind, n):
    lib = kv.load()
    u, rng = _universe(kind, n, 41)
    with kv.Context(0) as ctx:
        c = Caller(kv, ctx, kind, False, n)
        ref = _ref(kind)
        xs = _events(kind, u, 1, rng)
        _check(c.keyed(u, xs), _want(ref, kind, u, xs), "first")
        _mutate(kind, u, rng, 200)
        for at, dup in ((n // 3, False), (n - 2, True), (0, False)):   # unsorted, duplicate, the first pair
            sel = np.arange(n)
            sel[at], sel[at + 1] = (sel[at], sel[at]) if dup else (sel[at + 1], sel[at])
            with pytest.raises(kv.KvgError) as e:
                c.keyed(u[sel], xs)
            assert e.value.rc == kv._lib.KVG_EINVAL and "ascending" in str(e.value)
        cap = 1024 if kind == "mdev" else 4096                          # KVG_HEALTH_MAX_XID / KVG_HEALTH_MAX_GROUPS
        with pytest.raises(kv.KvgError) as e:
            c.keyed(u, np.arange(cap + 1, dtype=np.uint32))
        assert e.value.rc == kv._lib.KVG_EINVAL
        res = C.POINTER(kv._lib.HealthDeltaC)()
        buf = np.ascontiguousarray(u)
        if kind == "mdev":
            rc = lib.kvg_health_rescan_mdev_keyed(ctx.handle, buf.ctypes.data, n, N_TYPES, None, 3, C.byref(res))
        else:
            rc = lib.kvg_health_rescan_groups_keyed(ctx.handle, buf.ctypes.data, n, None, 3, C.byref(res))
        assert rc == -1
        _check(c.keyed(u, xs), _want(ref, kind, u, xs), "after")        # continues from the first call's list
        d = c.keyed(u[:0], xs)                                          # n = 0: the reset
        assert (d.n_records, d.n_alive, len(d.changed)) == (0, 0, 0)
        ref.reset()
        _check(c.keyed(u, xs), _want(ref, kind, u, xs), "reset")


@pytest.mark.parametrize("kind", KINDS)
def test_keyed_state_is_isolated(kv, kind):
    """Index-keyed ticks of the same kind and their resets, PCI health ticks, delta scans and a pci.ids load between
    keyed ticks change neither the keyed list nor the index-keyed state."""
    import util
    text = util.pciids_text()
    ids = O.nv_ids(text)
    u, rng = _universe(kind, 20_000, 9)
    with kv.Context(0) as ctx:
        ctx.pciids_load(text)
        c = Caller(kv, ctx, kind, False, 20_000)
        kref = _ref(kind)
        iref = HM.HealthMdevRef() if kind == "mdev" else HG.HealthGroupsRef()
        sel = np.arange(100, 19_000)
        precs = O.gen_pci(2, 12_000, ids, 0)
        types = O.gen_type_names(N_TYPES)
        for t in range(6):
            _mutate(kind, u, rng, 60)
            sel = _edit(sel, len(u), t, rng)
            xs = _events(kind, u, t, rng)
            _check(c.keyed(u[sel], xs), _want(kref, kind, u[sel], xs), ("keyed", t))
            iw = iref.rescan(u, N_TYPES, xs) if kind == "mdev" else iref.rescan(u, xs)
            _check(c.index(u, xs), iw, ("index", t))
            ctx.health_rescan(precs)
            ctx.scan_mdev_delta(O.gen_mdev(t, 3000), types)
            ctx.scan_pci_delta(precs)
            ctx.pciids_load(text)
            if t == 3:                                                  # resets the index-keyed state only
                (ctx.health_mdev_reset if kind == "mdev" else ctx.health_groups_reset)()
                iref.reset()
                ctx.scan_pci_delta_reset()


@pytest.mark.parametrize("kind", KINDS)
def test_small_form_tick_is_one_launch(kv, kind):
    u, rng = _universe(kind, SMALL_MAX, 2)
    with kv.Context(0) as ctx:
        c = Caller(kv, ctx, kind, False, SMALL_MAX)
        c.keyed(u[1:], _events(kind, u, 0, rng))
        before = ctx.launch_count
        c.keyed(u, _events(kind, u, 1, rng))                            # a key inserted at the front: the miss path
        assert ctx.launch_count - before == 1
