"""kvg_health_rescan_groups on the H100 against the numpy state machine of tests/health_groups_ref.py, on both sides of
every threshold the host uses to pick a kernel: k_health_small<GroupHealthRule> up to 32,768 records with kernel
timing off, k_compact<HealthOp<GroupHealthRule>, 256, 8> above it or with timing on, on the same state.  Pinned
snapshots are changed in place and read in place; pageable ones are staged.  Also: P1 against kvg_health_rescan on a second
context, P2 with every record alive, the 4,096-handle cap, re-arming, and the state kept apart from the PCI and vGPU
health states and from every scan, delta and pci.ids load in both directions."""
import ctypes as C

import numpy as np
import pytest

import health_groups_ref as H
import health_mdev_ref
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

SMALL_MAX = 32 * 1024
SIZES = [1, 1023, SMALL_MAX, SMALL_MAX + 1, 100_000]
CAP = 4096


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


def _per_group(n):
    return max(4, -(-n // CAP))


def _check(d, want, n, what):
    assert d.n_records == n and d.n_alive == want.n_alive, what
    assert np.array_equal(d.changed, want.changed), (what, len(d.changed), len(want.changed))


def _node_sets(groups, rng):
    """One tick's raw node list per entry (at most CAP handles, duplicates and foreign handles included)."""
    gone = rng.choice(groups, max(1, len(groups) // 5), replace=False)
    kept = np.setdiff1d(groups, gone)
    return [
        groups,
        list(kept[::-1]) + [int(g) for g in kept[:1]] * 2 + [0, 0xFFFFFFF0],
        [],
        [int(groups[len(groups) // 2])],
        rng.permutation(groups),
    ]


@pytest.mark.parametrize("pinned", [False, True])
def test_health_groups_regimes(kv, pinned):
    import torch
    ctx = kv.Context(0)
    rng = np.random.default_rng(31 + pinned)
    keep = []
    try:
        ref = H.HealthGroupsRef()
        ctx.health_groups_reset()
        for n in SIZES + [1023]:                       # every new size re-arms
            base = H.make_recs(n, rng, _per_group(n))
            if pinned:
                t = torch.empty(n * 16, dtype=torch.uint8, pin_memory=True)
                keep.append(t)
                recs = t.numpy().view(kv.PCI_REC)
                recs[:] = base
            else:
                recs = base
            groups = np.unique(recs["iommu_group"])
            for tick, nodes in enumerate(_node_sets(groups, rng)):
                if tick:
                    f = rng.integers(0, n, 24)
                    H.kill(recs, f[:12], rng)
                    H.revive(recs, f[12:])
                timed = tick == 2
                if timed:
                    ctx.set_kernel_timing(True)
                d = ctx.health_rescan_groups(recs, nodes)
                if timed:
                    labels = {name for name, _ in ctx.kernel_times(1 << 16)}
                    ctx.set_kernel_timing(False)
                    assert "health_groups_compact" in labels and "health_groups_small" not in labels, sorted(labels)
                _check(d, ref.rescan(recs, nodes), n, (n, tick))
        ctx.health_groups_reset()
        d = ctx.health_rescan_groups(np.zeros(0, dtype=kv.PCI_REC), [1, 2])
        assert (d.n_records, d.n_alive, len(d.changed)) == (0, 0, 0)
    finally:
        torch.cuda.synchronize()
        ctx.close()
        del keep


@pytest.mark.parametrize("n", [10_000, 50_000])
def test_every_node_present_is_kvg_health_rescan(kv, n):
    """P1: with a node for every group, the deltas are kvg_health_rescan's on the same snapshots (second context)."""
    rng = np.random.default_rng(n)
    recs = H.make_recs(n, rng, _per_group(n), alive_frac=0.7)
    with kv.Context(0) as a, kv.Context(0) as b:
        for tick in range(5):
            if tick:
                f = rng.integers(0, n, 40)
                H.kill(recs, f[:20], rng)
                H.revive(recs, f[20:])
            g = a.health_rescan_groups(recs, np.unique(recs["iommu_group"]))
            p = b.health_rescan(recs)
            assert (g.n_records, g.n_alive) == (p.n_records, p.n_alive) and np.array_equal(g.changed, p.changed), tick


@pytest.mark.parametrize("n", [10_000, 50_000])
def test_a_group_flips_as_a_whole(kv, n):
    """P2: every record alive; a vanished node turns every device of its group unhealthy, its return healthy."""
    rng = np.random.default_rng(n + 1)
    recs = H.make_recs(n, rng, _per_group(n), alive_frac=1.0)
    groups = np.unique(recs["iommu_group"])
    with kv.Context(0) as ctx:
        d = ctx.health_rescan_groups(recs, groups)
        assert d.n_alive == len(recs) and len(d.changed) == len(recs)
        g = int(groups[777])
        members = np.nonzero(recs["iommu_group"] == g)[0].astype(np.uint32)
        d = ctx.health_rescan_groups(recs, np.setdiff1d(groups, [g]))
        assert np.array_equal(d.changed, members << 1) and d.n_alive == len(recs) - len(members)
        d = ctx.health_rescan_groups(recs, groups)
        assert np.array_equal(d.changed, (members << 1) | 1) and d.n_alive == len(recs)


def test_small_path_is_one_launch(kv):
    """An untimed tick of 32,768 records is one kernel launch and nothing else (kernel timing would move it to the
    look-back form, so the launch count shows the path)."""
    rng = np.random.default_rng(3)
    recs = H.make_recs(SMALL_MAX, rng, 8)
    groups = np.unique(recs["iommu_group"])
    with kv.Context(0) as ctx:
        ctx.health_rescan_groups(recs, groups)
        for nodes in (groups[1:], groups):
            before = ctx.launch_count
            ctx.health_rescan_groups(recs, nodes)
            assert ctx.launch_count - before == 1


@pytest.mark.parametrize("n", [5000, 40_000])
def test_node_sets_at_the_cap_and_refused(kv, n):
    lib = kv.load()
    rng = np.random.default_rng(n + 2)
    recs = H.make_recs(n, rng, _per_group(n))
    groups = np.unique(recs["iommu_group"])
    full = np.concatenate([groups, np.setdiff1d(np.arange(1, 3 * CAP, dtype=np.uint32), groups)[:CAP - len(groups)]])
    assert len(full) == CAP
    with kv.Context(0) as ctx:
        ref = H.HealthGroupsRef()
        _check(ctx.health_rescan_groups(recs, full), ref.rescan(recs, full), n, "cap")
        H.kill(recs, rng.integers(0, n, 30), rng)
        with pytest.raises(kv.KvgError) as e:
            ctx.health_rescan_groups(recs, np.arange(1, CAP + 2, dtype=np.uint32))
        assert e.value.rc == kv._lib.KVG_EINVAL
        res = C.POINTER(kv._lib.HealthDeltaC)()
        buf = np.ascontiguousarray(recs)
        assert lib.kvg_health_rescan_groups(ctx.handle, buf.ctypes.data, n, None, 3, C.byref(res)) == kv._lib.KVG_EINVAL
        # the state is as it was: the next tick continues from the one before the refusals
        _check(ctx.health_rescan_groups(recs, groups[::2]), ref.rescan(recs, groups[::2]), n, "after")


def test_rearm_on_reset_and_on_a_new_size(kv):
    rng = np.random.default_rng(9)
    recs = H.make_recs(3000, rng)
    groups = np.unique(recs["iommu_group"])
    with kv.Context(0) as ctx:
        ctx.health_rescan_groups(recs, groups)
        assert len(ctx.health_rescan_groups(recs, groups).changed) == 0
        ctx.health_groups_reset()
        d = ctx.health_rescan_groups(recs, groups)                      # everything healthy is a transition again
        assert np.array_equal(d.changed, (np.nonzero(util.pci_alive(recs))[0].astype(np.uint32) << 1) | 1)
        d = ctx.health_rescan_groups(recs[:2999], groups)               # a new n re-arms
        assert len(d.changed) == d.n_alive == int(util.pci_alive(recs[:2999]).sum())


def test_health_groups_state_is_isolated(kv):
    """PCI and vGPU health ticks, their resets, scans, deltas and a pci.ids load between group ticks change no
    state but their own, in both directions."""
    text = util.pciids_text()
    ids = O.nv_ids(text)
    rng = np.random.default_rng(4)
    n_types = 200
    with kv.Context(0) as ctx:
        ctx.pciids_load(text)
        gref, mref, pprev = H.HealthGroupsRef(), health_mdev_ref.HealthMdevRef(), None
        grecs = H.make_recs(20_000, rng, 5)
        groups = np.unique(grecs["iommu_group"])
        mrecs = O.gen_mdev(1, 20_000)
        precs = O.gen_pci(2, 12_000, ids, 0)
        types = O.gen_type_names(n_types)
        for tick in range(5):
            H.kill(grecs, rng.integers(0, len(grecs), 12), rng)
            mrecs["flags"][rng.integers(0, len(mrecs), 12)] ^= 2
            precs["driver"][rng.integers(0, len(precs), 12)] = rng.integers(0, 5, 12)
            nodes = np.setdiff1d(groups, groups[tick * 11:tick * 11 + 5])
            _check(ctx.health_rescan_groups(grecs, nodes), gref.rescan(grecs, nodes), len(grecs), ("groups", tick))
            xids = [int(mrecs["parent"][tick])]
            _check(ctx.health_rescan_mdev(mrecs, n_types, xids), mref.rescan(mrecs, n_types, xids), len(mrecs),
                   ("mdev", tick))
            d = ctx.health_rescan(precs)
            now = util.pci_alive(precs)
            prev = np.zeros(len(precs), dtype=bool) if pprev is None else pprev
            idx = np.nonzero(now != prev)[0]
            assert np.array_equal(d.changed, (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)), tick
            pprev = now
            ctx.scan_pci(precs)
            ctx.scan_pci_delta(precs)
            ctx.scan_mdev_delta(mrecs, types)
            ctx.pciids_load(text)
            if tick == 2:                               # re-arms the PCI and vGPU states only
                ctx.health_reset()
                ctx.health_mdev_reset()
                mref.reset()
                pprev = None
