"""kvg_health_rescan_mdev on the H100 against the numpy state machine of tests/health_mdev_ref.py, on both sides of
every threshold the host uses to pick a kernel: k_health_small<MdevHealthRule> up to 32,768 records with kernel timing
off (6 rows of 1024 records per TMA round), k_compact<HealthOp<MdevHealthRule>, 256, 8> above it or with timing on, on
the same state.  Pinned snapshots are changed in place and read in place; pageable ones are staged.  Also: the state is
separate from the PCI health state and from every scan, delta and pci.ids load; bad XID lists are refused and leave
the state as it was."""
import ctypes as C

import numpy as np
import pytest

import health_mdev_ref as H
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ROUND = 6 * 1024
SMALL_MAX = 32 * 1024
SIZES = [1, ROUND, ROUND + 1, 2 * ROUND + 1, SMALL_MAX, SMALL_MAX + 1, 100_000]
N_TYPES = 200


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


def _flip_points(n, rng):
    edges = [0, n - 1]
    for b in (1024, ROUND, 2 * ROUND, 2048, SMALL_MAX):
        edges += [b - 1, b, b + 1]
    pts = [p for p in edges if 0 <= p < n] + list(rng.integers(0, n, 8))
    return np.unique(np.array(pts, dtype=np.int64))


def _check(d, want, n, what):
    assert d.n_records == n and d.n_alive == want.n_alive, what
    assert np.array_equal(d.changed, want.changed), (what, len(d.changed), len(want.changed))


@pytest.mark.parametrize("pinned", [False, True])
def test_health_mdev_regimes(kv, pinned):
    import torch
    ctx = kv.Context(0)
    rng = np.random.default_rng(23 + pinned)
    keep = []
    try:
        ref = H.HealthMdevRef()
        ctx.health_mdev_reset()
        for n in SIZES + [ROUND, 1]:                   # every new size re-arms
            if pinned:
                t = torch.empty(n * 32, dtype=torch.uint8, pin_memory=True)
                keep.append(t)
                recs = t.numpy().view(kv.MDEV_REC)
                recs[:] = O.gen_mdev(n, n)
            else:
                recs = O.gen_mdev(n, n)
            parents = np.unique(recs["parent"])
            for tick in range(5):
                xids = []
                if tick:
                    f = _flip_points(n, rng)
                    recs["flags"][f] ^= rng.integers(0, 4, len(f)).astype(np.uint8)
                    xids = [int(parents[tick % len(parents)]), int(parents[0]), 0xfffffff0][:tick]
                timed = tick == 2
                if timed:
                    ctx.set_kernel_timing(True)
                d = ctx.health_rescan_mdev(recs, N_TYPES, xids)
                if timed:
                    labels = {name for name, _ in ctx.kernel_times(1 << 16)}
                    ctx.set_kernel_timing(False)
                    assert "health_mdev_compact" in labels and "health_mdev_small" not in labels, sorted(labels)
                _check(d, ref.rescan(recs, N_TYPES, xids), n, (n, tick))
        ctx.health_mdev_reset()
        d = ctx.health_rescan_mdev(np.zeros(0, dtype=kv.MDEV_REC), N_TYPES)
        assert (d.n_records, d.n_alive, len(d.changed)) == (0, 0, 0)
    finally:
        torch.cuda.synchronize()
        ctx.close()
        del keep


def test_small_path_is_one_launch(kv):
    """An untimed tick of 32,768 records is one kernel launch and nothing else (kernel timing would move it to the
    look-back form, so the launch count shows the path)."""
    with kv.Context(0) as ctx:
        recs = O.gen_mdev(0, SMALL_MAX)
        ctx.health_rescan_mdev(recs, N_TYPES)
        before = ctx.launch_count
        ctx.health_rescan_mdev(recs, N_TYPES, [int(recs["parent"][5])])
        assert ctx.launch_count - before == 1


def test_health_mdev_state_is_isolated(kv):
    """PCI health ticks, an mdev delta scan and a pci.ids load between vGPU health ticks change neither state."""
    text = util.pciids_text()
    ids = O.nv_ids(text)
    rng = np.random.default_rng(4)
    with kv.Context(0) as ctx:
        ctx.pciids_load(text)
        mref, pprev = H.HealthMdevRef(), None
        mrecs = O.gen_mdev(1, 20_000)
        precs = O.gen_pci(2, 12_000, ids, 0)
        types = O.gen_type_names(N_TYPES)
        parents = np.unique(mrecs["parent"])
        for tick in range(4):
            mrecs["flags"][rng.integers(0, len(mrecs), 12)] ^= 2
            precs["driver"][rng.integers(0, len(precs), 12)] = rng.integers(0, 5, 12)
            xids = [int(parents[3 * tick])]
            _check(ctx.health_rescan_mdev(mrecs, N_TYPES, xids), mref.rescan(mrecs, N_TYPES, xids), len(mrecs), tick)
            d = ctx.health_rescan(precs)
            now = util.pci_alive(precs)
            prev = np.zeros(len(precs), dtype=bool) if pprev is None else pprev
            idx = np.nonzero(now != prev)[0]
            assert np.array_equal(d.changed, (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)), tick
            pprev = now
            ctx.scan_mdev_delta(mrecs, types)
            ctx.pciids_load(text)
            if tick == 2:                               # re-arms the PCI state only
                ctx.health_reset()
                pprev = None


def test_bad_xid_lists_are_refused(kv):
    lib = kv.load()
    with kv.Context(0) as ctx:
        ref = H.HealthMdevRef()
        recs = O.gen_mdev(5, 5000)
        parents = np.unique(recs["parent"])
        _check(ctx.health_rescan_mdev(recs, N_TYPES, [int(parents[1])]), ref.rescan(recs, N_TYPES, [int(parents[1])]),
               5000, "arm")
        with pytest.raises(kv.KvgError) as e:
            ctx.health_rescan_mdev(recs, N_TYPES, np.arange(1025, dtype=np.uint32))
        assert e.value.rc == kv._lib.KVG_EINVAL
        res = C.POINTER(kv._lib.HealthDeltaC)()
        buf = np.ascontiguousarray(recs)
        assert lib.kvg_health_rescan_mdev(ctx.handle, buf.ctypes.data, len(recs), N_TYPES, None, 3, C.byref(res)) == -1
        # the state is as it was: the next tick continues from the armed one
        recs["flags"][:40] ^= 1
        _check(ctx.health_rescan_mdev(recs, N_TYPES, [int(parents[2])]), ref.rescan(recs, N_TYPES, [int(parents[2])]),
               5000, "after")
