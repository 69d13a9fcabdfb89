"""The mdev re-scan delta (kvg_scan_mdev_delta, K7) on the H100: sequences of snapshots with hot-added and destroyed
mdevs, retypes, parent moves, NUMA changes and a reordered dictionary at about 0.1 % of the records per step, at
4,096 records, 65,536 (config 3) and just over 2 Mi.  Every step must return exactly what kvg_scan_mdev returns, the
exact delta of mdev_delta_ref.expect_mdev_delta, and maps patched by apply_mdev_delta that dump like maps rebuilt from
scratch.  Every test here needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

import delta_ref
import mdev_delta_ref
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

Mi = 1 << 20
NT = 256


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


@pytest.fixture(scope="module")
def ctx(kv):
    c = kv.Context(0)
    c.pciids_load(util.pciids_text())
    yield c
    c.close()


def snapshot(n, seed=1, nt=NT):
    """n synthetic mdev records with canonical UUIDs spaced by 4 in their first word (room for hot-adds in between),
    packed-BDF parents and types of an nt-entry dictionary."""
    recs = O.gen_mdev(seed, n)
    recs["uuid"][:, :4] = (np.arange(n, dtype=np.uint32) * 4).astype(">u4").view(np.uint8).reshape(n, 4)
    recs["type_idx"] %= nt
    return recs


def step(recs, types, kind, rng):
    """One snapshot later (about 0.1 % of the records); returns (recs, raw type names)."""
    r = recs.copy()
    k = max(1, len(r) // 1000)
    pick = rng.choice(len(r), k, replace=False)
    if kind == "hot_add":
        add = r[pick].copy()
        add["uuid"][:, 15] ^= 0x5a                     # differs from its neighbour in the last byte only
        add["uuid"][:, 3] += 1 + (rng.integers(0, 3, k)).astype(np.uint8)
        add["flags"] = 0
        key = lambda a: np.ascontiguousarray(a["uuid"]).view("V16").ravel()
        add = add[~np.isin(key(add), key(r))]
        add = add[np.unique(key(add), return_index=True)[1]]
        both = np.concatenate([r, add])
        return both[np.argsort(key(both), kind="stable")], types
    if kind == "destroy":
        return np.delete(r, pick), types
    if kind == "retype":
        r["type_idx"][pick] = rng.integers(0, len(types), k)
    elif kind == "reparent":
        r["parent"][pick] = r["parent"][rng.choice(len(r), k)]
    elif kind == "numa":
        r["parent_numa"][pick] = (r["parent_numa"][pick] + 1) % 4
    elif kind == "reorder":                            # the same labels under other raw indices
        perm = rng.permutation(len(types))
        inv = np.argsort(perm)
        types = [types[i] for i in perm]
        r["type_idx"] = inv[r["type_idx"]]
    return r, types


KINDS = ("hot_add", "destroy", "retype", "reparent", "numa", "reorder")


def same_result(a, b):
    for f in ("n_records", "survivors", "type_keys", "type_off", "type_perm", "labels", "type_canon", "type_names",
              "par_keys", "par_off", "par_perm"):
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def check_delta(kv, got, prev, now, n_prev=None):
    want = mdev_delta_ref.expect_mdev_delta(prev.survivors, now.survivors, prev.labels, now.labels, kv.MDEV_CHANGE)
    assert got.n_prev == (len(prev.survivors) if n_prev is None else n_prev)
    for f in ("changes", "type_dirty", "par_dirty", "par_gone"):
        assert np.array_equal(getattr(got, f), want[f]), f
    assert got.type_gone == want["type_gone"]


def empty(kv):
    return kv.MdevResult(0, np.zeros(0, kv.MDEV_SURV), *([np.zeros(0, np.uint32)] * 3), [], np.zeros(0, np.uint16), [],
                         *([np.zeros(0, np.uint32)] * 3))


@pytest.mark.parametrize("n", [4096, 65_536, 2 * Mi + 1000])
def test_snapshot_sequence_matches_reference(kv, ctx, n):
    rng = np.random.default_rng(n)
    recs, types = snapshot(n), O.gen_type_names(NT)
    ctx.scan_mdev_delta_reset()
    res, delta = ctx.scan_mdev_delta(recs, types)
    same_result(res, ctx.scan_mdev(recs, types))
    assert (delta.changes["what"] == kv._lib.CH_ADDED).all()
    check_delta(kv, delta, empty(kv), res, n_prev=0)
    maps = kv.mdev_maps_from_result(res)
    shared = maps.gpuVgpuMap
    prev = res
    for kind in KINDS:
        recs, types = step(recs, types, kind, rng)
        res, delta = ctx.scan_mdev_delta(recs, types)
        same_result(res, ctx.scan_mdev(recs, types))
        check_delta(kv, delta, prev, res)
        assert (len(delta.changes) > 0) == (kind != "reorder"), kind
        touched = kv.apply_mdev_delta(maps, res, delta)
        assert maps.gpuVgpuMap is shared
        assert kv.canonical_dump(maps) == kv.canonical_dump(kv.mdev_maps_from_result(res)), kind
        assert len(touched.type_dirty) == len(delta.type_dirty) and len(touched.par_gone) == len(delta.par_gone)
        prev = res


def test_first_call_and_reset_report_everything_added(kv, ctx):
    recs, types = snapshot(20_000, seed=3), O.gen_type_names(NT)
    ctx.scan_mdev_delta_reset()
    res, d0 = ctx.scan_mdev_delta(recs, types)
    assert d0.n_prev == 0 and len(d0.changes) == len(res.survivors)
    assert len(d0.type_dirty) == len(res.type_keys) and len(d0.par_dirty) == len(res.par_keys)
    assert d0.type_gone == [] and len(d0.par_gone) == 0
    _, d1 = ctx.scan_mdev_delta(recs, types)
    assert d1.n_prev == len(res.survivors) and len(d1.changes) == 0 and len(d1.type_dirty) == 0
    ctx.scan_mdev_delta_reset()
    _, d2 = ctx.scan_mdev_delta(recs, types)
    check_delta(kv, d2, empty(kv), res, n_prev=0)
    ctx.scan_mdev_delta_reset()
    res_e, de = ctx.scan_mdev_delta(recs[:0], types)
    assert len(res_e.survivors) == 0 and de.n_prev == 0 and len(de.changes) == 0
    _, d3 = ctx.scan_mdev_delta(recs, types)          # from an empty previous result
    check_delta(kv, d3, res_e, res)


def test_other_calls_leave_both_previous_results_alone(kv, ctx):
    rng = np.random.default_rng(7)
    ids = O.nv_ids(util.pciids_text())
    a, types = snapshot(50_000, seed=4), O.gen_type_names(NT)
    p = O.gen_pci(2, 30_000, ids, 16)
    p["addr"] = np.arange(len(p), dtype=np.uint32) * 4
    ctx.scan_mdev_delta_reset()
    ctx.scan_pci_delta_reset()
    ra, _ = ctx.scan_mdev_delta(a, types)
    ctx.scan_pci_delta(p)
    ctx.scan_pci(O.gen_pci(9, 300_000, ids, 16))
    ctx.scan_mdev(snapshot(200_000, seed=9), O.gen_type_names(1000))
    ctx.health_rescan(p[:20_000])
    ctx.pciids_load(util.pciids_text())
    c, types = step(a, types, "retype", rng)
    rc, dc = ctx.scan_mdev_delta(c, types)
    check_delta(kv, dc, ra, rc)
    # and mdev delta calls in between leave the PCI delta's previous result alone
    rp2, _ = ctx.scan_pci_delta(p)
    ctx.scan_mdev_delta(snapshot(10_000, seed=5), types)
    rp3, dp3 = ctx.scan_pci_delta(p[::3].copy())
    w = delta_ref.expect_pci_delta(rp2.survivors, rp3.survivors, kv.PCI_CHANGE)
    assert np.array_equal(dp3.changes, w["changes"]) and np.array_equal(dp3.dev_gone, w["dev_gone"])


def test_refusals_keep_the_previous_result(kv, ctx):
    rng = np.random.default_rng(8)
    a, types = snapshot(40_000, seed=5), O.gen_type_names(NT)
    ctx.scan_mdev_delta_reset()
    ra, _ = ctx.scan_mdev_delta(a, types)
    alive = np.nonzero((a["flags"] & 3) == 0)[0]
    bad = a.copy()
    bad["uuid"][alive[5000]] = bad["uuid"][alive[4999]]      # two survivors with one UUID
    with pytest.raises(kv.KvgError) as e:
        ctx.scan_mdev_delta(bad, types)
    assert e.value.rc == -1 and "ascending" in str(e.value)
    swapped = a.copy()
    far = alive[len(alive) // 2]
    swapped["uuid"][[alive[100], far]] = a["uuid"][[far, alive[100]]]
    with pytest.raises(kv.KvgError):
        ctx.scan_mdev_delta(swapped, types)
    with pytest.raises(kv.KvgError) as e:
        ctx.scan_mdev_delta(a, [b"t%05d" % k for k in range(65_536)])
    assert e.value.rc == -6
    c, types = step(a, types, "destroy", rng)
    rc, dc = ctx.scan_mdev_delta(c, types)
    check_delta(kv, dc, ra, rc)


def test_65535_distinct_labels_on_both_sides(kv, ctx):
    rng = np.random.default_rng(9)
    n, nt = 300_000, 65_535
    t0 = [b"GRID T%05d\n" % k for k in range(nt)]
    t1 = [b"GRID T%05d\n" % k if k % 3 else b"NVIDIA U%05d" % k for k in range(nt)]   # two thirds shared
    t1 = [t1[i] for i in rng.permutation(nt)]
    recs = snapshot(n, seed=11, nt=nt)
    recs["type_idx"] = rng.integers(0, nt, n)
    ctx.scan_mdev_delta_reset()
    r0, _ = ctx.scan_mdev_delta(recs, t0)
    r1, d1 = ctx.scan_mdev_delta(recs, t1)
    same_result(r1, ctx.scan_mdev(recs, t1))
    check_delta(kv, d1, r0, r1)
    assert len(d1.type_gone) > 10_000 and len(d1.changes) > 0


@pytest.mark.parametrize("n", [4096, 1 * Mi])
def test_launch_budget_and_labels(kv, ctx, n):
    """Exactly three launches beyond kvg_scan_mdev on the same input, each under a stable label."""
    recs, types = snapshot(n, seed=6), O.gen_type_names(NT)
    ctx.scan_mdev(recs, types)                 # the radix pass-set hint settles on this input
    c0 = ctx.launch_count
    ctx.scan_mdev(recs, types)
    c1 = ctx.launch_count
    ctx.scan_mdev_delta(recs, types)
    c2 = ctx.launch_count
    assert (c2 - c1) - (c1 - c0) == 3
    ctx.set_kernel_timing(True)
    try:
        ctx.scan_mdev_delta(recs, types)
        labels = [name for name, _ in ctx.kernel_times()]
    finally:
        ctx.set_kernel_timing(False)
    assert labels[-3:] == ["mdev_delta_types", "mdev_delta_merge", "mdev_delta_lists"]
