"""The re-scan delta (kvg_scan_pci_delta, K7) on the H100: sequences of snapshots with hot-adds, hot-removes,
driver re-binds, regroups, device-id and NUMA changes at about 0.1 % of the records per step, at 10 k records (one
copy), 200 k (pipelined) and just over 2 Mi (split classify and final steps).  Every step must return exactly what
kvg_scan_pci returns, the exact delta of delta_ref.expect_pci_delta, and maps patched by apply_pci_delta that dump like
maps rebuilt from scratch.  Every test here needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

import delta_ref
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

Mi = 1 << 20


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


@pytest.fixture(scope="module")
def pciids():
    return util.pciids_text()


@pytest.fixture(scope="module")
def ids(pciids):
    return O.nv_ids(pciids)


@pytest.fixture(scope="module")
def ctx(kv, pciids):
    c = kv.Context(0)
    c.pciids_load(pciids)
    yield c
    c.close()


def snapshot(n, ids, seed=1):
    """n synthetic records with packed-BDF-like handles spaced by 4, so that hot-adds have room in between."""
    recs = O.gen_pci(seed, n, ids, 16)
    recs["addr"] = np.arange(n, dtype=np.uint32) * 4
    return recs


def step(recs, kind, rng, ids):
    """One snapshot later: about 0.1 % of the records hot-added, hot-removed, re-bound, regrouped, re-identified or
    moved to another NUMA node."""
    r = recs.copy()
    k = max(1, len(r) // 1000)
    pick = rng.choice(np.nonzero(util.pci_alive(r))[0], k, replace=False)   # records that survive now
    if kind == "hot_add":
        add = r[pick].copy()
        add["addr"] += 1 + rng.integers(0, 3, k).astype(np.uint32)
        add["vendor"], add["driver"], add["flags"] = 0x10DE, 1, 0
        add = add[~np.isin(add["addr"], r["addr"])]
        return np.sort(np.concatenate([r, add]), order="addr", kind="stable")
    if kind == "hot_remove":
        return np.delete(r, pick)
    if kind == "rebind":
        r["driver"][pick] = 3                                 # bound to another driver: no longer advertised
    elif kind == "regroup":
        r["iommu_group"][pick] = rng.integers(0, 1 << 20, k)
    elif kind == "device":
        r["device"][pick] = rng.choice(ids, k)
    elif kind == "numa":
        r["numa"][pick] = (r["numa"][pick] + 1) % 4
    return r


KINDS = ("hot_add", "hot_remove", "rebind", "regroup", "device", "numa")


def same_result(a, b):
    for f in ("n_records", "survivors", "dev_keys", "dev_off", "dev_perm", "dev_name_slot", "grp_keys", "grp_off",
              "grp_perm", "name_pool"):
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def check_delta(kv, got, prev_surv, now_surv, n_prev=None):
    want = delta_ref.expect_pci_delta(prev_surv, now_surv, kv.PCI_CHANGE)
    assert got.n_prev == (len(prev_surv) if n_prev is None else n_prev)
    for f in ("changes", "dev_dirty", "dev_gone", "grp_dirty", "grp_gone"):
        assert np.array_equal(getattr(got, f), want[f]), f


@pytest.mark.parametrize("n", [10_000, 200_000, 2 * Mi + 1000])
def test_snapshot_sequence_matches_reference(kv, ctx, ids, n):
    rng = np.random.default_rng(n)
    recs = snapshot(n, ids)
    ctx.scan_pci_delta_reset()
    res, delta = ctx.scan_pci_delta(recs)
    same_result(res, ctx.scan_pci(recs))
    assert (delta.changes["what"] == kv._lib.CH_ADDED).all()
    check_delta(kv, delta, res.survivors[:0], res.survivors, n_prev=0)
    maps = kv.pci_maps_from_result(res)
    prev = res
    for kind in KINDS:
        recs = step(recs, kind, rng, ids)
        res, delta = ctx.scan_pci_delta(recs)
        same_result(res, ctx.scan_pci(recs))
        check_delta(kv, delta, prev.survivors, res.survivors)
        assert len(delta.changes) > 0, kind
        touched = kv.apply_pci_delta(maps, res, delta)
        assert kv.canonical_dump(maps) == kv.canonical_dump(kv.pci_maps_from_result(res)), kind
        assert len(touched.dev_dirty) == len(delta.dev_dirty) and len(touched.grp_gone) == len(delta.grp_gone)
        prev = res


def test_first_call_and_reset_report_everything_added(kv, ctx, ids):
    recs = snapshot(30_000, ids, seed=3)
    ctx.scan_pci_delta_reset()
    res, d0 = ctx.scan_pci_delta(recs)
    assert d0.n_prev == 0 and len(d0.changes) == len(res.survivors)
    assert len(d0.dev_dirty) == len(res.dev_keys) and len(d0.grp_dirty) == len(res.grp_keys)
    assert len(d0.dev_gone) == 0 and len(d0.grp_gone) == 0
    _, d1 = ctx.scan_pci_delta(recs)
    assert d1.n_prev == len(res.survivors) and len(d1.changes) == 0 and len(d1.dev_dirty) == 0
    ctx.scan_pci_delta_reset()
    _, d2 = ctx.scan_pci_delta(recs)
    check_delta(kv, d2, res.survivors[:0], res.survivors, n_prev=0)
    ctx.scan_pci_delta_reset()
    res_e, de = ctx.scan_pci_delta(recs[:0])
    assert len(res_e.survivors) == 0 and de.n_prev == 0 and len(de.changes) == 0
    _, d3 = ctx.scan_pci_delta(recs)          # from an empty previous result
    check_delta(kv, d3, res.survivors[:0], res.survivors)


def test_other_calls_leave_the_previous_result_alone(kv, ctx, ids):
    rng = np.random.default_rng(7)
    a = snapshot(50_000, ids, seed=4)
    ctx.scan_pci_delta_reset()
    ra, _ = ctx.scan_pci_delta(a)
    other = snapshot(300_000, ids, seed=9)
    ctx.scan_pci(other)                                   # pipelined: rewrites the survivors and both orderings
    ctx.scan_mdev(O.gen_mdev(0, 5000), O.gen_type_names(64))
    ctx.health_rescan(other[:20_000])
    ctx.health_rescan(other)
    ctx.pciids_load(util.pciids_text())
    c = step(a, "regroup", rng, ids)
    rc, dc = ctx.scan_pci_delta(c)
    check_delta(kv, dc, ra.survivors, rc.survivors)


def test_non_ascending_input_is_refused_and_keeps_the_previous_result(kv, ctx, ids):
    rng = np.random.default_rng(8)
    a = snapshot(40_000, ids, seed=5)
    ctx.scan_pci_delta_reset()
    ra, _ = ctx.scan_pci_delta(a)
    bad = a.copy()
    alive = np.nonzero(util.pci_alive(bad))[0]
    bad["addr"][alive[5000]] = bad["addr"][alive[4999]]    # two survivors with one address
    with pytest.raises(kv.KvgError) as e:
        ctx.scan_pci_delta(bad)
    assert e.value.rc == -1 and "ascending" in str(e.value)
    swapped = a.copy()
    far = alive[len(alive) // 2]
    swapped["addr"][alive[100]], swapped["addr"][far] = a["addr"][far], a["addr"][alive[100]]
    with pytest.raises(kv.KvgError):
        ctx.scan_pci_delta(swapped)
    c = step(a, "hot_remove", rng, ids)
    rc, dc = ctx.scan_pci_delta(c)
    check_delta(kv, dc, ra.survivors, rc.survivors)


@pytest.mark.parametrize("n", [10_000, 1 * Mi])
def test_launch_budget_and_labels(kv, ctx, ids, n):
    """At most three launches beyond kvg_scan_pci on the same input (two are used), each under a stable label."""
    recs = snapshot(n, ids, seed=6)
    ctx.scan_pci(recs)                       # the radix pass-set hint settles on this input
    c0 = ctx.launch_count
    ctx.scan_pci(recs)
    c1 = ctx.launch_count
    ctx.scan_pci_delta(recs)
    c2 = ctx.launch_count
    assert (c2 - c1) - (c1 - c0) == 2
    ctx.set_kernel_timing(True)
    try:
        ctx.scan_pci_delta(recs)
        labels = [name for name, _ in ctx.kernel_times()]
    finally:
        ctx.set_kernel_timing(False)
    assert labels[-2:] == ["delta_merge", "delta_lists"]
