"""kvg_pci_allocate_check on the H100: the passthrough plugin's Allocate decisions (the group re-check and the EGM match)
for every container request of a call in one launch, against the C-ABI contract of tests/allocate_check_cases.py, from
empty requests to 1,000 requests in one call, one request of 100,000 members and 4,096 EGM devices; one launch per call
and none for an empty call or a refusal; every refusal (KVG_EINVAL, outputs untouched); and isolation: a call between
a device scan and its fetch, between two PCI delta scans or between two keyed group health ticks changes none of their
results, and the scan after a call launches as many kernels as the scan without one."""
import ctypes as C

import numpy as np
import pytest

import allocate_check_cases as AC
import group_check_cases as GC
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

KVG_EINVAL = -1
THREADS = 1024


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


def check(ctx, c):
    before = ctx.launch_count
    bad, take = ctx.pci_allocate_check(**c)
    assert ctx.launch_count - before == (1 if len(c["n_members"]) else 0)
    want_bad, want_take = AC.contract(**c)
    assert bad.tolist() == want_bad.tolist()
    assert np.array_equal(take, want_take)
    return bad, take


@pytest.mark.parametrize("name", sorted(AC.named_calls()))
def test_named_quirks(ctx, name):
    check(ctx, AC.named_calls()[name])


def test_seeded_calls(ctx):
    rng = np.random.default_rng(23)
    for _ in range(300):
        check(ctx, AC.random_call(rng, int(rng.integers(0, 17)), max_members=int(rng.integers(0, 80))))


def test_a_thousand_requests_in_one_call(ctx):
    rng = np.random.default_rng(1000)
    c = AC.random_call(rng, 1000, max_members=24, n_egm=16)
    bad, take = check(ctx, c)
    assert (bad < np.array(c["n_members"])).any() and (bad == np.array(c["n_members"])).any()
    assert take.any() and not take.all()


@pytest.mark.parametrize("n", [1, 33, THREADS - 1, THREADS, THREADS + 1, 5000, 100_000])
def test_one_large_request(ctx, n):
    rng = np.random.default_rng(n)
    for at in GC.failure_sets(n, rng):
        recs, want = GC.with_failures(n, at, rng)
        c = AC.make_call(recs, want, [n], [0, 1, 5], [3], [[0, 1], [2], []], 3)
        bad, take = check(ctx, c)
        assert int(bad[0]) == (min(at) if at else n)
        assert take.tolist() == [[True, False, True]]


def test_4096_egm_devices(ctx):
    rng = np.random.default_rng(4096)
    n_egm, n_gpus = 4096, 20_000
    lists = [[int(g) for g in rng.choice(n_gpus, int(rng.integers(0, 9)), replace=False)] for _ in range(n_egm)]
    n_reqs = 40
    ids, n_ids = [], []
    for r in range(n_reqs):
        mine = [g for e in rng.integers(0, n_egm, 300) for g in lists[int(e)]]   # about 300 devices held whole
        mine = mine[:-1] if r % 2 else mine                                        # ... or all but one GPU of one
        mine += [int(g) for g in rng.integers(0, n_gpus + 10, 200)]
        ids += mine
        n_ids.append(len(mine))
    n_members = [int(rng.integers(0, 50)) for _ in range(n_reqs)]
    recs, want = AC.records(n_members, rng)
    bad, take = check(ctx, AC.make_call(recs, want, n_members, ids, n_ids, lists, n_gpus))
    assert take.shape == (n_reqs, n_egm) and 0 < take.sum() < take.size


def test_group_check_still_launches_once(ctx):
    """kvg_pci_group_check is the one-request case of the same launch: one launch, the same answer."""
    rng = np.random.default_rng(8)
    for n in (1, 5000):
        for at in GC.failure_sets(n, rng):
            recs, want = GC.with_failures(n, at, rng)
            before = ctx.launch_count
            got = ctx.pci_group_check(recs, want)
            assert ctx.launch_count == before + 1
            bad, _ = check(ctx, AC.make_call(recs, want, [n], [], [0], []))
            assert (n if got is None else got) == int(bad[0]) == GC.first_bad(recs, want)


# ---- the C-ABI's refusals -------------------------------------------------------------------------
def _args(kv, ctx, c, first_bad, take):
    """The raw call's arguments for the call dict c, and the arrays they point into."""
    reqs = np.zeros(len(c["n_members"]), dtype=kv._lib.ALLOC_REQ)
    reqs["n_members"], reqs["n_ids"] = c["n_members"], c["n_ids"]
    recs = np.ascontiguousarray(c["recs"])
    want, ids = np.ascontiguousarray(c["want"], np.uint32), np.ascontiguousarray(c["ids"], np.uint32)
    off, gpu = np.ascontiguousarray(c["egm_off"], np.uint32), np.ascontiguousarray(c["egm_gpu"], np.uint32)
    keep = (reqs, recs, want, ids, off, gpu)
    args = [ctx.handle, reqs.ctypes.data, len(reqs), recs.ctypes.data, want.ctypes.data, len(recs), ids.ctypes.data,
            len(ids), off.ctypes.data, gpu.ctypes.data, max(len(off) - 1, 0), c["n_egm_gpus"], first_bad.ctypes.data,
            take.ctypes.data]
    return args, keep


def test_empty_call_launches_nothing(kv, ctx):
    lib = kv.load()
    before = ctx.launch_count
    assert lib.kvg_pci_allocate_check(ctx.handle, None, 0, None, None, 0, None, 0, None, None, 0, 0, None, None) == 0
    c = AC.make_call(np.zeros(0, dtype=kv._lib.PCI_REC), [], [], [], [], [[0], []], 1)
    assert [x.tolist() for x in ctx.pci_allocate_check(**c)] == [[], []]
    assert ctx.launch_count == before
    # requests with empty lists still launch, once
    bad, take = check(ctx, AC.make_call(np.zeros(0, dtype=kv._lib.PCI_REC), [], [0, 0], [], [0, 0], [[0], []], 1))
    assert bad.tolist() == [0, 0] and take.tolist() == [[False, True], [False, True]]
    assert ctx.launch_count == before + 1


def test_refusals_launch_nothing_and_leave_the_outputs_alone(kv, ctx):
    lib = kv.load()
    calls = AC.refused_calls()
    first_bad = np.full(8, 0x77, dtype=np.uint32)
    take = np.full(64, 0x77, dtype=np.uint8)
    base, keep = _args(kv, ctx, calls["accepted"], first_bad, take)
    before = ctx.launch_count
    assert lib.kvg_pci_allocate_check(*base) == 0 and ctx.launch_count == before + 1
    variants = []
    for name, c in calls.items():
        if name != "accepted":
            args, k = _args(kv, ctx, c, first_bad, take)
            keep += k
            variants.append((name, args))
    nulls = {0: "ctx", 1: "reqs", 3: "recs", 4: "want_group", 6: "ids", 8: "egm_off", 9: "egm_gpu", 12: "first_bad",
             13: "egm_take"}
    for i, what in nulls.items():
        args = list(base)
        args[i] = None
        variants.append(("%s NULL" % what, args))
    for i, v in ((5, 1 << 32), (7, 1 << 32)):                         # n_recs / n_ids do not fit in uint32
        args = list(base)
        args[i] = v
        variants.append(("count %d above UINT32_MAX" % i, args))
    for name, args in variants:
        first_bad[:], take[:] = 0x77, 0x77
        assert lib.kvg_pci_allocate_check(*args) == KVG_EINVAL, name
        assert (first_bad == 0x77).all() and (take == 0x77).all(), name
    assert ctx.launch_count == before + 1
    # the cap itself, the largest handle under it, and NULL EGM arrays with no EGM device are accepted
    c = AC.named_calls()["n_egm_gpus at the cap"]
    check(ctx, c)
    args, k = _args(kv, ctx, AC.make_call(c["recs"], c["want"], c["n_members"], c["ids"], c["n_ids"], []),
                    first_bad, take)
    args[8] = args[9] = args[13] = None
    assert lib.kvg_pci_allocate_check(*args) == 0 and ctx.launch_count == before + 3


def test_length_mismatch_is_refused_in_python(kv, ctx):
    before = ctx.launch_count
    with pytest.raises(ValueError):
        ctx.pci_allocate_check(np.zeros(3, dtype=kv._lib.PCI_REC), [0, 0], [3], [], [0], [], [], 0)
    with pytest.raises(kv.KvgError):
        ctx.pci_allocate_check(np.zeros(3, dtype=kv._lib.PCI_REC), [0, 0, 0], [2], [], [0], [], [], 0)
    assert ctx.launch_count == before


# ---- isolation ----------------------------------------------------------------------------------
def _same(a, b):
    for f in a.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def _check_in_between(ctx):
    rng = np.random.default_rng(11)
    check(ctx, AC.random_call(rng, 16, max_members=3000, n_egm=64))
    recs, want = GC.with_failures(5000, [4000], rng)
    check(ctx, AC.make_call(recs, want, [5000], [0], [1], [[0]]))


@pytest.fixture(scope="module")
def ids():
    return O.nv_ids(util.pciids_text())


@pytest.mark.parametrize("n", [16, 50_000])
def test_device_scan_and_fetch_are_untouched(ctx, ids, n):
    import torch
    recs = O.gen_pci(3, n, ids, 9)
    buf = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    try:
        ctx.dev_scan_pci(buf.data_ptr(), n)
        want = ctx.dev_scan_pci_fetch()
        ctx.dev_scan_pci(buf.data_ptr(), n)
        _check_in_between(ctx)
        _same(ctx.dev_scan_pci_fetch(), want)
    finally:
        torch.cuda.synchronize()
        del buf


def test_pci_delta_is_untouched(ctx, ids):
    a, b = O.gen_pci(4, 20_000, ids, 9), O.gen_pci(4, 20_000, ids, 9)
    b["iommu_group"][::97] += 1
    b["flags"][::301] ^= 1
    b = np.delete(b, np.arange(50, 20_000, 503))
    ctx.scan_pci_delta_reset()
    ctx.scan_pci_delta(a)
    want_res, want = ctx.scan_pci_delta(b)
    ctx.scan_pci_delta_reset()
    ctx.scan_pci_delta(a)
    _check_in_between(ctx)
    got_res, got = ctx.scan_pci_delta(b)
    _same(got_res, want_res)
    _same(got, want)
    assert len(want.changes) > 0


@pytest.mark.parametrize("n", [1000, 40_000])
def test_keyed_group_health_is_untouched(ctx, ids, n):
    recs = O.gen_pci(6, n, ids, 9)
    recs = recs[np.unique(recs["addr"], return_index=True)[1]]        # keys ascend strictly
    groups = [int(g) for g in np.unique(recs["iommu_group"])]
    ticks = [(recs, groups[:3000:2]), (recs[1:], groups[1:4000:3]), (recs, groups[:4096])]

    def run(between):
        ctx.health_rescan_groups_keyed(recs[:0])                   # an empty list resets
        out = []
        for r, x in ticks:
            if between:
                _check_in_between(ctx)
            d = ctx.health_rescan_groups_keyed(r, x)
            out.append((d.n_records, d.n_alive, d.changed.tobytes()))
        return out
    want = run(False)
    assert run(True) == want
    assert any(len(c) for _, _, c in want)


@pytest.mark.parametrize("n", [16, 50_000])
def test_next_scan_launches_as_many_kernels(ctx, ids, n):
    recs = O.gen_pci(8, n, ids, 9)
    ctx.scan_pci(recs)

    def scan_launches():
        before = ctx.launch_count
        res = ctx.scan_pci(recs)
        return ctx.launch_count - before, res
    plain, want = scan_launches()
    _check_in_between(ctx)
    after, got = scan_launches()
    assert after == plain
    _same(got, want)
