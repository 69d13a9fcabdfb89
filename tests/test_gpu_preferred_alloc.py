"""kvg_preferred_allocation on the H100: GetPreferredAllocation's NUMA packing for every container request of a call in
one launch, against the reference rule serve.preferred_allocation (through serve.NumaPacker) and the C-ABI contract of
tests/preferred_cases.py, from empty requests to one request of 100,000 entries and 1,000 requests in one call; one
launch per call and none for an empty call or a refusal; every refusal (KVG_EINVAL, res untouched); and isolation: a
call between a device scan and its fetch, between two PCI delta scans or between two keyed group health ticks changes
none of their results, and the scan after a call launches as many kernels as the scan without one."""
import ctypes as C

import numpy as np
import pytest

import preferred_cases as PC
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


def check(ctx, devs, requests):
    """One call through NumaPacker answers as the reference, in one launch; its raw output is the contract's."""
    rec = PC.Recorder(ctx.preferred_allocation)
    before = ctx.launch_count
    got = PC.packed(devs, requests, rec)
    assert ctx.launch_count - before == (1 if requests else 0)
    assert got == PC.reference(devs, requests), (len(requests), [len(r[0]) for r in requests][:8])
    ids, n_must, n_avail, sizes, raw = rec.calls[0]
    want = PC.contract(ids, n_must, n_avail, sizes)
    assert [(n, p, pos.tolist()) for n, p, pos in raw] == [(n, p, pos.tolist()) for n, p, pos in want]
    return got


def test_golden_vectors_edges_and_quirks(ctx):
    for devs, requests in PC.golden_calls() + list(PC.named_calls().values()):
        check(ctx, devs, requests)


def test_seeded_calls(ctx):
    rng = np.random.default_rng(17)
    for _ in range(300):
        check(ctx, *PC.random_call(rng, int(rng.integers(1, 9)), int(rng.integers(1, 60))))


def _large(n, rng, size, n_must=0, n_nodes=4):
    """One request of n available entries over n_nodes nodes and the -1 group, with duplicates and unknown IDs."""
    pool = ["p%d" % k for k in range(max(1, n // 2))]
    nodes = list(range(n_nodes)) + [-1, None, -2]
    devs = [(d, nodes[k % len(nodes)]) for k, d in enumerate(pool)]
    known = pool + ["ghost"]
    available = [known[int(k)] for k in rng.integers(0, len(known), n)]
    must = [known[int(k)] for k in rng.integers(0, len(known), n_must)]
    return devs, [(available, must, size)]


@pytest.mark.parametrize("n", [0, 1, 33, THREADS - 1, THREADS, THREADS + 1, 5000, 100_000])
def test_every_size_regime(ctx, n):
    rng = np.random.default_rng(n)
    for size in sorted({0, 1, 2, n // 9, n // 3, n - 1, n + 3, THREADS, THREADS + 1}):
        for n_must in (0, 3):
            check(ctx, *_large(n, rng, size, n_must))


def test_many_nodes(ctx):
    """As many distinct nodes as entries: the node slots are sized from the entries, with no cap."""
    rng = np.random.default_rng(5)
    n = 20_000
    devs = [("x%d" % k, k) for k in range(n)]
    available = ["x%d" % k for k in rng.permutation(n)]
    for size in (1, 2, 7):
        check(ctx, devs, [(available, ["x3"], size)])
    check(ctx, devs, [(available + available[:5], [], 2)])          # the duplicated IDs' nodes qualify, distinct fill short


def test_a_thousand_requests_in_one_call(ctx):
    rng = np.random.default_rng(1000)
    devs, requests = PC.random_call(rng, 1000, 16)
    check(ctx, devs, requests)
    ok = [(a, m, max(s, len(set(m)))) for a, m, s in requests]
    assert check(ctx, devs, ok)[0] == "ok"
    ok[613] = (["d0"], ["d0", "d1"], 1)
    assert check(ctx, devs, ok) == ("error", "number of MustIncludeDeviceIDs (2) exceeds allocation size (1)")


# ---- the C-ABI's refusals -------------------------------------------------------------------------
def _raw(kv, requests):
    """(reqs, ids, res, pos) arrays for the raw call: each request = (n_must, n_avail, size), handles = positions."""
    reqs = np.zeros(len(requests), dtype=kv._lib.PREF_REQ)
    for r, (m, a, s) in enumerate(requests):
        reqs[r] = (m, a, s, 0)
    n_ids = int(sum(m + a for m, a, _ in requests))
    ids = np.zeros(n_ids, dtype=kv._lib.PREF_ID)
    at = 0
    for m, a, _ in requests:
        ids["handle"][at:at + m + a] = np.arange(m + a)
        ids["node"][at:at + m + a] = 0
        at += m + a
    res = np.full(len(requests), 0x77, dtype=kv._lib.PREF_RES)
    pos = np.full(max(n_ids, 1), 0xeeeeeeee, dtype=np.uint32)
    return reqs, ids, res, pos


def test_empty_call_launches_nothing(kv, ctx):
    lib = kv.load()
    before = ctx.launch_count
    assert lib.kvg_preferred_allocation(ctx.handle, None, 0, None, 0, None, None) == 0
    assert ctx.preferred_allocation(np.zeros(0, dtype=kv._lib.PREF_ID), [], [], []) == []
    assert ctx.launch_count == before
    # requests with empty lists still take the size test, in one launch
    out = ctx.preferred_allocation(np.zeros(0, dtype=kv._lib.PREF_ID), [0, 0, 0], [0, 0, 0], [0, -1, 5])
    assert [(n, p, list(x)) for n, p, x in out] == [(0, 0, []), (-1, 0, []), (0, 0, [])]
    assert ctx.launch_count == before + 1


def test_refusals_launch_nothing_and_leave_res_alone(kv, ctx):
    lib = kv.load()
    reqs, ids, res, pos = _raw(kv, [(2, 3, 2), (0, 4, 1)])
    h = ctx.handle
    R, I, S, Q = reqs.ctypes.data, ids.ctypes.data, res.ctypes.data, pos.ctypes.data
    before = ctx.launch_count
    assert lib.kvg_preferred_allocation(h, R, 2, I, 9, S, Q) == 0
    assert res.tolist() == [(2, 2), (1, 0)] and ctx.launch_count == before + 1

    def bad_ids(**change):
        x = ids.copy()
        for k, (field, v) in change.items():
            x[field][int(k[1:])] = v
        return x
    keep = []
    variants = [
        (None, R, 2, I, 9, S, Q),                        # ctx NULL
        (h, None, 2, I, 9, S, Q),                        # reqs NULL, n_reqs > 0
        (h, R, 2, I, 9, None, Q),                        # res NULL, n_reqs > 0
        (h, R, 2, None, 9, S, Q),                        # ids NULL, n_ids > 0
        (h, R, 2, I, 9, S, None),                        # out_pos NULL, n_ids > 0
        (h, R, 2, I, 1 << 32, S, Q),                     # n_ids does not fit in uint32
        (h, R, 2, I, 8, S, Q),                           # fewer entries than the requests hold
        (h, R, 2, I, 10, S, Q),                          # more entries than the requests hold
        (h, R, 1, I, 9, S, Q),                           # the same, from the request side
        (h, R, 0, I, 9, S, Q),
    ]
    for change in ({"e0": ("handle", 5)}, {"e8": ("handle", 4)}, {"e4": ("node", 5)}, {"e6": ("node", 4)},
                   {"e1": ("node", 0xfffffffe)}):
        x = bad_ids(**change)
        keep.append(x)
        variants.append((h, R, 2, x.ctypes.data, 9, S, Q))  # a handle or node out of its request's range
    for i, args in enumerate(variants):
        res[:] = (0x77, 0x77)
        assert lib.kvg_preferred_allocation(*args) == KVG_EINVAL, i
        assert res.tolist() == [(0x77, 0x77)] * 2, i
    assert ctx.launch_count == before + 1
    # the largest handle and node in range, and PREF_NODE_NONE, are accepted
    x = bad_ids(e4=("handle", 4), e3=("node", 4), e8=("node", kv._lib.PREF_NODE_NONE))
    assert lib.kvg_preferred_allocation(h, R, 2, x.ctypes.data, 9, S, Q) == 0
    assert ctx.launch_count == before + 2


def test_length_mismatch_is_refused_in_python(kv, ctx):
    before = ctx.launch_count
    with pytest.raises(ValueError):
        ctx.preferred_allocation(np.zeros(3, dtype=kv._lib.PREF_ID), [1], [2, 0], [1])
    assert ctx.launch_count == before


# ---- isolation ----------------------------------------------------------------------------------
def _same(a, b):
    for f in a.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def _pack_in_between(ctx):
    rng = np.random.default_rng(11)
    check(ctx, *_large(5000, rng, 1200, 3))
    check(ctx, *PC.random_call(rng, 16, 16))


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
        _pack_in_between(ctx)
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
    _pack_in_between(ctx)
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
                _pack_in_between(ctx)
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
    _pack_in_between(ctx)
    after, got = scan_launches()
    assert after == plain
    _same(got, want)
