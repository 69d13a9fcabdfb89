"""kvg_pci_group_check on the H100: the passthrough plugin's Allocate-time re-check, one launch per call, against its
rule restated in numpy (tests/group_check_cases.py) for every combination of the fields the rule reads and at 1 to
100,000 records; every refusal (KVG_EINVAL, nothing launched, first_bad untouched); and isolation: a check between a
device scan and its fetch, between two PCI delta scans or between two keyed group health ticks changes none of their
results, and the scan after a check launches as many kernels as the scan without one."""
import ctypes as C

import numpy as np
import pytest

import group_check_cases as GC
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

KVG_EINVAL = -1
SIZES = [1, 31, 32, 33, 1023, 1024, 1025, 5000, 100_000]


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


def checked(ctx, recs, want):
    before = ctx.launch_count
    got = ctx.pci_group_check(recs, want)
    assert ctx.launch_count - before == (1 if len(recs) else 0)
    fb = GC.first_bad(recs, want)
    assert got == (None if fb == len(recs) else fb), (len(recs), fb, got)
    return got


def test_every_combination_of_the_fields_the_rule_reads(ctx):
    rng = np.random.default_rng(1)
    combos = GC.combinations()
    for combo in combos:
        for _ in range(4):
            recs, want = GC.noise(1, rng)
            GC.apply(recs, want, 0, combo)
            ok = not combo[0] and not combo[1] and combo[2] == 0x10de and combo[3]
            assert checked(ctx, recs, want) == (None if ok else 0), combo
    recs, want = GC.noise(len(combos), rng)
    for i, combo in enumerate(combos):
        GC.apply(recs, want, i, combo)
    for _ in range(16):
        p = rng.permutation(len(combos))
        checked(ctx, recs[p], want[p])


def test_ignored_fields_never_fail_a_record(ctx):
    rng = np.random.default_rng(2)
    recs, want = GC.noise(100_000, rng)
    recs["flags"][::3] |= 2 | 8                             # DRIVER_ERR | DEVICE_ERR
    recs["driver"][1::3] = 0
    recs["device"][2::3] = 0
    assert checked(ctx, recs, want) is None


@pytest.mark.parametrize("n", SIZES)
def test_smallest_failing_index_wins(ctx, n):
    rng = np.random.default_rng(n)
    for at in GC.failure_sets(n, rng):
        recs, want = GC.with_failures(n, at, rng)
        assert checked(ctx, recs, want) == (min(at) if at else None), at


def test_empty_call_launches_nothing(ctx):
    recs, want = GC.noise(0, np.random.default_rng(0))
    assert checked(ctx, recs, want) is None


def test_refusals_launch_nothing_and_leave_first_bad_alone(kv, ctx):
    lib = kv.load()
    recs, want = GC.with_failures(4, [2], np.random.default_rng(3))
    first = C.c_size_t(0xdead)
    h, r, w = ctx.handle, recs.ctypes.data, want.ctypes.data
    before = ctx.launch_count
    assert lib.kvg_pci_group_check(h, r, w, 4, C.byref(first)) == 0
    assert first.value == 2 and ctx.launch_count == before + 1
    before = ctx.launch_count
    cases = [
        (None, r, w, 4, C.byref(first)),                 # ctx NULL
        (h, r, w, 4, None),                              # first_bad NULL
        (h, None, w, 4, C.byref(first)),                 # recs NULL, n > 0
        (h, r, None, 4, C.byref(first)),                 # want_group NULL, n > 0
        (h, r, w, 1 << 32, C.byref(first)),              # n does not fit in uint32
        (h, r, w, (1 << 64) - 1, C.byref(first)),
    ]
    for i, args in enumerate(cases):
        first.value = 0xdead
        assert lib.kvg_pci_group_check(*args) == KVG_EINVAL, i
        assert first.value == 0xdead, i
    assert ctx.launch_count == before
    # n = 0: *first_bad = 0, nothing launched, with or without arrays
    for args in ((h, None, None, 0), (h, r, w, 0)):
        first.value = 0xdead
        assert lib.kvg_pci_group_check(*args, C.byref(first)) == 0
        assert first.value == 0
    assert ctx.launch_count == before
    assert lib.kvg_pci_group_check(h, r, w, 2, C.byref(first)) == 0
    assert first.value == 2 and ctx.launch_count == before + 1      # all pass: n


def test_length_mismatch_is_refused_in_python(ctx):
    recs, want = GC.noise(3, np.random.default_rng(4))
    before = ctx.launch_count
    with pytest.raises(ValueError):
        ctx.pci_group_check(recs, want[:2])
    assert ctx.launch_count == before


# ---- isolation ----------------------------------------------------------------------------------
def _same(a, b):
    for f in a.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def _check_in_between(ctx):
    rng = np.random.default_rng(11)
    recs, want = GC.with_failures(5000, [4321, 4999], rng)
    assert checked(ctx, recs, want) == 4321
    recs, want = GC.noise(16, rng)
    assert checked(ctx, recs, want) is None


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
    groups = [int(g) for g in np.unique(recs["iommu_group"])]      # at most KVG_HEALTH_MAX_GROUPS per tick
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
