"""kvg_pci_allocate_response on the H100: the passthrough plugin's AllocateResponse from the raw reads, against the
Go-exact restatement of tests/allocate_response_cases.py: every named edge with iommufd on and off, the refusals,
300 seeded calls, 1,000 requests of 24 members and one request of 100,000 members with 4,096 EGM entries; the launch
counts of include/kvgpu.h; a refused call hands out nothing; isolation from a device scan and its fetch, the PCI
delta and keyed group health; and with iommufd off, the decisions equal kvg_pci_allocate_raw's."""
import numpy as np
import pytest

import allocate_raw_cases as AR
import allocate_response_cases as RC
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

KVG_EINVAL, KVG_ERANGE = -1, -6


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


def launches(requests, egm):
    n_mem = sum(len(v) for _, visits, _ in requests for v in visits)
    return ((n_mem > 0) + (n_mem > 0 or len(egm) > 1) + (len(egm) > 0) + 2 * (len(requests) > 0)
            if requests or egm else 0)


def check(kv, ctx, requests, egm, iommufd):
    before = ctx.launch_count
    packed = kv.pack_alloc_response(requests, egm, iommufd)
    try:
        want = RC.allocate_response(requests, egm, iommufd)
    except AR.RawError as e:
        with pytest.raises(kv.KvgError) as got:
            ctx.pci_allocate_response(*packed)
        assert got.value.rc == (KVG_ERANGE if e.kind == "range" else KVG_EINVAL)
        assert ctx.launch_count - before == launches(requests, egm)
        return None
    got = ctx.pci_allocate_response(*packed)
    assert ctx.launch_count - before == launches(requests, egm)
    assert got == want
    return got


@pytest.mark.parametrize("name,requests,egm,iommufd", RC.edge_calls(),
                         ids=["%s-%s" % (c[0], "iommufd" if c[3] else "noiommufd") for c in RC.edge_calls()])
def test_edges(kv, ctx, name, requests, egm, iommufd):
    check(kv, ctx, requests, egm, iommufd)


@pytest.mark.parametrize("name,requests,egm,iommufd", RC.edge_refusals(), ids=[c[0] for c in RC.edge_refusals()])
def test_refusals_hand_out_nothing(kv, ctx, name, requests, egm, iommufd):
    assert check(kv, ctx, requests, egm, iommufd) is None


def test_refused_before_launch(kv, ctx):
    raw, resp = kv.pack_alloc_response([RC.one([[RC.mem(RC.A[0])]])], [], True)
    resp.id_members = np.array([2], dtype=np.uint32)   # the visit counts do not add up
    before = ctx.launch_count
    with pytest.raises(kv.KvgError) as e:
        ctx.pci_allocate_response(raw, resp)
    assert e.value.rc == KVG_EINVAL and ctx.launch_count == before
    assert ctx.pci_allocate_response(*kv.pack_alloc_response([], [], True)) == []
    assert ctx.launch_count == before


def test_seeded_calls(kv, ctx):
    rng = np.random.default_rng(20261019)
    for _ in range(300):
        check(kv, ctx, *RC.random_call(rng))


def _big(n_reqs, n_mem, rng, n_egm=0):
    """n_reqs requests of n_mem members each, 1-8 listing entries per member, groups of 4 members"""
    reqs = []
    for r in range(n_reqs):
        visits = []
        for v in range(n_mem // 4):
            g = b"%d" % (r * 100_000 + v)
            visit = []
            for k in range(4):
                listing = [(b"vfio%d" % x, bool(x % 3)) for x in rng.integers(0, 50, size=int(rng.integers(1, 9)))]
                listing.append((b"vfio%d" % (v * 4 + k), True))
                visit.append((b"0000:%02x:%02x.%d" % (r % 256, v % 256, k), b"../" + g, b"0x10de\n", g, listing))
            visits.append(visit)
        reqs.append(([v[0][0] for v in visits], visits, False))
    egm = [(b"egm%05d" % e, b"0000:00:%02x.0" % (e % 256), True) for e in range(n_egm)]
    return reqs, egm


def test_a_thousand_requests_of_24_members(kv, ctx):
    reqs, egm = _big(1000, 24, np.random.default_rng(3), 16)
    got = check(kv, ctx, reqs, egm, True)
    assert all(r[0] == RC.OK for r in got)


def test_one_request_of_100000_members_and_4096_egm_entries(kv, ctx):
    reqs, egm = _big(1, 100_000, np.random.default_rng(4), 4096)
    got = check(kv, ctx, reqs, egm, True)
    assert got[0][0] == RC.OK and got[0][2][-1] == b"/dev/egm04095"


def test_decisions_equal_allocate_raw_without_iommufd(kv, ctx):
    rng = np.random.default_rng(7)
    for _ in range(100):
        requests, egm, _ = RC.random_call(rng)
        requests = [(ids, [[(a, l, v, visit[0][3], x) for a, l, v, _, x in visit] for visit in visits], lk)
                    for ids, visits, lk in requests]
        raw, resp = kv.pack_alloc_response(requests, egm, False)
        try:
            first_bad, panic, _, take = ctx.pci_allocate_raw(raw)
        except kv.KvgError:
            continue
        got = ctx.pci_allocate_response(raw, resp)
        for r, (err, at, paths, _) in enumerate(got):
            n = int(raw.n_members[r])
            if first_bad[r] < n:   # the member error is the first, unless an earlier ID was not found
                assert err in (RC.UNKNOWN_ID, RC.PANIC if panic[r] else RC.UNKNOWN_MEMBER)
                if err != RC.UNKNOWN_ID:
                    assert at == first_bad[r]
            else:
                assert err in (RC.OK, RC.UNKNOWN_ID)
            if err == RC.OK:
                taken = [b"/dev/" + egm[e][0] for e in range(len(egm)) if take[r, e]]
                assert paths[len(paths) - len(taken):] == taken


# ---- isolation ----------------------------------------------------------------------------------
def _same(a, b):
    for f in a.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def _in_between(kv, ctx):
    rng = np.random.default_rng(11)
    for _ in range(3):
        check(kv, ctx, *RC.random_call(rng))
    check(kv, ctx, *_big(1, 4000, rng, 8), True)


@pytest.fixture(scope="module")
def ids():
    return O.nv_ids(util.pciids_text())


def test_device_scan_and_fetch_are_untouched(kv, ctx, ids):
    import torch
    n = 50_000
    recs = O.gen_pci(3, n, ids, 9)
    buf = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    try:
        ctx.dev_scan_pci(buf.data_ptr(), n)
        want = ctx.dev_scan_pci_fetch()
        ctx.dev_scan_pci(buf.data_ptr(), n)
        _in_between(kv, ctx)
        _same(ctx.dev_scan_pci_fetch(), want)
    finally:
        torch.cuda.synchronize()
        del buf


def test_pci_delta_is_untouched(kv, ctx, ids):
    a, b = O.gen_pci(4, 20_000, ids, 9), O.gen_pci(4, 20_000, ids, 9)
    b["iommu_group"][::97] += 1
    b = np.delete(b, np.arange(50, 20_000, 503))
    ctx.scan_pci_delta_reset()
    ctx.scan_pci_delta(a)
    want_res, want = ctx.scan_pci_delta(b)
    ctx.scan_pci_delta_reset()
    ctx.scan_pci_delta(a)
    _in_between(kv, ctx)
    got_res, got = ctx.scan_pci_delta(b)
    _same(got_res, want_res)
    _same(got, want)


def test_keyed_group_health_is_untouched(kv, ctx, ids):
    recs = O.gen_pci(6, 4000, ids, 9)
    recs = recs[np.unique(recs["addr"], return_index=True)[1]]
    groups = [int(g) for g in np.unique(recs["iommu_group"])]
    ticks = [(recs, groups[:3000:2]), (recs[1:], groups[1:4000:3]), (recs, groups[:4096])]

    def run(between):
        ctx.health_rescan_groups_keyed(recs[:0])
        out = []
        for r, x in ticks:
            if between:
                _in_between(kv, ctx)
            d = ctx.health_rescan_groups_keyed(r, x)
            out.append((d.n_records, d.n_alive, d.changed.tobytes()))
        return out
    assert run(True) == run(False)
