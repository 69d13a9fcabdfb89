"""kvg_pci_allocate_raw on the H100: the passthrough plugin's Allocate decisions from the raw reads, against the
Go-exact restatement of tests/allocate_raw_cases.py: every named edge and refusal, seeded calls, 1,000 requests in one
call and one request of 100,000 members with 4,096 EGM entries; the launch counts of include/kvgpu.h, none for an
empty call or a call refused before launch; every refusal leaves the outputs alone; isolation: a call between a device
scan and its fetch, between two PCI delta scans or between two keyed group health ticks changes none of their
results; and on ASCII inputs the decisions equal kvg_pci_allocate_check's fed by AllocateCheck's host interning."""
import ctypes as C

import numpy as np
import pytest

import allocate_raw_cases as AR
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
    n_mem = sum(len(m) for m, _ in requests)
    return (n_mem > 0) + (len(egm) > 0) + (len(requests) > 0)


def check(kv, ctx, requests, egm):
    before = ctx.launch_count
    try:
        want = AR.allocate_raw(requests, egm)
    except AR.RawError as e:
        with pytest.raises(kv.KvgError) as got:
            ctx.pci_allocate_raw(kv.pack_alloc_raw(requests, egm))
        assert got.value.rc == (KVG_EINVAL if e.kind == "miss" else KVG_ERANGE)
        assert ctx.launch_count - before == launches(requests, egm)
        return got.value
    got = ctx.pci_allocate_raw(kv.pack_alloc_raw(requests, egm))
    assert ctx.launch_count - before == launches(requests, egm)
    for g, w in zip(got, want):
        assert g.tolist() == w.tolist()
    return got


@pytest.mark.parametrize("name,requests", AR.edge_requests(), ids=[n for n, _ in AR.edge_requests()])
def test_member_edges(kv, ctx, name, requests):
    assert isinstance(check(kv, ctx, requests, []), tuple)


@pytest.mark.parametrize("name,requests,egm", AR.edge_refusals(), ids=[n for n, _, _ in AR.edge_refusals()])
def test_reached_reads_not_made_are_refused(kv, ctx, name, requests, egm):
    e = check(kv, ctx, requests, egm)
    assert isinstance(e, kv.KvgError) and "was not made" in str(e)


def test_egm_edges(kv, ctx):
    got = check(kv, ctx, [([AR.ok_member()], ids) for ids in AR.edge_id_sets()], AR.edge_egm())
    assert got[2].any() and got[3].any()


def test_seeded_calls(kv, ctx):
    for seed in range(300):
        check(kv, ctx, *AR.random_call(np.random.default_rng(seed)))


def test_a_thousand_requests_in_one_call(kv, ctx):
    rng = np.random.default_rng(1000)
    reqs, egm = AR.random_call(rng, 0)
    vend, links = list(AR.VENDORS.values()), list(AR.LINKS.values())
    for r in range(1000):
        members = [AR.ok_member() if rng.random() < 0.995 else (links[rng.integers(len(links))],
                                                                 vend[rng.integers(len(vend))], AR.G)
                   for _ in range(24)]
        reqs.append((members, [AR.BDF[k] for k in rng.integers(0, 4, size=3)] + [AR.IDS[r % len(AR.IDS)]]))
    egm = [(b"egm%d" % e, g, True) for e, g in enumerate(AR.GPU_DEVICES.values())]
    check(kv, ctx, reqs, egm)


def test_one_large_request_and_4096_egm_entries(kv, ctx):
    bdfs = [b"0000:%02x:%02x.%x" % (k >> 8, (k >> 3) & 31, k & 7) for k in range(100_000 // 8)]
    members = [AR.ok_member()] * 100_000
    members[77_777] = (AR.LINK_OK, b"", AR.G)                         # the panic, behind 77,777 passing members
    egm = [(b"egm%04d" % e, b" ".join(bdfs[2 * e:2 * e + 2]).upper() + b"\n", e % 7 != 3) for e in range(4096)]
    ids = bdfs[::2] + bdfs[1:5000:2]
    got = check(kv, ctx, [(members, ids)], egm)
    assert int(got[0][0]) == 77_777 and got[1][0]
    assert got[3][0].sum() == sum(1 for e in range(2500) if e % 7 != 3)


def test_empty_call_launches_nothing(kv, ctx):
    before = ctx.launch_count
    got = ctx.pci_allocate_raw(kv.pack_alloc_raw([], []))
    assert ctx.launch_count == before and all(len(x) == 0 for x in got)
    assert isinstance(check(kv, ctx, [([], [])], []), tuple)                  # one request: the check kernel only
    assert isinstance(check(kv, ctx, [], [(b"egm0", b"a", True)]), tuple)    # EGM entries only: the key kernel only


def test_refusals_launch_nothing_and_leave_the_outputs_alone(kv, ctx):
    lib = ctx._lib
    raw = kv.pack_alloc_raw([([AR.ok_member(), (AR.LINK_OK, b"0x10de", AR.G)], [AR.BDF[0]])],
                            [(b"egm0", AR.BDF[0], True)])
    keep = []

    def call(mutate=None, reqs_counts=(2, 1)):
        arr = lambda a, t: np.array(a, dtype=t)   # noqa: E731
        f = {"member_off": arr(raw.member_off, np.uint32), "member_state": arr(raw.member_state, np.uint16),
             "id_off": arr(raw.id_off, np.uint32), "egm_off": arr(raw.egm_off, np.uint32),
             "egm_state": arr(raw.egm_state, np.uint16)}
        blobs = [np.frombuffer(b + b"\0", dtype=np.uint8) for b in (raw.member_bytes, raw.id_bytes, raw.egm_bytes)]
        arg = kv._lib.AllocRawC(2, f["member_off"].ctypes.data, blobs[0].ctypes.data, f["member_state"].ctypes.data,
                                1, f["id_off"].ctypes.data, blobs[1].ctypes.data, 1, f["egm_off"].ctypes.data,
                                blobs[2].ctypes.data, f["egm_state"].ctypes.data)
        reqs = np.array([reqs_counts], dtype=np.uint32)
        outs = [np.full(1, 0xabcdabcd, np.uint32), np.full(1, 0xab, np.uint8), np.full(1, 0xab, np.uint8),
                np.full(1, 0xab, np.uint8)]
        if mutate:
            mutate(arg, f)
        keep.append((f, blobs, arg))
        before = ctx.launch_count
        rc = lib.kvg_pci_allocate_raw(ctx._h, reqs.ctypes.data, 1, C.byref(arg), *[o.ctypes.data for o in outs])
        return rc, ctx.launch_count - before, outs

    rc, n, outs = call()
    assert rc == 0 and n == 3 and outs[0][0] == 2
    for mutate, counts in [(lambda a, f: setattr(a, "member_off", None), (2, 1)),
                           (lambda a, f: setattr(a, "egm_state", None), (2, 1)),
                           (lambda a, f: setattr(a, "id_bytes", None), (2, 1)),
                           (None, (3, 1)), (None, (2, 0)),
                           (lambda a, f: f["member_off"].__setitem__(0, 1), (2, 1)),
                           (lambda a, f: f["id_off"].__setitem__(0, 5), (2, 1)),
                           (lambda a, f: f["egm_off"].__setitem__(2, 0), (2, 1)),
                           (lambda a, f: setattr(a, "n_members", 1 << 32), (2, 1))]:
        rc, n, outs = call(mutate, counts)
        assert rc == KVG_EINVAL and n == 0
        assert [int(o[0]) for o in outs] == [0xabcdabcd, 0xab, 0xab, 0xab]
    # found on the device: the outputs stay as they were too
    rc, n, outs = call(lambda a, f: f["member_state"].__setitem__(1, 1 << 0))
    assert rc == KVG_EINVAL and n == 3 and [int(o[0]) for o in outs] == [0xabcdabcd, 0xab, 0xab, 0xab]


def test_key_cap_both_sides(kv, ctx):
    keys = [b"%05x" % k for k in range(65536)]
    egm = [(b"egm%04d" % e, b" ".join(keys[e * 16:(e + 1) * 16]), True) for e in range(4096)]
    reqs = [([AR.ok_member()], keys[:16])]
    got = check(kv, ctx, reqs, egm[:4095] + [(b"egm4095", b" ".join(keys[65520:65535] + [keys[3]]), True)])
    assert got[3][0, 0] and got[2].all()
    e = check(kv, ctx, reqs, egm)
    assert isinstance(e, kv.KvgError) and e.rc == KVG_ERANGE and "egm4095" in str(e)


# ---- on ASCII inputs, the decisions of kvg_pci_allocate_check fed by AllocateCheck's host interning ------------------
def test_ascii_calls_equal_the_interned_check(kv, ctx):
    from kvgpu import serve
    rng = np.random.default_rng(5)
    for _ in range(100):
        reqs, egm = AR.random_call(rng)
        # ASCII without \x1c-\x1f, which Python's str.split() and str.strip() take for spaces and Go does not
        plain = lambda b: b is None or (b.isascii() and not any(0x1C <= c <= 0x1F for c in b))   # noqa: E731
        reqs = [([m for m in members if all(plain(x) for x in m)], [i for i in ids if plain(i)])
                for members, ids in reqs]
        egm = [(n, g, s) for n, g, s in egm if plain(g)]
        fb, panic, kept, take = ctx.pci_allocate_raw(kv.pack_alloc_raw(reqs, egm))
        # AllocateCheck's form: group strings interned per call, EGM strings by egm_key, kept entries only
        devs = [serve.EGMDeviceInfo("/dev/" + n.decode(), g.decode().split())
                for (n, g, s), k in zip(egm, kept) if k]
        intern, recs, want, ids, n_members, n_ids = {}, [], [], [], [], []
        eh, eoff, egpu = {}, [0] if devs else [], []
        for d in devs:
            egpu.extend(eh.setdefault(serve.egm_key(g), len(eh)) for g in d.gpu_bdfs)
            eoff.append(len(egpu))
        for members, dids in reqs:
            for link, vendor, group in members:
                w = intern.setdefault(group, len(intern))
                flags, v, g = 0, 0xFFFF, 0
                if link is None:
                    flags |= kv._lib.PF_IOMMU_ERR
                else:
                    g = intern.setdefault(link.rsplit(b"/", 1)[-1], len(intern))
                if vendor is None or len(vendor) < 2:
                    flags |= kv._lib.PF_VENDOR_ERR
                elif vendor[2:].strip(b"\n") == b"10de":
                    v = 0x10DE
                recs.append((len(recs), v, 0, g, 0, flags, 0))
                want.append(w)
            ids.extend(eh.get(serve.egm_key(i.decode()), len(eh)) for i in dids)
            n_members.append(len(members))
            n_ids.append(len(dids))
        bad, t = ctx.pci_allocate_check(np.array(recs, dtype=kv.PCI_REC), want, n_members, ids, n_ids, eoff, egpu,
                                        len(eh))
        assert fb.tolist() == bad.tolist()
        kept_idx = np.nonzero(kept)[0]
        assert np.array_equal(take[:, kept_idx], t) and not take[:, ~kept].any()


# ---- isolation ----------------------------------------------------------------------------------
def _same(a, b):
    for f in a.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def _in_between(kv, ctx):
    rng = np.random.default_rng(11)
    for _ in range(3):
        check(kv, ctx, *AR.random_call(rng))
    check(kv, ctx, [([AR.ok_member()] * 5000, AR.IDS)], AR.edge_egm())


@pytest.fixture(scope="module")
def ids():
    return O.nv_ids(util.pciids_text())


@pytest.mark.parametrize("n", [16, 50_000])
def test_device_scan_and_fetch_are_untouched(kv, ctx, ids, n):
    import torch
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
    assert len(want.changes) > 0


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
    want = run(False)
    assert run(True) == want
    assert any(len(c) for _, _, c in want)
