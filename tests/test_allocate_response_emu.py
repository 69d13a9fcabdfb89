"""kvg_pci_allocate_response's kernels (csrc/kvg_alloc_resp.cuh after those of kvg_alloc_raw.cuh) executed on the CPU
from their real source under the warp emulator of tools/emu/, in the library's launch order, against the Go-exact
restatement of tests/allocate_response_cases.py: every named edge with iommufd on and off, the refusals, and 300
seeded calls."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import allocate_raw_cases as AR
import allocate_response_cases as RC
import kvgpu
from kvgpu import _lib as L

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

MISS_LINK, MISS_VENDOR, EV_MISS = 3, 4, 7   # ARAW_MISS_*, ARESP_EV_MISS
NONE = (1 << 64) - 1


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("alloc_resp"))
    lib.emu_pci_allocate_response.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(L.AllocRawC),
                                              C.POINTER(L.AllocRespInC)] + [C.c_void_p] * 13
    return lib


def c_args(raw, resp):
    """(reqs, AllocRawC, AllocRespInC, keep-alive) as Context.pci_allocate_response builds them"""
    arr = lambda a, t: np.ascontiguousarray(a, dtype=t)   # noqa: E731
    blob = lambda b: np.frombuffer(bytes(b) + b"\0", dtype=np.uint8)   # noqa: E731
    reqs = np.zeros(max(len(raw.n_members), 1), dtype=L.ALLOC_REQ)
    reqs["n_members"][:len(raw.n_members)], reqs["n_ids"][:len(raw.n_ids)] = raw.n_members, raw.n_ids
    keep = [arr(raw.member_off, np.uint32), blob(raw.member_bytes), arr(raw.member_state, np.uint16),
            arr(raw.id_off, np.uint32), blob(raw.id_bytes), arr(raw.egm_off, np.uint32), blob(raw.egm_bytes),
            arr(raw.egm_state, np.uint16)]
    a = L.AllocRawC(len(raw.member_state), keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data,
                    len(raw.id_off) - 1, keep[3].ctypes.data, keep[4].ctypes.data, len(raw.egm_state),
                    keep[5].ctypes.data, keep[6].ctypes.data, keep[7].ctypes.data)
    k2 = [arr(resp.n_visited, np.uint32), arr(resp.lookup_error, np.uint8), arr(resp.id_members, np.uint32),
          arr(resp.addr_off, np.uint32), blob(resp.addr_bytes), arr(resp.vfio_first, np.uint32),
          arr(resp.vfio_off, np.uint32), blob(resp.vfio_bytes), arr(resp.vfio_dir, np.uint8),
          arr(resp.vfio_state, np.uint8)]
    b = L.AllocRespInC(int(resp.iommufd), *[x.ctypes.data for x in k2])
    return reqs, a, b, keep + k2


def run(emu, requests, egm, iommufd):
    """the kernels, then what the library's driver reads from their outputs -> the restatement's form, or raises
    AR.RawError"""
    raw, resp = kvgpu.pack_alloc_response(requests, egm, iommufd)
    reqs, a, b, keep = c_args(raw, resp)
    n, n_mem = len(requests), len(raw.member_state)
    sizes = np.zeros(2, dtype=np.uint64)
    nul = [None] * 12
    assert emu.emu_pci_allocate_response(reqs.ctypes.data, n, C.byref(a), C.byref(b), sizes.ctypes.data, *nul) == 0
    u32 = lambda k: np.zeros(max(k, 1), dtype=np.uint32)   # noqa: E731
    u8 = lambda k: np.zeros(max(k, 1), dtype=np.uint8)   # noqa: E731
    bad, err, at, first, nspec, elen = u32(n), u8(n), u32(n), u32(n), u32(n), u32(n)
    span, pool, ekey = u32(2 * int(sizes[0])), u8(int(sizes[1])), u8(n)
    env, code, verd = u8(int(resp.addr_off[-1]) + n_mem), u8(n_mem), np.zeros(4, dtype=np.uint64)
    rc = emu.emu_pci_allocate_response(reqs.ctypes.data, n, C.byref(a), C.byref(b), sizes.ctypes.data,
                                       *[x.ctypes.data for x in (bad, err, at, first, nspec, span, pool, elen, ekey,
                                                                 env, code, verd)])
    assert rc == 0
    if int(verd[2]) != NONE:
        raise AR.RawError("group", int(verd[2]))
    if int(verd[3]) != NONE:
        raise AR.RawError("order", int(verd[3]))
    if int(verd[0]) != NONE:
        raise AR.RawError("miss", ("egm", int(verd[0]) >> 8, {1: "gpu_devices", 2: "stat"}[int(verd[0]) & 0xFF]))
    m0 = 0
    for r in range(n):
        k = int(raw.n_members[r])
        if bad[r] < k and code[m0 + bad[r]] in (MISS_LINK, MISS_VENDOR):
            raise AR.RawError("miss", ("member", r, int(bad[r])))
        if err[r] == EV_MISS:
            raise AR.RawError("miss", ("listing", r, int(at[r])))
        m0 += k
    if int(verd[1]) != NONE:
        raise AR.RawError("range", ("egm", int(verd[1]) >> 8))
    out = []
    for r in range(n):
        paths = [bytes(pool[span[2 * (first[r] + s)]:span[2 * (first[r] + s)] + span[2 * (first[r] + s) + 1]])
                 for s in range(int(nspec[r]))]
        out.append((int(err[r]), int(at[r]), paths, bytes(env[:elen[r]]) if ekey[r] else None))
    return out


def check(emu, requests, egm, iommufd):
    try:
        want = RC.allocate_response(requests, egm, iommufd)
    except AR.RawError as e:
        with pytest.raises(AR.RawError) as got:
            run(emu, requests, egm, iommufd)
        assert (got.value.kind, got.value.where) == (e.kind, e.where)
        return None
    got = run(emu, requests, egm, iommufd)
    assert got == want, (requests, egm, iommufd)
    return got


@pytest.mark.parametrize("name,requests,egm,iommufd", RC.edge_calls(),
                         ids=["%s-%s" % (c[0], "iommufd" if c[3] else "noiommufd") for c in RC.edge_calls()])
def test_edges(emu, name, requests, egm, iommufd):
    check(emu, requests, egm, iommufd)


@pytest.mark.parametrize("name,requests,egm,iommufd", RC.edge_refusals(), ids=[c[0] for c in RC.edge_refusals()])
def test_refusals(emu, name, requests, egm, iommufd):
    with pytest.raises(AR.RawError):
        RC.allocate_response(requests, egm, iommufd)
    check(emu, requests, egm, iommufd)


def test_named_outcomes(emu):
    """the matrix's key outcomes, stated outright"""
    calls = {(n, f): (r, e) for n, r, e, f in RC.edge_calls()}

    def got(name, iommufd=True):
        return run(emu, *calls[(name, iommufd)], iommufd)
    assert got("vfio10_before_vfio3")[0][2][0] == b"/dev/vfio/devices/vfio10"
    assert got("file_before_dir")[0][2][0] == b"/dev/vfio/devices/vfio1"
    assert got("symlink_only")[0][:2] == (RC.VFIO_NONE, 0)
    assert got("failed_listing")[0][:2] == (RC.VFIO_READ, 0)
    assert got("unreached_missing")[0][:2] == (RC.UNKNOWN_MEMBER, 0)
    assert got("group_vfio")[0][2] == [b"/dev/vfio/devices/vfio3", b"/dev/vfio/vfio", b"/dev/iommu"]
    assert got("group_empty")[0][2][2] == b"/dev/vfio" and got("group_dotdot")[0][2][2] == b"/dev"
    r = got("id_twice")[0]
    assert r[2] == [b"/dev/vfio/devices/vfio3", b"/dev/vfio/devices/vfio4", b"/dev/vfio/vfio", b"/dev/vfio/42",
                    b"/dev/iommu"]
    assert r[3] == b",".join([RC.A[0], RC.A[1]] * 2)
    assert got("id_absent_vs_vfio_none")[0][:2] == (RC.VFIO_NONE, 1)
    assert got("id_absent", False)[0][:2] == (RC.UNKNOWN_ID, 0)
    assert got("lookup_after_visits")[0][:2] == (RC.UNKNOWN_ID, 1)
    assert got("panic_before_listing_error")[0][:2] == (RC.PANIC, 0)
    e = got("env_empty_then_full")
    assert e[0][3] is None and e[1][3] == RC.A[0]
    e = got("env_full_then_empty")
    assert e[0][3] == RC.A[0] and e[1][3] == RC.A[0]
    assert got("egm_high_bytes")[0][2][-2:] == [b"/dev/egm0", b"/dev/egm\x80"]


def test_seeded_calls(emu):
    rng = np.random.default_rng(20261019)
    kinds = set()
    for _ in range(300):
        requests, egm, iommufd = RC.random_call(rng)
        got = check(emu, requests, egm, iommufd)
        kinds |= {r[0] for r in got or []}
    assert kinds == set(range(6))
