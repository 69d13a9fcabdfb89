"""kvg_pci_allocate_raw's kernels (csrc/kvg_alloc_raw.cuh, then k_pci_allocate_check) executed on the CPU from their
real source under the warp emulator of tools/emu/, in the library's launch order, against the Go-exact restatement of
tests/allocate_raw_cases.py: every named edge, a few hundred seeded calls, both sides of the EGM key cap, and the
device's unicode.ToLower for every code point.  Also: tools/gen_case_table.py reproduces the committed table."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import conftest
import allocate_raw_cases as AR
import kvgpu

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

PASS, FAIL, PANIC, MISS_LINK, MISS_VENDOR = range(5)   # ARAW_*
BDF0 = AR.BDF[0]


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("alloc_raw"))
    lib.emu_pci_allocate_raw.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 3 + [C.c_uint32] + \
        [C.c_void_p] * 2 + [C.c_uint32] + [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 5
    lib.emu_case_lower.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    return lib


def run(emu, requests, egm):
    """the kernels, then what the library's driver reads from their outputs -> (first_bad, panic, kept, take), or
    raises AR.RawError"""
    raw = kvgpu.pack_alloc_raw(requests, egm)
    n_reqs, n_egm, n_mem = len(requests), len(egm), len(raw.member_state)
    reqs = np.zeros((max(n_reqs, 1), 2), dtype=np.uint32)
    reqs[:n_reqs, 0], reqs[:n_reqs, 1] = raw.n_members, raw.n_ids
    arr = lambda a, t: np.ascontiguousarray(a, dtype=t)   # noqa: E731
    moff, mst, ioff = arr(raw.member_off, np.uint32), arr(raw.member_state, np.uint16), arr(raw.id_off, np.uint32)
    eoff, est = arr(raw.egm_off, np.uint32), arr(raw.egm_state, np.uint16)
    mb, ib, eb = (np.frombuffer(b + b"\0", dtype=np.uint8) for b in (raw.member_bytes, raw.id_bytes, raw.egm_bytes))
    first_bad = np.zeros(max(n_reqs, 1), dtype=np.uint32)
    code = np.zeros(max(n_mem, 1), dtype=np.uint8)
    kept = np.zeros(max(n_egm, 1), dtype=np.uint8)
    take = np.zeros(max(n_reqs * n_egm, 1), dtype=np.uint8)
    verdict = np.zeros(2, dtype=np.uint64)
    rc = emu.emu_pci_allocate_raw(reqs.ctypes.data, n_reqs, moff.ctypes.data, mst.ctypes.data, mb.ctypes.data, n_mem,
                                  ioff.ctypes.data, ib.ctypes.data, len(ioff) - 1, eoff.ctypes.data, est.ctypes.data,
                                  eb.ctypes.data, n_egm, first_bad.ctypes.data, code.ctypes.data, kept.ctypes.data,
                                  take.ctypes.data, verdict.ctypes.data)
    assert rc == 0
    none = (1 << 64) - 1
    if int(verdict[0]) != none:
        w = int(verdict[0])
        raise AR.RawError("miss", ("egm", w >> 8, {1: "gpu_devices", 2: "stat"}[w & 0xFF]))
    m0 = 0
    for r in range(n_reqs):
        n = int(raw.n_members[r])
        if first_bad[r] < n and code[m0 + first_bad[r]] in (MISS_LINK, MISS_VENDOR):
            raise AR.RawError("miss", ("member", r, int(first_bad[r])))
        m0 += n
    if int(verdict[1]) != none:
        raise AR.RawError("range", ("egm", int(verdict[1]) >> 8))
    panic, m0 = [], 0
    for r in range(n_reqs):
        n = int(raw.n_members[r])
        panic.append(bool(first_bad[r] < n and code[m0 + first_bad[r]] == PANIC))
        m0 += n
    return (first_bad[:n_reqs], np.array(panic, dtype=bool), kept[:n_egm].astype(bool),
            take[:n_reqs * n_egm].reshape(n_reqs, n_egm).astype(bool))


def check(emu, requests, egm):
    try:
        want = AR.allocate_raw(requests, egm)
    except AR.RawError as e:
        with pytest.raises(AR.RawError) as got:
            run(emu, requests, egm)
        assert (got.value.kind, got.value.where) == (e.kind, e.where)
        return None
    got = run(emu, requests, egm)
    for g, w in zip(got, want):
        assert g.tolist() == w.tolist(), (requests, egm)
    return got


@pytest.mark.parametrize("name,requests", AR.edge_requests(), ids=[n for n, _ in AR.edge_requests()])
def test_member_edges(emu, name, requests):
    got = check(emu, requests, [])
    assert got is not None


def test_member_edge_answers(emu):
    want = {"vendor_empty": (1, True), "vendor_x": (1, True), "vendor_0x": (1, False), "vendor_0x10de": (2, False),
            "vendor_0x10de_nl": (2, False), "vendor_0x10DE": (1, False), "vendor_failed": (1, False),
            "link_path": (2, False), "link_bare": (2, False), "link_trailing_slash": (1, False),
            "link_zero_padded": (1, False), "link_failed": (1, False), "link_nl": (1, False),
            "panic_behind_failure": (1, False), "panic_behind_failed_link": (0, False),
            "panic_behind_moved_link": (0, False)}
    for name, requests in AR.edge_requests():
        if name in want:
            fb, p, _, _ = run(emu, requests, [])
            assert (int(fb[0]), bool(p[0])) == want[name], name
    fb, p, _, _ = run(emu, dict(AR.edge_requests())["later_request_panics"], [])
    assert fb.tolist() == [0, 0, 1] and p.tolist() == [False, True, False]


@pytest.mark.parametrize("name,requests,egm", AR.edge_refusals(), ids=[n for n, _, _ in AR.edge_refusals()])
def test_refusals(emu, name, requests, egm):
    assert check(emu, requests, egm) is None


def test_egm_edges(emu):
    egm = AR.edge_egm()
    reqs = [([AR.ok_member()], ids) for ids in AR.edge_id_sets()]
    got = check(emu, reqs, egm)
    kept = dict(zip([e[0] for e in egm], got[2]))
    assert not kept[b"egm_whitespace"] and not kept[b"egm_failed"] and not kept[b"egm_nonode"]
    assert not kept[b"gpu0"] and not kept[b"eg"] and not kept[b"Egm1"] and not kept[b"egm_notread_nofields"]
    assert kept[b"egm_x1c"] and kept[b"egm_ff"] and kept[b"egm"]
    col = {e[0]: k for k, e in enumerate(egm)}
    ids = AR.edge_id_sets()
    t = lambda i, name: bool(got[3][i, col[name]])   # noqa: E731
    assert t(ids.index([b"0000:01:00.0\x1c0000:02:00.0"]), b"egm_x1c")   # \x1c is not a space: one field
    assert not t(2, b"egm_x1c") and t(2, b"egm_nbsp") and t(2, b"egm_ideographic") and t(2, b"egm_plain")
    assert not t(2, b"egm_raw_x85") and t(2, b"egm_u0085")               # a raw \x85 byte is RuneError, not U+0085
    assert t(ids.index([b"\xfe"]), b"egm_ff")                            # "\xff" and "\xfe" are one key
    assert t(ids.index([b"K", BDF0]), b"egm_kelvin")                     # U+212A lowers to "k"
    assert t(ids.index([b"\t0000:01:00.0 ", b"ID", b"0000:02:00.0"]), b"egm_dotted_i")   # "İd" lowers to "id"
    assert t(ids.index([b"0000:0a:00.0", b"0000:02:00.0"]), b"egm_upper")
    assert not t(2, b"egm_invalid") and t(8, b"egm") and t(8, b"egm_one")


@pytest.mark.parametrize("seed", range(300))
def test_seeded_calls(emu, seed):
    rng = np.random.default_rng(seed)
    check(emu, *AR.random_call(rng))


def test_key_cap_both_sides(emu):
    # 65,535 distinct keys fit; the 65,536th is the range error of the entry that carries it
    keys = [b"%05x" % k for k in range(65536)]
    egm = [(b"egm%04d" % e, b" ".join(keys[e * 16:(e + 1) * 16]), True) for e in range(4096)]
    last = (b"egm4095", b" ".join(keys[4095 * 16:65535] + [keys[0]]), True)
    reqs = [([AR.ok_member()], [k.upper() if j % 2 else k for j, k in enumerate(keys[:16])]),
            ([AR.ok_member()], keys[1:17])]
    got = check(emu, reqs, egm[:4095] + [last])
    assert got[2].all() and got[3][0].tolist() == [True] + [False] * 4095 and not got[3][1].any()
    assert check(emu, reqs, egm) is None


def test_case_lower_every_code_point(emu):
    cps = np.arange(0x110000, dtype=np.uint32)
    out = np.zeros_like(cps)
    emu.emu_case_lower(cps.ctypes.data, out.ctypes.data, len(cps))
    want = np.array([AR.go_lower(int(c)) for c in cps], dtype=np.uint32)
    bad = np.nonzero(out != want)[0]
    assert len(bad) == 0, ["U+%04X" % c for c in bad[:10]]
    assert int(out[0x130]) == 0x69 and int(out[0x212A]) == ord("k") and int(out[ord("A")]) == ord("a")


def test_generator_reproduces_the_committed_table():
    gen = os.path.join(conftest.ROOT, "tools", "gen_case_table.py")
    got = subprocess.run([sys.executable, gen, "--stdout"], capture_output=True, check=True).stdout
    with open(os.path.join(conftest.ROOT, "kubevirt-gpu-device-plugin_b200", "csrc", "kvg_case.cuh"), "rb") as f:
        assert got == f.read()
    assert b"1407 mappings" in got
