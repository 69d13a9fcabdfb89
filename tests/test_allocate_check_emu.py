"""k_pci_allocate_check (kvg_pci_allocate_check's kernel) executed on the CPU from its real source under the warp
emulator of tools/emu/, in its launch shape (one CTA per container request), against the C-ABI contract restated in
tests/allocate_check_cases.py: 0 to 64 requests per call, 0 to 5,000 members per request, 0 to 64 EGM devices of 0 to 8
GPUs each, the named quirks of the EGM match, and the one-request form kvg_pci_group_check launches, which gives what
the group check gave before it shared this kernel."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import allocate_check_cases as AC
import conftest
import group_check_cases as GC
from kvgpu import _lib as L

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

THREADS = 1024  # GROUP_CHECK_THREADS


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build_classify())
    lib.emu_pci_allocate_check.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_uint32] + \
        [C.c_void_p] * 3
    lib.emu_pci_group_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]

    def call(recs, want, n_members, ids, n_ids, egm_off, egm_gpu, n_egm_gpus):
        """Context.pci_allocate_check's shape on the emulator; outputs poisoned before the launch."""
        assert AC.refusal(recs, want, n_members, ids, n_ids, egm_off, egm_gpu, n_egm_gpus) is None
        reqs = np.zeros(len(n_members), dtype=L.ALLOC_REQ)
        reqs["n_members"], reqs["n_ids"] = n_members, n_ids
        recs, want = np.ascontiguousarray(recs), np.ascontiguousarray(want, dtype=np.uint32)
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        egm_off, egm_gpu = np.ascontiguousarray(egm_off, np.uint32), np.ascontiguousarray(egm_gpu, np.uint32)
        n_egm = max(len(egm_off) - 1, 0)
        first_bad = np.full(max(len(reqs), 1), 0xeeeeeeee, dtype=np.uint32)
        take = np.full(max(len(reqs) * n_egm, 1), 0x5a, dtype=np.uint8)
        seq = np.zeros(1, dtype=np.uint32)
        rc = lib.emu_pci_allocate_check(reqs.ctypes.data, len(reqs), recs.ctypes.data, want.ctypes.data,
                                        ids.ctypes.data, egm_off.ctypes.data, egm_gpu.ctypes.data, n_egm, n_egm_gpus,
                                        first_bad.ctypes.data, take.ctypes.data, seq.ctypes.data)
        if len(reqs) == 0:
            assert rc == -1                               # no launch, as the library makes none
            return np.zeros(0, np.uint32), np.zeros((0, n_egm), bool)
        assert rc == 0 and seq[0] == 7
        assert set(np.unique(take[:len(reqs) * n_egm]).tolist()) <= {0, 1}
        return first_bad[:len(reqs)], take[:len(reqs) * n_egm].reshape(len(reqs), n_egm).astype(bool)
    call.lib = lib
    return call


def check(emu, c):
    got_bad, got_take = emu(**c)
    want_bad, want_take = AC.contract(**c)
    assert got_bad.tolist() == want_bad.tolist()
    assert np.array_equal(got_take, want_take)


@pytest.mark.parametrize("name", sorted(AC.named_calls()))
def test_named_quirks(emu, name):
    check(emu, AC.named_calls()[name])


def test_seeded_calls(emu):
    rng = np.random.default_rng(3)
    for _ in range(60):
        check(emu, AC.random_call(rng, int(rng.integers(0, 9))))


@pytest.mark.parametrize("n_reqs", [0, 1, 2, 17, 64])
def test_requests_per_call(emu, n_reqs):
    rng = np.random.default_rng(100 + n_reqs)
    for _ in range(3):
        check(emu, AC.random_call(rng, n_reqs, max_members=60, n_egm=int(rng.integers(0, 65))))


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, THREADS - 1, THREADS, THREADS + 1, 5000])
def test_members_per_request(emu, n):
    """The block reduction at every size regime, with a small request on either side."""
    rng = np.random.default_rng(n)
    for at in (GC.failure_sets(n, rng) if n else [[]]):
        recs, want = GC.with_failures(n, at, rng)
        tiny_r, tiny_w = AC.records([2, 3], rng)
        c = AC.make_call(np.concatenate([tiny_r[:2], recs, tiny_r[2:]]), np.concatenate([tiny_w[:2], want, tiny_w[2:]]),
                         [2, n, 3], [0, 1, 2, 0, 1], [1, 3, 1], [[0], [0, 1, 2]], 3)
        bad, take = emu(**c)
        assert int(bad[1]) == (min(at) if at else n), at
        assert take.tolist() == [[True, False], [True, True], [False, False]]
        check(emu, c)


@pytest.mark.parametrize("n_egm", [1, 8, 33, 64])
def test_egm_devices(emu, n_egm):
    """0 to 8 GPUs per device, requests that hold all, all but one, or none of a device's GPUs."""
    rng = np.random.default_rng(n_egm)
    for _ in range(4):
        lists = [[int(g) for g in rng.choice(200, int(rng.integers(0, 9)), replace=False)] for _ in range(n_egm)]
        n_reqs = int(rng.integers(1, 9))
        ids, n_ids = [], []
        for r in range(n_reqs):
            e = lists[r % n_egm]
            mine = list(e) if r % 3 == 0 else e[1:] if r % 3 == 1 else []
            mine += [int(g) for g in rng.integers(0, 260, 6)]
            ids += mine
            n_ids.append(len(mine))
        n_members = [int(rng.integers(0, 20)) for _ in range(n_reqs)]
        recs, want = AC.records(n_members, rng)
        check(emu, AC.make_call(recs, want, n_members, ids, n_ids, lists, 200))


def test_one_request_without_egm_is_the_group_check(emu):
    """emu_pci_group_check is kvg_pci_group_check's launch; it answers as the one-request call, and as the group
    check's numpy rule answered before the two shared a kernel."""
    rng = np.random.default_rng(5)
    for n in (1, 32, 1000, 3000):
        for at in GC.failure_sets(n, rng):
            recs, want = GC.with_failures(n, at, rng)
            out = np.array([0xeeeeeeee, 0], dtype=np.uint32)
            assert emu.lib.emu_pci_group_check(recs.ctypes.data, want.ctypes.data, n, out[:1].ctypes.data,
                                               out[1:].ctypes.data) == 0
            assert out[1] == 7
            bad, take = emu(**AC.make_call(recs, want, [n], [], [0], []))
            assert int(out[0]) == int(bad[0]) == GC.first_bad(recs, want)
            assert take.shape == (1, 0)


def test_contract_refusals():
    """The contract refuses what the header refuses, and accepts the call each refusal is one change away from."""
    calls = AC.refused_calls()
    for name, c in calls.items():
        why = AC.refusal(**c)
        assert (why is None) == (name == "accepted"), (name, why)
        if why:
            with pytest.raises(ValueError):
                AC.contract(**c)
