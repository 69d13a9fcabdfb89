"""k_pci_group_check (kvg_pci_group_check's kernel) executed on the CPU from its real source under the warp emulator of
tools/emu/, in its launch shape (one CTA, striding), against the passthrough plugin's Allocate-time rule restated in
numpy (tests/group_check_cases.py): every combination of the fields the rule reads, random values in every field it
ignores, and the smallest failing index at every size regime of the block reduction."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import group_check_cases as GC

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

THREADS = 1024  # GROUP_CHECK_THREADS


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_classify())
    L.emu_pci_group_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    return L


def run(emu, recs, want) -> int:
    recs = np.ascontiguousarray(recs)
    want = np.ascontiguousarray(want, dtype=np.uint32)
    out = np.array([0xeeeeeeee, 0], dtype=np.uint32)      # first_bad, sequence word
    assert emu.emu_pci_group_check(recs.ctypes.data, want.ctypes.data, len(recs), out[:1].ctypes.data,
                                   out[1:].ctypes.data) == 0
    assert int(out[1]) == 7
    return int(out[0])


def test_every_combination_of_the_fields_the_rule_reads(emu):
    rng = np.random.default_rng(1)
    combos = GC.combinations()
    assert len(combos) == 32
    for combo in combos:
        for _ in range(4):                                  # the ignored fields drawn anew each time
            recs, want = GC.noise(1, rng)
            GC.apply(recs, want, 0, combo)
            ok = not combo[0] and not combo[1] and combo[2] == 0x10de and combo[3]
            assert run(emu, recs, want) == (1 if ok else 0), combo
    # all 32 in one call, in every order: the first failing one is found
    recs, want = GC.noise(len(combos), rng)
    for i, combo in enumerate(combos):
        GC.apply(recs, want, i, combo)
    for _ in range(8):
        p = rng.permutation(len(combos))
        assert run(emu, recs[p], want[p]) == GC.first_bad(recs[p], want[p])


def test_ignored_fields_never_fail_a_record(emu):
    rng = np.random.default_rng(2)
    recs, want = GC.noise(3000, rng)
    recs["flags"][::3] |= 2 | 8                             # DRIVER_ERR | DEVICE_ERR
    recs["driver"][1::3] = 0
    recs["device"][2::3] = 0
    assert GC.first_bad(recs, want) == len(recs)
    assert run(emu, recs, want) == len(recs)


@pytest.mark.parametrize("n", [1, 31, 32, 33, THREADS - 1, THREADS, THREADS + 1, 5000])
def test_smallest_failing_index_wins(emu, n):
    rng = np.random.default_rng(n)
    for at in GC.failure_sets(n, rng):
        recs, want = GC.with_failures(n, at, rng)
        want_idx = min(at) if at else n
        assert GC.first_bad(recs, want) == want_idx
        assert run(emu, recs, want) == want_idx, at
