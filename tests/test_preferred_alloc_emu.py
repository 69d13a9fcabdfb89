"""k_preferred_alloc (kvg_preferred_allocation's kernel) executed on the CPU from its real source under the warp emulator
of tools/emu/, in its launch shape (one CTA per container request, poisoned scratch), against the reference rule
serve.preferred_allocation through serve.NumaPacker's marshalling, and against the C-ABI contract restated in
tests/preferred_cases.py: the same picks, counts and error texts on every generated call, from empty requests to 5,000
entries per request and up to 64 requests per call."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import preferred_cases as PC
from kvgpu import _lib as L

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

THREADS = 1024  # PREF_THREADS


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build_classify())
    lib.emu_preferred_allocation.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                             C.c_void_p]

    def call(ids, n_must, n_avail, sizes):
        """Context.preferred_allocation's shape on the emulator."""
        ids = np.ascontiguousarray(ids, dtype=L.PREF_ID)
        reqs = np.zeros(len(sizes), dtype=L.PREF_REQ)
        reqs["n_must"], reqs["n_avail"], reqs["size"] = n_must, n_avail, sizes
        res = np.full(len(reqs), 0x5a, dtype=L.PREF_RES)
        pos = np.full(max(len(ids), 1), 0xeeeeeeee, dtype=np.uint32)
        seq = np.zeros(1, dtype=np.uint32)
        assert lib.emu_preferred_allocation(reqs.ctypes.data, len(reqs), ids.ctypes.data, len(ids), res.ctypes.data,
                                            pos.ctypes.data, seq.ctypes.data) == 0
        assert seq[0] == 7
        out, at = [], 0
        for r in range(len(reqs)):
            n = int(res["n_out"][r])
            out.append((n, int(res["n_must_distinct"][r]), pos[at:at + max(n, 0)].astype(np.int64)))
            at += int(n_must[r]) + int(n_avail[r])
        return out
    return call


def same_raw(a, b):
    assert len(a) == len(b)
    for (n, p, pos), (n2, p2, pos2) in zip(a, b):
        assert (n, p) == (n2, p2)
        assert pos.tolist() == pos2.tolist()


def check(emu, devs, requests):
    """The emulated kernel through NumaPacker answers as the reference; its raw output is the contract's."""
    rec = PC.Recorder(emu)
    got = PC.packed(devs, requests, rec)
    assert got == PC.reference(devs, requests), (devs, requests)
    assert len(rec.calls) == 1
    ids, n_must, n_avail, sizes, raw = rec.calls[0]
    same_raw(raw, PC.contract(ids, n_must, n_avail, sizes))
    return got


def test_golden_vectors_and_edges(emu):
    for devs, requests in PC.golden_calls():
        check(emu, devs, requests)


@pytest.mark.parametrize("name", sorted(PC.named_calls()))
def test_named_quirks(emu, name):
    devs, requests = PC.named_calls()[name]
    check(emu, devs, requests)


def test_seeded_calls(emu):
    rng = np.random.default_rng(7)
    for _ in range(100):
        check(emu, *PC.random_call(rng, int(rng.integers(1, 7)), int(rng.integers(1, 40))))


def _large(n, rng, size, n_must=0):
    """One request of n available entries over a few nodes (one of them -1), with duplicates and unknown IDs."""
    pool = ["p%d" % k for k in range(max(1, n // 2))]
    nodes = [0, 1, 2, -1, None]
    devs = [(d, nodes[k % len(nodes)]) for k, d in enumerate(pool)]
    known = pool + ["ghost"]
    available = [known[int(k)] for k in rng.integers(0, len(known), n)]
    must = [known[int(k)] for k in rng.integers(0, len(known), n_must)]
    return devs, [(available, must, size)]


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, THREADS - 1, THREADS, THREADS + 1, 2 * THREADS + 1, 5000])
def test_every_chunk_regime(emu, n):
    """Sizes that stop the fill and the fallback inside the first chunk, on a chunk edge and several chunks in."""
    rng = np.random.default_rng(n)
    for size in sorted({0, 2, n // 7, n // 2, n - 1, n + 3, THREADS, THREADS + 1}):
        for n_must in (0, 3):
            check(emu, *_large(n, rng, size, n_must))


def test_sixty_four_requests_per_call(emu):
    rng = np.random.default_rng(64)
    for _ in range(3):
        check(emu, *PC.random_call(rng, 64, 40))
    devs, requests = PC.random_call(rng, 64, 40)
    requests = [(av, must, max(size, len(set(must)))) for av, must, size in requests]
    requests[37] = (["a", "b"], ["x", "y", "z"], 2)               # the one error, in the middle
    assert check(emu, devs, requests) == ("error", "number of MustIncludeDeviceIDs (3) exceeds allocation size (2)")
    # several large requests in one call, each CTA on its own slice of the scratch
    big = [_large(n, rng, s, m)[1][0] for n, s, m in ((3000, 1500, 2), (1025, 1025, 0), (4000, 7, 3), (0, 0, 0))]
    check(emu, _large(4000, rng, 0)[0], big)
