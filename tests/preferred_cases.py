"""Calls of the passthrough plugin's GetPreferredAllocation (generic_device_plugin.go:470-608) for the NUMA packing on the
GPU (kvg_preferred_allocation), and its C-ABI contract restated in plain Python.

A call is (devs, requests): devs as GenericDevicePlugin builds them, [(device id, NUMA node or None)], and requests
[(available, must_include, size)] in request order.  `reference` answers a call with serve.preferred_allocation, the
reference rule, request by request; `contract` answers the C-ABI's question (entry positions in, picks as positions
out) without the GPU, and stands in for Context.preferred_allocation on the CPU."""
import json
import os

import numpy as np

import conftest  # noqa: F401  (sys.path)
from kvgpu import _lib as L
from kvgpu import serve

HERE = os.path.dirname(os.path.abspath(__file__))
NONE = L.PREF_NODE_NONE


# ---- the two answers ---------------------------------------------------------------------------------------------
def reference(devs, requests):
    """("ok", [[ids] per request]) or ("error", text of the first failing request), by serve.preferred_allocation."""
    out = []
    for available, must, size in requests:
        try:
            out.append(serve.preferred_allocation(devs, available, must, size))
        except serve.AllocateError as e:
            return "error", str(e)
    return "ok", out


def contract(ids, n_must, n_avail, sizes) -> list:
    """kvg_preferred_allocation on the CPU: (n_out, n_must_distinct, positions) per request, as
    Context.preferred_allocation returns them.  Handles and nodes are the interned values of include/kvgpu.h."""
    out, at = [], 0
    for m, a, size in zip(n_must, n_avail, sizes):
        m, a, size = int(m), int(a), int(size)
        h = [int(x) for x in ids["handle"][at:at + m + a]]
        nd = [int(x) for x in ids["node"][at:at + m + a]]
        at += m + a
        first = {}
        for p, x in enumerate(h):
            first.setdefault(x, p)
        picks = [p for p in range(m) if first[h[p]] == p]      # distinct must-include IDs, in order
        n_p = len(picks)
        if n_p > size:
            out.append((-1, n_p, np.zeros(0, dtype=np.int64)))
            continue
        fresh = [p for p in range(m, m + a) if first[h[p]] == p]    # available IDs that are not must-include, once
        if n_p < size:
            sel, free, key = {}, {}, {}
            for p in range(m + a):
                key.setdefault(nd[p], p)                         # must nodes first, then order of first appearance
            for p in picks:
                sel[nd[p]] = sel.get(nd[p], 0) + 1
            for p in range(m, m + a):
                if first[h[p]] >= m:
                    free[nd[p]] = free.get(nd[p], 0) + 1         # duplicates counted
            qualify = [key[n] for n in key if sel.get(n, 0) + free.get(n, 0) >= size]
            target = nd[min(qualify)] if qualify else NONE
            if target != NONE:                                   # the -1 node stops the search without a fill
                picks += [p for p in fresh if nd[p] == target][:size - len(picks)]
            taken = set(picks)
            picks += [p for p in fresh if p not in taken][:size - len(picks)]
        out.append((len(picks), n_p, np.array(picks, dtype=np.int64)))
    return out


# ---- the calls -----------------------------------------------------------------------------------------------------
def golden_calls() -> list:
    """The reference's own vectors (tests/golden/plugin_vectors.json) and every case of test_preferred_allocation_edges,
    one request per call."""
    p = json.load(open(os.path.join(HERE, "golden", "plugin_vectors.json")))["preferred_allocation"]
    devs = [(d["id"], d["numa"]) for d in p["devs"]]
    calls = [(devs, [(c["available"], c["must_include"], c["size"])]) for c in p["cases"]]
    edges = [("a", 0), ("b", 0), ("c", 1), ("d", None), ("e", None)]
    for available, must, size in ((["c", "a", "b"], [], 2), (["c", "a", "b"], [], 1), (["a", "c"], [], 2),
                                  (["d", "e", "a", "b"], [], 2), (["a", "b", "c"], ["c", "c"], 1), (["a", "b"], [], 0),
                                  (["a"], [], 3), (["a", "b", "c"], ["x"], 2)):
        calls.append((edges, [(available, must, size)]))
    return calls


DEVS = [("a", 0), ("b", 0), ("c", 1), ("d", 1), ("e", 1), ("f", None), ("g", -1), ("h", -2), ("i", -2), ("j", 2)]


def named_calls() -> dict:
    """One call per quirk of the rule, by name."""
    one = lambda available, must, size, devs=DEVS: (devs, [(available, must, size)])  # noqa: E731
    return {
        "size 0": one(["a", "b"], [], 0),
        "size 0 with a must-include ID": one(["a", "b"], ["a"], 0),
        "negative size": one(["a", "b"], [], -1),
        "negative size with must-include IDs": one(["a", "b"], ["c"], -3),
        "size above the available entries": one(["a", "c", "z"], [], 9),
        "empty lists": one([], [], 0),
        "empty lists, size 1": one([], [], 1),
        "empty lists, negative size": one([], [], -1),
        "only must-include IDs": one([], ["c", "a"], 2),
        "only must-include IDs, short": one([], ["c", "a"], 4),
        "duplicate available IDs": one(["c", "c", "a", "c", "d"], [], 3),
        "duplicate must-include IDs": one(["a", "b", "c"], ["c", "a", "c", "a"], 3),
        "must-include IDs also available": one(["a", "c", "b", "d"], ["d", "a"], 3),
        "unknown must-include ID": one(["a", "b", "c"], ["zz", "zz"], 3),
        "unknown available IDs": one(["q", "a", "r", "b"], [], 2),
        "node -1 against no topology against unknown": one(["g", "f", "u", "a"], [], 3),
        "node -1 group first": one(["f", "g", "a", "b"], [], 2),
        "node -2 as the target": one(["a", "h", "c", "i"], [], 2),
        "node -2 from a must-include ID": one(["a", "b", "i"], ["h"], 2),
        "first qualifying candidate is -1, the fallback decides": one(["f", "a", "g", "b"], [], 2),
        "-1 candidate from an unknown must-include ID": one(["a", "b", "c", "d"], ["zz"], 2),
        "duplicates qualify a node but its distinct fill is short": one(["a", "a", "b"], [], 2, [("a", 0), ("b", 1)]),
        "duplicates qualify the must node": one(["c", "c", "a", "b"], ["d"], 3),
        "a must-include node wins over an earlier available node": one(["a", "b", "c", "d", "e"], ["e"], 2),
        "must-include node qualifies only with its must IDs": one(["a", "b", "c"], ["c", "d"], 3),
        "no node qualifies": one(["a", "c", "j"], [], 3),
        "duplicate device IDs, last with topology wins": one(
            ["x", "y", "a", "b", "c"], [], 2,
            [("x", 0), ("x", None), ("x", 1), ("y", 1), ("y", None), ("a", 0), ("b", 0), ("c", 1)]),
        "duplicate device IDs, advertised -1 last": one(["x", "a", "c"], [], 2, [("x", 0), ("x", -1), ("a", 0), ("c", 1)]),
        "several requests": (DEVS, [(["a", "b", "c"], [], 2), (["c", "d", "a"], ["a"], 2), ([], [], 0),
                                    (["f", "g", "h"], [], 3)]),
        "several requests, an error in the middle": (DEVS, [(["a", "b"], [], 1), (["a", "b", "c"], ["a", "c"], 1),
                                                            (["c", "d"], ["c", "d", "e"], 2)]),
        "several requests, the second error is not reported": (DEVS, [(["a"], ["a", "b"], 1), (["a"], [], -2)]),
    }


def random_call(rng, n_reqs: int, max_entries: int) -> tuple:
    """A seeded call: a device list with duplicates, every kind of node (ordinary, -1, -2, none), and per request
    available and must-include lists with duplicates and unknown IDs, and a size from below zero to past the list."""
    n_dev = int(rng.integers(1, max(2, max_entries // 2) + 1))
    n_nodes = int(rng.integers(1, 6))
    node_kinds = list(range(n_nodes)) + [-1, -2, None]
    pool = ["d%d" % k for k in range(n_dev)]
    devs = [(d, node_kinds[int(rng.integers(0, len(node_kinds)))]) for d in pool]
    if n_dev > 1:                                                 # a few IDs listed twice
        for k in rng.integers(0, n_dev, int(rng.integers(0, 3))):
            devs.append((pool[int(k)], node_kinds[int(rng.integers(0, len(node_kinds)))]))
    known = pool + ["ghost%d" % k for k in range(int(rng.integers(0, 3)))]
    requests = []
    for _ in range(n_reqs):
        n_avail = int(rng.integers(0, max_entries + 1))
        available = [known[int(k)] for k in rng.integers(0, len(known), n_avail)]
        n_must = int(rng.integers(0, min(4, max_entries) + 1)) if rng.random() < 0.6 else 0
        must = [(available + known)[int(k)] for k in rng.integers(0, len(available) + len(known), n_must)]
        size = int(rng.integers(-2, len(set(available)) + 4))
        requests.append((available, must, size))
    return devs, requests


def all_calls(seed: int = 0, n_random: int = 40, max_reqs: int = 6, max_entries: int = 24) -> list:
    rng = np.random.default_rng(seed)
    calls = golden_calls() + list(named_calls().values())
    calls += [random_call(rng, int(rng.integers(1, max_reqs + 1)), max_entries) for _ in range(n_random)]
    return calls


def packed(devs, requests, call) -> tuple:
    """The call through serve.NumaPacker on `call` (Context.preferred_allocation or a stand-in), in reference's shape."""
    try:
        return "ok", serve.NumaPacker(call)(devs, requests)
    except serve.AllocateError as e:
        return "error", str(e)


class Recorder:
    """Context.preferred_allocation, or the contract standing in for it, with the arguments and the answer of every
    call kept."""

    def __init__(self, call=contract):
        self.call, self.calls = call, []

    def __call__(self, ids, n_must, n_avail, sizes):
        out = self.call(ids, n_must, n_avail, sizes)
        self.calls.append((np.array(ids, copy=True), list(n_must), list(n_avail), list(sizes), out))
        return out
