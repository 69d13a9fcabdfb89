"""Calls of the passthrough plugin's Allocate decisions on the GPU (kvg_pci_allocate_check), and its C-ABI contract
restated in plain Python.

A call is a dict of the arguments of Context.pci_allocate_check: recs / want (every member of every request, request
after request), n_members, ids (every request's DevicesIDs as EGM handles, request after request), n_ids, egm_off /
egm_gpu (each EGM device's GPU handles) and n_egm_gpus.  `contract` answers a call without the GPU and stands in for
Context.pci_allocate_check on the CPU; `refusal` says which rule of the header refuses a call.  The records come from
tests/group_check_cases.py, so every field the re-check ignores is random."""
import numpy as np

import conftest  # noqa: F401  (sys.path)
import group_check_cases as GC
from kvgpu import _lib as L

CAP = L.ALLOC_MAX_EGM_GPUS


def refusal(recs, want, n_members, ids, n_ids, egm_off, egm_gpu, n_egm_gpus):
    """The header's KVG_EINVAL rule that refuses the call (other than a NULL pointer), or None."""
    if n_egm_gpus > CAP:
        return "n_egm_gpus above the cap"
    if sum(int(x) for x in n_members) != len(recs) or len(want) != len(recs):
        return "member counts do not add up"
    if sum(int(x) for x in n_ids) != len(ids):
        return "ID counts do not add up"
    if len(egm_off):
        if int(egm_off[0]) != 0:
            return "egm_off[0] is not 0"
        if any(int(b) < int(a) for a, b in zip(egm_off[:-1], egm_off[1:])):
            return "decreasing offsets"
        if any(int(g) >= n_egm_gpus for g in egm_gpu[:int(egm_off[-1])]):
            return "an egm_gpu value not below n_egm_gpus"
    return None


def contract(recs, want, n_members, ids, n_ids, egm_off, egm_gpu, n_egm_gpus):
    """kvg_pci_allocate_check on the CPU: (first_bad, take) as Context.pci_allocate_check returns them.  first_bad[r]
    is the smallest failing position within request r (GC.passes is the re-check), or n_members[r]; take[r, e] is
    True iff every handle device e lists is among request r's IDs (an empty list is taken)."""
    why = refusal(recs, want, n_members, ids, n_ids, egm_off, egm_gpu, n_egm_gpus)
    if why:
        raise ValueError(why)
    ok = GC.passes(recs, want)
    n_egm = max(len(egm_off) - 1, 0)
    lists = [[int(g) for g in egm_gpu[int(egm_off[e]):int(egm_off[e + 1])]] for e in range(n_egm)]
    first_bad = np.zeros(len(n_members), dtype=np.uint32)
    take = np.zeros((len(n_members), n_egm), dtype=bool)
    at = id_at = 0
    for r, (m, k) in enumerate(zip(n_members, n_ids)):
        m, k = int(m), int(k)
        bad = np.flatnonzero(~ok[at:at + m])
        first_bad[r] = bad[0] if len(bad) else m
        held = {int(x) for x in ids[id_at:id_at + k]}
        for e, gpus in enumerate(lists):
            take[r, e] = all(g in held for g in gpus)
        at += m
        id_at += k
    return first_bad, take


def make_call(recs, want, n_members, ids, n_ids, egm_lists, n_egm_gpus=None) -> dict:
    """A call from per-device lists of handles (n_egm_gpus: the largest handle + 1 unless given)."""
    egm_off = np.cumsum([0] + [len(g) for g in egm_lists]).astype(np.uint32) if egm_lists else np.zeros(0, np.uint32)
    egm_gpu = np.array([g for gpus in egm_lists for g in gpus], dtype=np.uint32)
    if n_egm_gpus is None:
        n_egm_gpus = int(egm_gpu.max()) + 1 if len(egm_gpu) else 0
    return dict(recs=recs, want=np.asarray(want, dtype=np.uint32), n_members=[int(x) for x in n_members],
                ids=np.asarray(ids, dtype=np.uint32), n_ids=[int(x) for x in n_ids], egm_off=egm_off, egm_gpu=egm_gpu,
                n_egm_gpus=int(n_egm_gpus))


def records(n_members, rng, p_fail=0.3):
    """The members of every request: noisy passing records, and in about p_fail of the requests a few failures."""
    total = int(sum(n_members))
    recs, want = GC.noise(total, rng)
    at = 0
    for m in n_members:
        if m and rng.random() < p_fail:
            for i in rng.integers(0, m, int(rng.integers(1, 4))):
                GC.apply(recs, want, at + int(i), GC.FAILING[int(rng.integers(0, len(GC.FAILING)))])
        at += m
    return recs, want


def random_call(rng, n_reqs, max_members=40, n_egm=None, max_gpus=8) -> dict:
    """n_reqs requests of 0..max_members members; n_egm EGM devices of 0..max_gpus GPUs each, drawn from a pool of
    handles; each request's IDs are mostly pool handles (so that some devices are taken), with duplicates and IDs that
    no device lists (values >= n_egm_gpus, up to 2**32 - 1)."""
    n_members = [int(rng.integers(0, max_members + 1)) for _ in range(n_reqs)]
    recs, want = records(n_members, rng)
    if n_egm is None:
        n_egm = int(rng.integers(0, 9))
    pool = int(rng.integers(1, 24))
    egm_lists = [[int(g) for g in rng.integers(0, pool, int(rng.integers(0, max_gpus + 1)))] for _ in range(n_egm)]
    n_egm_gpus = pool + int(rng.integers(0, 3))          # handles nobody lists are allowed
    ids, n_ids = [], []
    for _ in range(n_reqs):
        k = int(rng.integers(0, 12))
        mine = []
        if egm_lists and rng.random() < 0.6:               # hold every GPU of one device, and more
            mine += egm_lists[int(rng.integers(0, n_egm))]
        mine += [int(g) for g in rng.integers(0, pool, k)]
        mine += [n_egm_gpus + int(x) for x in rng.integers(0, 5, int(rng.integers(0, 3)))]
        if rng.random() < 0.2:
            mine.append(0xFFFFFFFF)
        rng.shuffle(mine)
        ids += mine
        n_ids.append(len(mine))
    return make_call(recs, want, n_members, ids, n_ids, egm_lists, n_egm_gpus)


def named_calls() -> dict:
    """Quirks of the EGM match, each with one passing and one failing request so that first_bad is exercised too."""
    rng = np.random.default_rng(99)
    recs, want = records([3, 2], rng, p_fail=0)
    GC.apply(recs, want, 4, GC.FAILING[0])

    def call(egm_lists, ids_a, ids_b, n_egm_gpus=None):
        return make_call(recs, want, [3, 2], list(ids_a) + list(ids_b), [len(ids_a), len(ids_b)], egm_lists,
                         n_egm_gpus)
    return {
        "no EGM device": call([], [1, 2], []),
        "empty EGM lists are taken": call([[], [0], []], [], [0]),
        "a GPU listed twice": call([[0, 0, 1], [1, 1]], [0, 1], [1]),
        "an ID that is not an EGM GPU": call([[0, 1]], [0, 2, 7], [0, 1, 2]),
        "duplicate IDs": call([[0, 1], [2]], [0, 0, 0], [1, 1, 0, 0, 2, 2]),
        "no IDs": call([[0], [1]], [], []),
        "handles nobody lists": call([[0]], [5, 0], [3], n_egm_gpus=6),
        "n_egm_gpus at the cap": call([[CAP - 1, 0], [CAP - 1], [31, 32, 4095]],
                                      [CAP - 1, 0], [CAP - 1, 31, 32, 4095], n_egm_gpus=CAP),
        "the largest handle at the cap": call([[CAP - 1]], [CAP], [CAP - 1, 0xFFFFFFFF], n_egm_gpus=CAP),
        "empty requests": make_call(recs[:0], [], [0, 0, 0], [], [0, 0, 0], [[], [0]], 1),
    }


def refused_calls() -> dict:
    """Calls the header refuses (other than a NULL pointer), each one change away from an accepted call."""
    rng = np.random.default_rng(98)
    base = random_call(rng, 3, n_egm=3, max_gpus=3)
    base["egm_gpu"] = np.array([0, 1, 2, 0], dtype=np.uint32)
    base["egm_off"] = np.array([0, 2, 3, 4], dtype=np.uint32)
    base["n_egm_gpus"] = 3
    assert refusal(**base) is None

    def but(**change):
        c = dict(base)
        c.update(change)
        return c
    n_m, n_i = base["n_members"], base["n_ids"]
    return {
        "accepted": base,
        "member counts above n_recs": but(n_members=[n_m[0] + 1] + n_m[1:]),
        "member counts below n_recs": but(recs=np.concatenate([base["recs"], base["recs"][:1]]),
                                          want=np.append(base["want"], np.uint32(0))),
        "ID counts above n_ids": but(n_ids=[n_i[0] + 1] + n_i[1:]),
        "ID counts below n_ids": but(ids=np.append(base["ids"], np.uint32(0))),
        "egm_off[0] is not 0": but(egm_off=np.array([1, 2, 3, 4], dtype=np.uint32)),
        "decreasing offsets": but(egm_off=np.array([0, 3, 2, 4], dtype=np.uint32)),
        "an egm_gpu value at n_egm_gpus": but(egm_gpu=np.array([0, 1, 3, 0], dtype=np.uint32)),
        "n_egm_gpus above the cap": but(n_egm_gpus=CAP + 1),
    }
