"""Latency of the vGPU health re-scan (kvg_health_rescan_mdev) and of the passthrough health re-scan by IOMMU group
(kvg_health_rescan_groups) in a 1 kHz poll loop, beside the PCI health re-scan (kvg_health_rescan; --pci-sizes, by
default 10,000 records as in BASELINE.json config 5 and 65,536, which runs the look-back form) in the same process.

The group leg (--group-sizes) puts 4 functions in each group, gives every group up to the 4,096-handle cap a node,
flips the driver of 10 records per tick, makes one node vanish every 100 ticks and brings it back 50 ticks later,
and checks every tick against the numpy state machine of tests/health_groups_ref.py (outside the timed span).  Up to
32,768 records it runs k_health_small<GroupHealthRule>, at 65,536 k_compact<HealthOp<GroupHealthRule>, 256, 8>.

Each tick flips the type / parent read-error bits of 10 records of a pinned snapshot, and every 100th tick carries one
XID parent handle.  The host wall time of each call is recorded from "snapshot in the pinned buffer" to "transitions on
the host" (the call returns with them); 50 warm-up ticks, whose results are also checked against the numpy state
machine of tests/health_mdev_ref.py, precede the timed ones.  Sizes up to 32,768 records run the one-CTA
k_health_small<MdevHealthRule>; 65,536 (the config-3 vGPU count) runs k_compact<HealthOp<MdevHealthRule>, 256, 8>.
The PCI leg flips the driver of 10 records per tick and checks its warm-up ticks against numpy.  The card's
name, power limit and maximum SM clock are read with a read-only nvidia-smi query in the same run.

--keyed adds the keyed legs (kvg_health_rescan_mdev_keyed / _groups_keyed) in the same process: the same event
patterns plus one key inserted near the front every 100 ticks, every tick checked; the ticks with an edit are also
reported on their own.

    python tools/time_health_mdev.py [--sizes 10000,32768,65536] [--group-sizes 10000,32768,65536]
                                     [--pci-sizes 10000,65536] [--ticks 10000] [--keyed] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kvgpu  # noqa: E402
from oracle import oracle as O  # noqa: E402
import health_groups_ref  # noqa: E402
import health_mdev_ref  # noqa: E402
import util  # noqa: E402

WARMUP = 50
PERIOD = 1e-3
N_TYPES = 256
GROUP_CAP = 4096   # KVG_HEALTH_MAX_GROUPS


def pinned(n, itemsize):
    import torch
    t = torch.empty(n * itemsize, dtype=torch.uint8, pin_memory=True)
    return t, t.data_ptr()


def stats(lat):
    lat = np.array(lat) * 1e6
    return {"p50_us": float(np.percentile(lat, 50)), "p99_us": float(np.percentile(lat, 99)), "max_us": float(lat.max())}


def poll_loop(call, mutate, ticks, check=None, check_all=False, edit=None):
    """1 kHz loop: mutate the pinned snapshot, time one call; -> latencies in us of the timed ticks.  `check` runs on
    the warm-up ticks, or on every tick with check_all (outside the timed span, before the wait for the next tick).
    edit(tick) -> True marks the ticks whose list changed; they are also reported on their own ("edit")."""
    lat, lat_edit = [], []
    t_next = time.perf_counter()
    for tick in range(ticks + WARMUP):
        xids = mutate(tick)
        t0 = time.perf_counter()                        # the snapshot is in the pinned buffer
        res = call(xids)
        dt = time.perf_counter() - t0                   # the transitions are on the host
        if (tick < WARMUP or check_all) and check is not None:
            check(res, xids)
        kvgpu.load().kvg_result_free(res)
        if tick >= WARMUP:
            lat.append(dt)
            if edit is not None and edit(tick):
                lat_edit.append(dt)
        t_next += PERIOD
        while time.perf_counter() < t_next:
            pass
    out = stats(lat)
    if lat_edit:
        out["edit"] = dict(stats(lat_edit), ticks=len(lat_edit))
    return out


def mdev_leg(ctx, n, ticks):
    lib = kvgpu.load()
    buf, ptr = pinned(n, 32)
    view = buf.numpy().view(kvgpu.MDEV_REC)
    view[:] = O.gen_mdev(0, n)
    parents = np.unique(view["parent"])
    rng = np.random.default_rng(n)
    ref = health_mdev_ref.HealthMdevRef()
    lib.kvg_health_mdev_reset(ctx.handle)

    def mutate(tick):
        view["flags"][rng.integers(0, n, 10)] ^= rng.integers(1, 4, 10).astype(np.uint8)
        return [int(parents[rng.integers(0, len(parents))])] if tick % 100 == 99 else []

    def call(xids):
        x = np.array(xids, dtype=np.uint32)
        res = C.POINTER(kvgpu._lib.HealthDeltaC)()
        rc = lib.kvg_health_rescan_mdev(ctx.handle, ptr, n, N_TYPES, x.ctypes.data if len(x) else None, len(x),
                                        C.byref(res))
        assert rc == 0, ctx._lib.kvg_last_error(ctx.handle)
        return res

    def check(res, xids):
        r = res.contents
        got = np.ctypeslib.as_array(C.cast(r.changed, C.POINTER(C.c_uint32)), (r.n_changed,)) if r.n_changed else np.zeros(0, np.uint32)
        want = ref.rescan(view, N_TYPES, xids)
        assert r.n_alive == want.n_alive and np.array_equal(got, want.changed), "parity at %d records" % n

    out = poll_loop(call, mutate, ticks, check)
    out["path"] = "k_health_small<MdevHealthRule>" if n <= 32768 else "k_compact<HealthOp<MdevHealthRule>, 256, 8>"
    return out


def pci_leg(ctx, n, ticks, ids):
    lib = kvgpu.load()
    buf, ptr = pinned(n, 16)
    view = buf.numpy().view(kvgpu.PCI_REC)
    view[:] = O.gen_pci(0, n, ids, 12)
    rng = np.random.default_rng(5)
    prev = [np.zeros(n, dtype=bool)]
    lib.kvg_health_reset(ctx.handle)

    def mutate(tick):
        view["driver"][rng.integers(0, n, 10)] = rng.integers(0, 5, 10)
        return None

    def call(_):
        res = C.POINTER(kvgpu._lib.HealthDeltaC)()
        assert lib.kvg_health_rescan(ctx.handle, ptr, n, C.byref(res)) == 0
        return res

    def check(res, _):
        r = res.contents
        now = util.pci_alive(view)
        idx = np.nonzero(now != prev[0])[0]
        got = np.ctypeslib.as_array(C.cast(r.changed, C.POINTER(C.c_uint32)), (r.n_changed,)) if r.n_changed else np.zeros(0, np.uint32)
        assert r.n_alive == now.sum(), "PCI parity at %d records" % n
        assert np.array_equal(got, (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)), "PCI parity at %d records" % n
        prev[0] = now

    out = poll_loop(call, mutate, ticks, check)
    out["path"] = "k_health_small<PciHealthRule>" if n <= 32768 else "k_compact<HealthOp<PciHealthRule>, 256, 8>"
    return out


def groups_leg(ctx, n, ticks, ids):
    """kvg_health_rescan_groups: 4 functions per IOMMU group; every group up to the 4,096-handle cap has a node (at
    32,768 and 65,536 records the later groups have none, so the set copied per tick is the full 16 KiB).  Every
    100th tick one group's node vanishes, and it returns 50 ticks later.  Every tick is checked."""
    lib = kvgpu.load()
    buf, ptr = pinned(n, 16)
    view = buf.numpy().view(kvgpu.PCI_REC)
    view[:] = O.gen_pci(0, n, ids, 12)
    view["iommu_group"] = 1 + np.arange(n, dtype=np.uint32) // 4
    all_nodes = np.arange(1, min(-(-n // 4), GROUP_CAP) + 1, dtype=np.uint32)
    nodes = [all_nodes]
    rng = np.random.default_rng(n + 7)
    ref = health_groups_ref.HealthGroupsRef()
    lib.kvg_health_groups_reset(ctx.handle)

    def mutate(tick):
        view["driver"][rng.integers(0, n, 10)] = rng.integers(0, 5, 10)
        if tick % 100 == 0:
            g = int(rng.integers(1, len(all_nodes) + 1))
            nodes[0] = np.setdiff1d(all_nodes, [g])
        elif tick % 100 == 50:
            nodes[0] = all_nodes
        return nodes[0]

    def call(g):
        res = C.POINTER(kvgpu._lib.HealthDeltaC)()
        rc = lib.kvg_health_rescan_groups(ctx.handle, ptr, n, g.ctypes.data, len(g), C.byref(res))
        assert rc == 0, ctx._lib.kvg_last_error(ctx.handle)
        return res

    def check(res, g):
        r = res.contents
        got = np.ctypeslib.as_array(C.cast(r.changed, C.POINTER(C.c_uint32)), (r.n_changed,)) if r.n_changed else np.zeros(0, np.uint32)
        want = ref.rescan(view, g)
        assert r.n_alive == want.n_alive and np.array_equal(got, want.changed), "parity at %d records" % n

    out = poll_loop(call, mutate, ticks, check, check_all=True)
    out.update(groups_with_node=len(all_nodes),
               path="k_health_small<GroupHealthRule>" if n <= 32768 else "k_compact<HealthOp<GroupHealthRule>, 256, 8>")
    return out


def keyed_leg(ctx, kind, n, ticks, ids, per_group=4):
    """kvg_health_rescan_mdev_keyed / _groups_keyed on the event pattern of the index-keyed leg of the same kind, plus
    a list edit every 100 ticks: one key inserted near the front (the records after it move down one place, so every
    later record misses its same-position hint on that tick).  Keys are spaced two apart so that there is room.  Every
    tick is checked against the rules of tests/health_mdev_ref.py / health_groups_ref.py with the prior state kept per
    key (a new key starts at 0): the vectorised form of tests/health_keyed_ref.py for a list that only grows."""
    lib = kvgpu.load()
    cap = n + (ticks + WARMUP) // 100 + 1
    mdev = kind == "mdev"
    size = 32 if mdev else 16
    buf, ptr = pinned(cap, size)
    view = buf.numpy().view(kvgpu.MDEV_REC if mdev else kvgpu.PCI_REC)
    if mdev:
        univ = O.gen_mdev(0, 2 * cap)                   # uuid bytes 0..3 = BE32(index): ascending
        parents = np.unique(univ["parent"])
    else:
        univ = O.gen_pci(0, 2 * cap, ids, 12)
        univ["addr"] = np.arange(2 * cap, dtype=np.uint32)
        univ["iommu_group"] = 1 + np.arange(2 * cap, dtype=np.uint32) // (2 * per_group)
        all_nodes = np.arange(1, min(-(-n // per_group), GROUP_CAP) + 1, dtype=np.uint32)
        nodes = [all_nodes]
    m = [n]
    view[:n] = univ[0:2 * n:2]
    st = {"p": np.zeros(n, bool), "m": np.zeros(n, bool), "h": np.zeros(n, bool)}
    rng = np.random.default_rng(n + 11)
    edits = [0]
    if mdev:                                            # n = 0: the reset
        ctx.health_rescan_mdev_keyed(view[:0], N_TYPES)
    else:
        ctx.health_rescan_groups_keyed(view[:0])

    def is_edit(tick):
        return tick % 100 == 77

    def mutate(tick):
        k = m[0]
        if is_edit(tick):                               # key 2e+1 goes behind key 2e, at position 2e+1
            e = edits[0]
            edits[0] += 1
            at = 2 * e + 1
            view[at + 1:k + 1] = view[at:k].copy()
            view[at] = univ[2 * e + 1]
            for a in st:
                st[a] = np.insert(st[a], at, False)
            m[0] = k = k + 1
        idx = rng.integers(0, k, 10)
        if mdev:
            view["flags"][idx] ^= rng.integers(1, 4, 10).astype(np.uint8)
            return [int(parents[rng.integers(0, len(parents))])] if tick % 100 == 99 else []
        view["driver"][idx] = rng.integers(0, 5, 10)
        if tick % 100 == 0:
            nodes[0] = np.setdiff1d(all_nodes, [int(rng.integers(1, len(all_nodes) + 1))])
        elif tick % 100 == 50:
            nodes[0] = all_nodes
        return nodes[0]

    def call(xs):
        x = np.asarray(xs, dtype=np.uint32)
        res = C.POINTER(kvgpu._lib.HealthDeltaC)()
        if mdev:
            rc = lib.kvg_health_rescan_mdev_keyed(ctx.handle, ptr, m[0], N_TYPES, x.ctypes.data if len(x) else None,
                                                  len(x), C.byref(res))
        else:
            rc = lib.kvg_health_rescan_groups_keyed(ctx.handle, ptr, m[0], x.ctypes.data if len(x) else None, len(x),
                                                    C.byref(res))
        assert rc == 0, ctx._lib.kvg_last_error(ctx.handle)
        return res

    def check(res, xs):
        r = res.contents
        got = np.ctypeslib.as_array(C.cast(r.changed, C.POINTER(C.c_uint32)), (r.n_changed,)) if r.n_changed else np.zeros(0, np.uint32)
        if mdev:
            want, alive, st["p"], st["m"] = health_mdev_ref.step(view[:m[0]], N_TYPES, xs, st["p"], st["m"])
        else:
            want, alive, st["h"] = health_groups_ref.step(view[:m[0]], xs, st["h"])
        assert r.n_alive == alive and np.array_equal(got, want), "keyed parity at %d records" % m[0]

    out = poll_loop(call, mutate, ticks, check, check_all=True, edit=is_edit)
    out["path"] = "k_health_small<Keyed<%s>>" % ("MdevHealthRule" if mdev else "GroupHealthRule") if n + ticks // 100 < 32768 \
        else "k_compact<HealthOp<Keyed<%s>>, 256, 8>" % ("MdevHealthRule" if mdev else "GroupHealthRule")
    if not mdev:
        out["groups"] = int(-(-n // per_group))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,32768,65536")
    ap.add_argument("--group-sizes", default="10000,32768,65536")
    ap.add_argument("--pci-sizes", default="10000,65536")
    ap.add_argument("--ticks", type=int, default=10_000)
    ap.add_argument("--keyed", action="store_true", help="also the keyed legs: 10,000 and 65,536 vGPUs; 10,000 PCI "
                    "functions in 2,500 groups and 65,536 in 4,096")
    ap.add_argument("--out", default="health_mdev_out", help="directory for health_mdev.json")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    print(card, flush=True)
    ids = O.nv_ids(util.pciids_text())
    out = {"card": card, "poll_hz": 1000, "ticks": a.ticks, "warmup": WARMUP, "flips_per_tick": 10,
           "xid_every": 100, "what": "host wall time from snapshot-in-pinned-buffer to transitions on the host",
           "mdev": {}, "groups": {}, "pci": {}, "mdev_keyed": {}, "groups_keyed": {}}
    with kvgpu.Context(0) as ctx:
        for n in [int(s) for s in a.sizes.split(",") if s]:
            out["mdev"][n] = mdev_leg(ctx, n, a.ticks)
            print("mdev", n, json.dumps(out["mdev"][n]), flush=True)
        for n in [int(s) for s in a.group_sizes.split(",") if s]:
            out["groups"][n] = groups_leg(ctx, n, a.ticks, ids)
            print("groups", n, json.dumps(out["groups"][n]), flush=True)
        for n in [int(s) for s in a.pci_sizes.split(",") if s]:
            out["pci"][n] = pci_leg(ctx, n, a.ticks, ids)
            print("pci", n, json.dumps(out["pci"][n]), flush=True)
        if a.keyed:
            for n in (10_000, 65_536):
                out["mdev_keyed"][n] = keyed_leg(ctx, "mdev", n, a.ticks, ids)
                print("mdev_keyed", n, json.dumps(out["mdev_keyed"][n]), flush=True)
            for n, per in ((10_000, 4), (65_536, 16)):
                out["groups_keyed"][n] = keyed_leg(ctx, "groups", n, a.ticks, ids, per)
                print("groups_keyed", n, json.dumps(out["groups_keyed"][n]), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "health_mdev.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
