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

    python tools/time_health_mdev.py [--sizes 10000,32768,65536] [--group-sizes 10000,32768,65536]
                                     [--pci-sizes 10000,65536] [--ticks 10000] [--out DIR]
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


def poll_loop(call, mutate, ticks, check=None, check_all=False):
    """1 kHz loop: mutate the pinned snapshot, time one call; -> latencies in us of the timed ticks.  `check` runs on
    the warm-up ticks, or on every tick with check_all (outside the timed span, before the wait for the next tick)."""
    lat = []
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
        t_next += PERIOD
        while time.perf_counter() < t_next:
            pass
    lat = np.array(lat) * 1e6
    return {"p50_us": float(np.percentile(lat, 50)), "p99_us": float(np.percentile(lat, 99)), "max_us": float(lat.max())}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,32768,65536")
    ap.add_argument("--group-sizes", default="10000,32768,65536")
    ap.add_argument("--pci-sizes", default="10000,65536")
    ap.add_argument("--ticks", type=int, default=10_000)
    ap.add_argument("--out", default="health_mdev_out", help="directory for health_mdev.json")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    print(card, flush=True)
    ids = O.nv_ids(util.pciids_text())
    out = {"card": card, "poll_hz": 1000, "ticks": a.ticks, "warmup": WARMUP, "flips_per_tick": 10,
           "xid_every": 100, "what": "host wall time from snapshot-in-pinned-buffer to transitions on the host",
           "mdev": {}, "groups": {}, "pci": {}}
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
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "health_mdev.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
