"""Latency of the passthrough health re-scan from raw reads (kvg_health_rescan_groups_raw) at the BASELINE.json
config-5 shape: 10,000 devices, 4 functions per IOMMU group, every group with a VFIO node, in a 1 kHz poll loop.

Three legs in one process, the first two with 50 warm-up ticks and --ticks timed ones:
  raw     Context.health_rescan_groups_raw on pre-read inputs (the raw reads and the node listing already in memory)
  keyed   Context.health_rescan_groups_keyed on the decoded records of the same reads (group handles interned once)
  tick    a whole tick: plugin.read_pci_ids_raw over a tmp sysfs tree, plugin.list_nodes_raw over a tmp VFIO
          directory, then the raw call (4 warm-up ticks and --tick-ticks timed ones: the reads dominate)
Every tick makes one node vanish or return (alternating), so each call lists a group's transitions.  The warm-up
ticks of the raw leg are checked against the keyed leg.  The card's name, power limit and maximum SM clock are read
with a read-only nvidia-smi query in the same run.

    python tools/time_health_raw.py [--n 10000] [--ticks 2000] [--tick-ticks 20] [--out DIR]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kvgpu  # noqa: E402
import util  # noqa: E402

WARMUP = 50
PERIOD = 1e-3


def stats(lat):
    lat = np.array(lat) * 1e6
    return {"p50_us": float(np.percentile(lat, 50)), "p99_us": float(np.percentile(lat, 99)), "max_us": float(lat.max())}


def loop(call, ticks, warmup=WARMUP):
    lat = []
    t_next = time.perf_counter()
    for tick in range(ticks + warmup):
        t0 = time.perf_counter()
        call(tick)
        dt = time.perf_counter() - t0
        if tick >= warmup:
            lat.append(dt)
        t_next += PERIOD
        time.sleep(max(0.0, t_next - time.perf_counter()))
    return stats(lat)


def note(what, t0):
    print("[%.1f s] %s" % (time.perf_counter() - t0, what), flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000)
    ap.add_argument("--ticks", type=int, default=2000)
    ap.add_argument("--tick-ticks", type=int, default=20, help="timed ticks of the whole-tick leg (sysfs reads)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    t0 = time.perf_counter()
    n, n_groups = a.n, (a.n + 3) // 4
    names = [kvgpu.format_bdf(((k // 8) << 8) | (k % 8)) for k in range(n)]   # 8 functions per bus, ascending
    group = {nm: "%d" % (k // 4) for k, nm in enumerate(names)}
    tmp = tempfile.mkdtemp(prefix="kvg")
    out = {"n": n, "groups": n_groups, "ticks": a.ticks, "card": card()}
    note("card: %s" % out["card"], t0)
    try:
        base = util.make_pci_tree(os.path.join(tmp, "sys"), {
            nm: dict(vendor="10de", device="2330", driver="vfio-pci", iommu_group=g, numa_node="0\n")
            for nm, g in group.items()})
        devdir = os.path.join(tmp, "vfio")
        os.makedirs(devdir)
        for g in range(n_groups):
            open(os.path.join(devdir, "%d" % g), "w").close()
        note("trees built", t0)
        raw = kvgpu.read_pci_ids_raw(base, names)
        all_nodes = kvgpu.list_nodes_raw(devdir)
        with kvgpu.Context(0) as ctx:
            intern = {}
            snap = kvgpu.snapshot_pci_ids(base, names, intern)
            recs = snap.recs
            handles = np.array(sorted(intern[x.decode()] for x in all_nodes), dtype=np.uint32)
            gone = os.fsencode("%d" % (n_groups // 2))
            nodes_without = [x for x in all_nodes if x != gone]
            h_without = np.array([h for h in handles if h != intern[gone.decode()]], dtype=np.uint32)

            def raw_call(t):
                return ctx.health_rescan_groups_raw(raw, all_nodes if t % 2 else nodes_without)

            def keyed_call(t):
                return ctx.health_rescan_groups_keyed(recs, handles if t % 2 else h_without)

            for t in range(WARMUP):    # the raw call against the keyed call on the decoded records
                d, e = raw_call(t), keyed_call(t)
                assert d.n_alive == e.n_alive and np.array_equal(d.changed, e.changed), t
                assert t == 0 or len(d.changed) == 4
            note("warm-up checked against the keyed call", t0)
            out["raw_call"] = loop(raw_call, a.ticks)
            note("raw leg %s" % out["raw_call"], t0)
            out["keyed_call"] = loop(keyed_call, a.ticks)
            note("keyed leg %s" % out["keyed_call"], t0)
            node = os.path.join(devdir, gone.decode())

            def whole_tick(t):
                if t % 2:
                    open(node, "w").close()
                elif os.path.exists(node):
                    os.remove(node)
                d = ctx.health_rescan_groups_raw(kvgpu.read_pci_ids_raw(base, names), kvgpu.list_nodes_raw(devdir))
                assert t < 2 or len(d.changed) == 4
            out["whole_tick"] = loop(whole_tick, a.tick_ticks, warmup=4)
            note("whole-tick leg %s" % out["whole_tick"], t0)
            before = ctx.launch_count
            raw_call(0)
            out["launches_per_call"] = ctx.launch_count - before
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_health_raw.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
