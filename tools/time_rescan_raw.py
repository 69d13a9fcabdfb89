#!/usr/bin/env python3
"""Host wall time per call of kvg_scan_pci_raw_delta / kvg_scan_mdev_raw_delta against kvg_scan_*_raw and against
kvg_scan_*_delta on the decoded records (event timing off), then, in a separate pass, the event time of the re-key
kernels (raw_rekey, raw_xlate) and of K7 inside the raw delta.  Inputs: sequences of raw snapshots with about 0.1 % of
the entries changed per step, at 10,000 and 1,000,000 entries, fully numeric and with every column in index mode
(PCI: gen_pci records, one device id in upper case, one group written "042", a non-BDF name; mdev: one parent that is
no BDF, a name that is no UUID).  The card's name and power limit are read in the same run.
    python tools/time_rescan_raw.py [steps]   -> one JSON line per size and mode"""
import json
import os
import subprocess
import sys
import time
import gzip

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"), os.path.join(ROOT, "tools")]
import kvgpu  # noqa: E402
from kvgpu import _lib as L  # noqa: E402
from oracle import oracle as O  # noqa: E402
from time_scan_raw import render  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import mdev_raw_cases as MC  # noqa: E402


def index_mode(raw: kvgpu.PciRaw, i: int) -> kvgpu.PciRaw:
    """entry i (one whose group and device reads are reached) with its device id in upper case and its group link
    written with a leading zero, and one dropped entry named "zz" at the end: every column in index mode"""
    b, off = bytearray(raw.bytes), raw.off.astype(np.int64)
    d0, d1 = int(off[6 * i + 5]), int(off[6 * i + 6])   # field KVG_RAW_DEVICE, "0x%04x\n"
    b[d0:d1] = bytes(b[d0:d1]).upper().replace(b"0X", b"0x")
    g0, g1 = int(off[6 * i + 3]), int(off[6 * i + 4])   # field KVG_RAW_GROUP
    b[g0:g1] = b"../042"
    off[6 * i + 4:] += 6 - (g1 - g0)
    tail = [b"zz", b"", b"", b"", b"", b""]
    off = np.concatenate([off, off[-1] + np.cumsum([len(t) for t in tail])])
    state = np.concatenate([raw.state, np.array([0x3E | 0x200], np.uint16)])   # its vendor read failed: dropped
    return kvgpu.PciRaw(list(raw.names) + ["zz"], off.astype(np.uint32), bytes(b) + b"".join(tail), state)


def pci_steps(n, steps, ids, rng):
    """numeric and index-mode raw snapshots of gen_pci records, about 0.1 % changed per step"""
    recs = [O.gen_pci(0, n, ids, 16)]
    for _ in range(steps):
        nxt = recs[-1].copy()
        m = max(2, n // 1000)
        sel = rng.choice(len(nxt), m, replace=False)
        nxt["numa"][sel[: m // 2]] ^= 1
        nxt["iommu_group"][sel[m // 2:]] += 1
        recs.append(np.delete(nxt, rng.choice(len(nxt), max(1, m // 4), replace=False)))
    raws = [render(r) for r in recs]
    reached = lambda r: np.flatnonzero((r["vendor"] == 0x10DE) & np.isin(r["driver"], (1, 2)) &
                                       ((r["flags"] & (L.PF_IOMMU_ERR | L.PF_DEVICE_ERR)) == 0))[0]
    return {"numeric": raws, "index": [index_mode(w, int(reached(r))) for w, r in zip(raws, recs)]}


def mdev_steps(n, steps, rng):
    """numeric and index-mode raw mdev snapshots (a parent that is no BDF, a name that is no UUID), about 0.1 % of the
    entries retyped, moved or destroyed per step"""
    types = [b"GRID T4-%dQ\n" % k for k in range(16)]
    ent = [(nm, {"type": types[rng.integers(16)], "link": MC.link_to(kvgpu.format_bdf(int(rng.integers(256)) << 8)
                                                                     .encode(), nm), "numa_node": b"0\n"})
           for nm in MC.canonical_names(rng, n)]
    seq = [ent]
    for _ in range(steps):
        nxt = [(nm, dict(e)) for nm, e in seq[-1]]
        m = max(2, n // 1000)
        for k in rng.choice(len(nxt), m, replace=False)[: m // 2]:
            nxt[k][1]["type"] = types[rng.integers(16)]
        for k in rng.choice(len(nxt), m, replace=False)[: m // 2]:
            nxt[k][1]["link"] = MC.link_to(kvgpu.format_bdf(int(rng.integers(256)) << 8).encode(), nxt[k][0])
        drop = set(rng.choice(len(nxt), max(1, m // 4), replace=False).tolist())
        seq.append([x for k, x in enumerate(nxt) if k not in drop])

    def index(e):
        e = [(nm, dict(x)) for nm, x in e]
        e[0][1]["link"] = MC.link_to(b"gpu-a", e[0][0])
        return e + [(b"zz", {"type": types[0], "link": MC.link_to(b"0000:01:00.0", b"zz"), "numa_node": b"0\n"})]
    return {"numeric": [MC.raw_of(e) for e in seq], "index": [MC.raw_of(index(e)) for e in seq]}


KERNELS = ("raw_rekey", "raw_xlate", "delta_merge", "delta_lists", "mdev_delta_types", "mdev_delta_merge",
           "mdev_delta_lists")


def measure(kind, rs, text):
    """pass 1: host wall time per call of the raw delta, the raw scan and the plain delta on the decoded records, event
    timing off; pass 2, on a fresh context over the same sequence: the event times of the delta's kernels"""
    raw_delta = "scan_%s_raw_delta" % kind
    t = {"raw_delta": [], "raw": [], "delta": []}
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(text)

        def plain(snap):
            return ctx.scan_pci_delta(snap.recs) if kind == "pci" else ctx.scan_mdev_delta(snap.recs, snap.raw_types)
        getattr(ctx, raw_delta)(rs[0])
        plain(getattr(ctx, "scan_%s_raw" % kind)(rs[0])[1])
        for r in rs[1:]:
            t0 = time.perf_counter()
            _, snap = getattr(ctx, "scan_%s_raw" % kind)(r)
            t1 = time.perf_counter()
            _, _, d = getattr(ctx, raw_delta)(r)
            t2 = time.perf_counter()
            plain(snap)
            t3 = time.perf_counter()
            t["raw"].append(t1 - t0)
            t["raw_delta"].append(t2 - t1)
            t["delta"].append(t3 - t2)
    dev = {}
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(text)
        getattr(ctx, raw_delta)(rs[0])
        for r in rs[1:]:
            ctx.set_kernel_timing(True)
            getattr(ctx, raw_delta)(r)
            for name, ms in ctx.kernel_times():
                if name in KERNELS:
                    dev.setdefault(name, []).append(ms * 1e3)
            ctx.set_kernel_timing(False)
    return t, dev, snap, d


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    text = gzip.open(os.path.join(ROOT, "tests", "golden", "pci.ids.gz"), "rb").read()
    ids = O.nv_ids(text)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    for kind in ("pci", "mdev"):
        for n in (10_000, 1_000_000):
            rng = np.random.default_rng(n)
            seqs = pci_steps(n, steps, ids, rng) if kind == "pci" else mdev_steps(n, steps, rng)
            for mode, rs in seqs.items():
                t, dev, snap, d = measure(kind, rs, text)
                print(json.dumps({
                    "kind": kind, "entries": n, "mode": mode, "steps": len(rs) - 1, "changes_last": int(len(d.changes)),
                    "host_ms_median": {k: round(float(np.median(v)) * 1e3, 3) for k, v in t.items()},
                    "host_ms_min": {k: round(float(np.min(v)) * 1e3, 3) for k, v in t.items()},
                    "host_ms_max": {k: round(float(np.max(v)) * 1e3, 3) for k, v in t.items()},
                    "device_us_median": {k: round(float(np.median(v)), 1) for k, v in dev.items()},
                    "card": card}), flush=True)


if __name__ == "__main__":
    main()
