#!/usr/bin/env python3
"""Host wall time of kvg_scan_mdev_raw (raw sysfs text in, GPU decode + scan) against the host snapshot (the decode of
the same reads into records and a type dictionary, as snapshot_mdev_tree does after its reads) plus kvg_scan_mdev, and
the decode kernel's event time.  Inputs: oracle gen_mdev records with its 256 type names, rendered as the sysfs text a
walk would read, at 8, 1,000, 65,536 (BASELINE.json config 3) and 1,000,000 entries.  The card's name and power limit
are read in the same run.   python tools/time_scan_mdev_raw.py [reps]   -> one JSON line per size"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"), os.path.join(ROOT, "tests")]
import kvgpu  # noqa: E402
from kvgpu import _lib as L  # noqa: E402
from oracle import oracle as O  # noqa: E402
import mdev_raw_cases as MC  # noqa: E402

HOST_PACK_MAX = 65_536   # the Python host snapshot is timed up to here; above it the packed records are given


def host_snapshot(raw):
    """the host's part of the packed path on the same bytes: UUIDs, the type dictionary, parents, numa_node"""
    n, F = len(raw.state), L.MRAW_FIELDS
    b, off = raw.bytes, raw.off
    recs = np.zeros(n, dtype=L.MDEV_REC)
    types = {}
    for i in range(n):
        g = lambda f: b[off[F * i + f]:off[F * i + f + 1]]
        st = int(raw.state[i])
        recs[i]["uuid"] = np.frombuffer(bytes.fromhex(g(0).replace(b"-", b"").decode()), dtype=np.uint8)
        if st & (1 << (8 + L.MRAW_TYPE)):
            recs[i]["flags"] = L.MF_TYPE_ERR
            continue
        recs[i]["type_idx"] = types.setdefault(g(1), len(types))
        if st & (1 << (8 + L.MRAW_LINK)):
            recs[i]["flags"] = L.MF_PARENT_ERR
            continue
        recs[i]["parent"] = kvgpu.parse_bdf(g(2).split(b"/")[-2].strip(b"\n").decode())
        if st & (1 << (8 + L.MRAW_NUMA)):
            recs[i]["flags"] = L.MF_NUMA_ERR
        else:
            recs[i]["parent_numa"] = int(g(3).strip())
    return recs, list(types)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    import gzip
    text = gzip.decompress(open(os.path.join(ROOT, "tests", "golden", "pci.ids.gz"), "rb").read())
    type_names = O.gen_type_names(256)
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(text)
        for n in (8, 1000, 65_536, 1_000_000):
            recs = O.gen_mdev(0, n)
            raw = MC.render_records(recs, type_names)
            _, snap = ctx.scan_mdev_raw(raw)
            ctx.scan_mdev(snap.recs, snap.raw_types)
            t_raw, t_pack = [], []
            for _ in range(reps):
                t0 = time.perf_counter()
                ctx.scan_mdev_raw(raw)
                t_raw.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                ctx.scan_mdev(*(host_snapshot(raw) if n <= HOST_PACK_MAX else (snap.recs, snap.raw_types)))
                t_pack.append(time.perf_counter() - t0)
            ctx.set_kernel_timing(True)
            ctx.scan_mdev_raw(raw)
            times = ctx.kernel_times()
            ctx.set_kernel_timing(False)
            dec = sum(ms for name, ms in times if name == "mraw_decode")
            print(json.dumps({"card": card, "entries": n, "raw_bytes": len(raw.bytes),
                              "scan_mdev_raw_ms_median": 1e3 * float(np.median(t_raw)),
                              "snapshot_plus_scan_mdev_ms_median": 1e3 * float(np.median(t_pack)),
                              "host_snapshot_timed": n <= HOST_PACK_MAX, "decode_kernel_ms": dec,
                              "kernels": sorted({name for name, _ in times})}), flush=True)


if __name__ == "__main__":
    main()
