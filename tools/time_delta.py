"""Timing of the re-scan delta (kvg_scan_pci_delta) against the plain scan (kvg_scan_pci) on one GPU.

A sequence of snapshots changes about 0.1 % of the records per step (regroups, NUMA moves, re-binds, hot-removes and
hot-adds in turn).  For each size both entry points walk the same sequence, alternating in rounds; the host wall
time of each C call (it returns with its result on the host) is recorded.  A separate pass with kernel timing on
reports the device time of the delta kernels.  The card name and power limit are read in the same run.

    python tools/time_delta.py [--sizes 10000,1000000] [--steps 200] [--out results.json]
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
import kvgpu  # noqa: E402
from kvgpu import _lib as L  # noqa: E402
from oracle import oracle as O  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests"))
import util  # noqa: E402


def snapshots(n, ids, steps, seed=1):
    rng = np.random.default_rng(seed)
    recs = O.gen_pci(seed, n, ids, 16)
    recs["addr"] = np.arange(n, dtype=np.uint32) * 4
    out = [recs]
    for s in range(steps):
        r = out[-1].copy()
        k = max(1, n // 1000)
        pick = rng.choice(np.nonzero(util.pci_alive(r))[0], k, replace=False)
        kind = s % 5
        if kind == 0:
            r["iommu_group"][pick] = rng.integers(0, 1 << 20, k)
        elif kind == 1:
            r["numa"][pick] = (r["numa"][pick] + 1) % 4
        elif kind == 2:
            r["driver"][pick] = 3
        elif kind == 3:
            r = np.delete(r, pick)
        else:
            add = r[pick].copy()
            add["addr"] += 1 + rng.integers(0, 3, k).astype(np.uint32)
            add = add[~np.isin(add["addr"], r["addr"])]
            r = np.sort(np.concatenate([r, add]), order="addr", kind="stable")
        out.append(np.ascontiguousarray(r))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,1000000")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", help="also write the JSON result to this file")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    text = util.pciids_text()
    ids = O.nv_ids(text)
    ctx = kvgpu.Context(0)
    ctx.pciids_load(text)
    lib, h = ctx._lib, ctx.handle
    out = {"card": card[0] if card else "unknown", "steps": a.steps, "sizes": {}}
    for n in [int(x) for x in a.sizes.split(",")]:
        seq = snapshots(n, ids, a.steps)
        res, dl = C.POINTER(L.PciResultC)(), C.POINTER(L.PciDeltaC)()

        def plain(r):
            t0 = time.perf_counter()
            rc = lib.kvg_scan_pci(h, r.ctypes.data, len(r), C.byref(res))
            t1 = time.perf_counter()
            assert rc == 0
            lib.kvg_result_free(res)
            return t1 - t0

        def delta(r):
            t0 = time.perf_counter()
            rc = lib.kvg_scan_pci_delta(h, r.ctypes.data, len(r), C.byref(res), C.byref(dl))
            t1 = time.perf_counter()
            assert rc == 0
            n_changes = int(dl.contents.n_changes)
            lib.kvg_result_free(res)
            lib.kvg_result_free(dl)
            return t1 - t0, n_changes

        for r in seq[:10]:                       # warm-up: buffers, pinned blocks, radix hints
            plain(r)
            delta(r)
        ctx.scan_pci_delta_reset()
        delta(seq[0])
        tp, td, changes = [], [], []
        for i in range(1, len(seq), 10):         # rounds of ten steps, alternating the two entry points
            chunk = seq[i:i + 10]
            tp += [plain(r) for r in chunk]      # leaves the retained previous result (seq[i - 1]) alone
            for r in chunk:
                t, c = delta(r)
                td.append(t)
                changes.append(c)
        ctx.set_kernel_timing(True)
        per = {}
        for r in seq[:20]:
            delta(r)
            for name, t in ctx.kernel_times():
                if name.startswith("delta_"):
                    per.setdefault(name, []).append(t * 1e3)
        ctx.set_kernel_timing(False)
        q = lambda v, p: round(float(np.percentile(np.array(v) * 1e6, p)), 1)
        out["sizes"][n] = {
            "scan_pci_us": {"p50": q(tp, 50), "p90": q(tp, 90)},
            "scan_pci_delta_us": {"p50": q(td, 50), "p90": q(td, 90)},
            "changes_per_step_median": int(np.median(changes)),
            "kernel_us_median": {k: round(float(np.median(v)), 2) for k, v in per.items()},
        }
        print(n, json.dumps(out["sizes"][n]), flush=True)
    ctx.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
