#!/usr/bin/env python3
"""Per-call host wall time and kernel event times of kvg_pci_allocate_response with iommufd on, next to
kvg_pci_allocate_raw on the same reads, at the four sizes of DESIGN §4.11.2: 1 x 8 members with 4 EGM entries,
16 x 8, 1,000 x 24, and one request of 100,000 members with 4,096 EGM entries; 1-8 vfio-dev entries per member.
Prints the card, its power limit and its maximum SM clock from the same run.  The timings are on inputs already
packed into arrays; the host's listing, reading and formatting are not in them.

    python tools/time_allocate_response.py [--reps 20]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"))
import kvgpu  # noqa: E402
from kvgpu import _lib as L  # noqa: E402

VENDOR = b"0x10de\n"


def call_of(n_reqs, n_members, n_egm, rng):
    """requests of groups of 8 members, each DevicesID the group's first member; EGM entries over those IDs"""
    reqs, firsts = [], []
    for r in range(n_reqs):
        visits = []
        for v in range(max(n_members // 8, 1)):
            g = b"%d" % (r * 20_000 + v)
            visit = []
            for k in range(min(8, n_members)):
                addr = b"%04x:%02x:%02x.%x" % (r, v >> 8, v & 255, k)
                listing = [(b"vfio%d" % x, bool(x % 3)) for x in rng.integers(0, 64, size=int(rng.integers(0, 8)))]
                visit.append((addr, b"../" + g, VENDOR, g, listing + [(b"vfio%d" % (1000 + k), True)]))
            visits.append(visit)
            firsts.append(visit[0][0])
        reqs.append(([v[0][0] for v in visits], visits, False))
    egm = [(b"egm%05d" % e, firsts[(2 * e) % len(firsts)] + b" " + firsts[(2 * e + 1) % len(firsts)] + b"\n", True)
           for e in range(n_egm)]
    return reqs, egm


def timed(ctx, fn, reps):
    """median host wall time of `reps` calls (kernel timing off), then the kernel event times of one more call"""
    fn()
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        wall.append((time.perf_counter() - t0) * 1e3)
    ctx.set_kernel_timing(True)
    fn()
    kern = ctx.kernel_times()
    ctx.set_kernel_timing(False)
    return float(np.median(wall)), ", ".join("%s %.1f us" % (n, 1e3 * ms) for n, ms in kern)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card, power limit, max SM clock: %s" % q)
    rng = np.random.default_rng(1)
    with kvgpu.Context(0) as ctx:
        for n_reqs, n_members, n_egm in ((1, 8, 4), (16, 8, 4), (1000, 24, 4), (1, 100_000, 4096)):
            reqs, egm = call_of(n_reqs, n_members, n_egm, rng)
            raw, resp = kvgpu.pack_alloc_response(reqs, egm, True)
            out = ctx.pci_allocate_response(raw, resp)
            assert all(r[0] == L.ARESP_OK for r in out)
            resp_w, resp_k = timed(ctx, lambda: ctx.pci_allocate_response(raw, resp), args.reps)
            raw_w, raw_k = timed(ctx, lambda: ctx.pci_allocate_raw(raw), args.reps)
            print("%5d x %6d members, %4d EGM: response call %.3f ms (%s) | raw call %.3f ms (%s)"
                  % (n_reqs, n_members, n_egm, resp_w, resp_k, raw_w, raw_k))


if __name__ == "__main__":
    main()
