#!/usr/bin/env python3
"""Per-call host wall time and kernel event times of kvg_pci_allocate_raw, next to AllocateCheck's form
(kvg_pci_allocate_check with the group and EGM strings interned on the host), at four sizes:
1 x 8 members with 4 EGM entries, 16 x 8, 1,000 x 24, and one request of 100,000 members with 4,096 EGM entries.
Prints the card, its power limit and its maximum SM clock from the same run.

    python tools/time_allocate_raw.py [--reps 20]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"))
import kvgpu  # noqa: E402
from kvgpu import serve  # noqa: E402

LINK, VENDOR = b"../../../kernel/iommu_groups/%d", b"0x10de\n"


def call_of(n_reqs, n_members, n_egm):
    bdfs = [b"0000:%02x:%02x.%x" % (k >> 8, (k >> 3) & 31, k & 7) for k in range(max(2 * n_egm, 64))]
    reqs = []
    for r in range(n_reqs):
        members = [(LINK % (m // 8), VENDOR, b"%d" % (m // 8)) for m in range(n_members)]
        reqs.append((members, bdfs[(2 * r) % len(bdfs):(2 * r) % len(bdfs) + max(n_members // 8, 1)]))
    egm = [(b"egm%d" % e, bdfs[2 * e] + b" " + bdfs[2 * e + 1] + b"\n", True) for e in range(n_egm)]
    return reqs, egm


def interned(reqs, egm):
    """AllocateCheck's host work: intern the group strings and the EGM keys, build records"""
    devs = [serve.EGMDeviceInfo("/dev/" + n.decode(), g.decode().split()) for n, g, _ in egm]
    eh, eoff, egpu = {}, [0] if devs else [], []
    for d in devs:
        egpu.extend(eh.setdefault(serve.egm_key(g), len(eh)) for g in d.gpu_bdfs)
        eoff.append(len(egpu))
    intern, recs, want, ids, n_members, n_ids = {}, [], [], [], [], []
    for members, dids in reqs:
        for link, vendor, group in members:
            want.append(intern.setdefault(group, len(intern)))
            g = intern.setdefault(link.rsplit(b"/", 1)[-1], len(intern))
            recs.append((len(recs), 0x10DE if vendor[2:].strip(b"\n") == b"10de" else 0xFFFF, 0, g, 0, 0, 0))
        ids.extend(eh.get(serve.egm_key(i.decode()), len(eh)) for i in dids)
        n_members.append(len(members))
        n_ids.append(len(dids))
    return (np.array(recs, dtype=kvgpu.PCI_REC), want, n_members, ids, n_ids, eoff, egpu, len(eh))


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
    with kvgpu.Context(0) as ctx:
        for n_reqs, n_members, n_egm in ((1, 8, 4), (16, 8, 4), (1000, 24, 4), (1, 100_000, 4096)):
            reqs, egm = call_of(n_reqs, n_members, n_egm)
            raw = kvgpu.pack_alloc_raw(reqs, egm)
            args_i = interned(reqs, egm)
            t0 = time.perf_counter()
            kvgpu.pack_alloc_raw(reqs, egm)
            pack_ms = (time.perf_counter() - t0) * 1e3
            t0 = time.perf_counter()
            interned(reqs, egm)
            intern_ms = (time.perf_counter() - t0) * 1e3
            raw_w, raw_k = timed(ctx, lambda: ctx.pci_allocate_raw(raw), args.reps)
            chk_w, chk_k = timed(ctx, lambda: ctx.pci_allocate_check(*args_i), args.reps)
            print("%5d x %6d members, %4d EGM: raw call %.3f ms (%s; packing %.2f ms) | "
                  "interned check %.3f ms (%s; host interning %.2f ms)"
                  % (n_reqs, n_members, n_egm, raw_w, raw_k, pack_ms, chk_w, chk_k, intern_ms))


if __name__ == "__main__":
    main()
