"""Latency of the request-path rules on the GPU: the vGPU plugin's label check (kvg_mdev_label_match), the passthrough
plugin's group check (kvg_pci_group_check), its Allocate decisions (kvg_pci_allocate_check) and its
GetPreferredAllocation packing (kvg_preferred_allocation), beside
the passthrough plugin's older re-validation batch (kvg_scan_pci, the figure bench.py reports as
allocate_revalidation) and the CPU rules of serve._read_vgpu_label and serve.preferred_allocation, in one process.

  (a) kvg_mdev_label_match at 1, 2, 4, 8 and 16 files, and at 4 containers x 4 files (one call per AllocateRequest:
      the 16 files of the four containers in request order);
  (b) kvg_scan_pci on a pinned batch of 16 records, as bench.py builds it;
  (c) on the CPU, the rule inside _read_vgpu_label (strip, re.sub, decode, compare) on the same bytes in memory;
  (d) kvg_pci_group_check at 1, 2, 4, 8 and 16 records, as serve.GroupCheck builds them: the group members of (b)
      with the groups the maps hold for them, one in three with a driver or device id the check must ignore;
  (e) kvg_preferred_allocation on requests as serve.NumaPacker interns them, beside serve.NumaPacker around it
      (interning, the call, the IDs mapped back) and serve.preferred_allocation, the CPU rule, on the same requests:
      1 request of 4, 8 and 16 available devices over two NUMA nodes, with 0 and 2 must-include IDs; 4 requests of 8
      in one call; 1 request of 10,000 and 1 of 100,000 available devices over eight nodes.  The two large legs take
      min(--calls, 100) timed calls;
  (f) kvg_pci_allocate_check, the group check and the EGM match of every container request in one call, as
      serve.AllocateCheck builds it: 1 request of 1, 2, 4, 8 and 16 members (the records of (d), one DevicesID per
      group) with 0, 1 and 2 EGM devices of two GPUs each, whose strings are the request's first DevicesIDs; and 4
      requests of 4 members in one call, beside what the plugin does without it: four kvg_pci_group_check calls and
      serve.egm_paths_for_allocated_gpus, the CPU rule, per request.

Each size: 50 warm-up calls, then the p50 and p99 of the host wall time of 1,000 calls; every result is checked
against the CPU rule, the group check's against its numpy restatement, the packing's against
serve.preferred_allocation, the allocate check's against the group check and the CPU EGM rule.  The file contents are those of a live
mdev_type/name ("GRID A100-4C\\n"), with one in four of another type.  The card's name, power limit and maximum SM
clock are read with a read-only nvidia-smi query in the same run.

    python tools/time_allocate.py [--calls 1000] [--out DIR]
"""
import argparse
import ctypes as C
import gzip
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"))
import kvgpu  # noqa: E402

WARMUP = 50
NAME = b"GRID_A100-4C"
GROUP_SIZES = (1, 2, 4, 8, 16)
# (label, requests, available devices per request, must-include IDs per request, NUMA nodes)
PREF_LEGS = [("1x4 must0", 1, 4, 0, 2), ("1x4 must2", 1, 4, 2, 2), ("1x8 must0", 1, 8, 0, 2), ("1x8 must2", 1, 8, 2, 2),
             ("1x16 must0", 1, 16, 0, 2), ("1x16 must2", 1, 16, 2, 2), ("4x8", 4, 8, 0, 2),
             ("1x10000", 1, 10_000, 2, 8), ("1x100000", 1, 100_000, 2, 8)]


def stats(lat):
    lat = np.array(lat) * 1e6
    return {"p50_us": round(float(np.percentile(lat, 50)), 2), "p99_us": round(float(np.percentile(lat, 99)), 2)}


def timed(fn, calls):
    lat = []
    for it in range(WARMUP + calls):
        t0 = time.perf_counter()
        fn()
        dt = time.perf_counter() - t0
        if it >= WARMUP:
            lat.append(dt)
    return stats(lat)


def cpu_rule(raw):
    return re.sub(rb"[\t\n\f\r ]+", b"_", raw.strip(b"\n")).decode("latin-1")


def group_rule(recs, want):
    """generic_device_plugin.go:388-397 on kvg_pci_rec: the smallest failing index, or len(recs)."""
    ok = (((recs["flags"] & (kvgpu._lib.PF_IOMMU_ERR | kvgpu._lib.PF_VENDOR_ERR)) == 0)
          & (recs["iommu_group"] == want) & (recs["vendor"] == 0x10de))
    bad = np.flatnonzero(~ok)
    return int(bad[0]) if len(bad) else len(recs)


def pref_call(n_reqs, n_avail, n_must, n_nodes):
    """(devs, requests): n_avail devices spread over n_nodes nodes in runs, each request listing them all in kubelet
    order; the must-include IDs sit on the last node and the size is half a node's devices plus one, so the packing
    fills from one node: the must-include node when there is one."""
    devs = [("0000:%02x:%02x.0" % (i >> 8, i & 0xff), i * n_nodes // n_avail) for i in range(n_avail)]
    ids = [d for d, _ in devs]
    reqs = [(ids, ids[n_avail - n_must:], n_avail // n_nodes // 2 + 1) for _ in range(n_reqs)]
    return devs, reqs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    print(card, flush=True)
    lib = kvgpu.load()
    out = {"card": card, "calls": a.calls, "warmup": WARMUP, "what": "host wall time of one call", "label_match": {},
           "scan_pci_16": None, "cpu_rule": {}, "group_check": {}, "preferred_allocation": {}, "numa_packer": {},
           "preferred_cpu_rule": {}, "allocate_check": {}, "allocate_check_4x4": None, "group_check_4x4_egm_cpu": None}
    legs = [("%d" % k, k) for k in (1, 2, 4, 8, 16)] + [("4x4", 16)]
    with kvgpu.Context(0) as ctx:
        with gzip.open(os.path.join(ROOT, "tests", "golden", "pci.ids.gz"), "rb") as f:
            ctx.pciids_load(f.read())                                  # a scan joins names: it needs the table
        for label, k in legs:
            files = [b"GRID A100-4C\n" if i % 4 != 3 else b"GRID A100-8C\n" for i in range(k)]
            want = np.array([cpu_rule(f) == NAME.decode() for f in files], dtype=np.uint8)
            td, keep = ctx._type_dict(files)
            match = np.zeros(k, dtype=np.uint8)

            def gpu():
                assert lib.kvg_mdev_label_match(ctx.handle, C.byref(td), NAME, len(NAME), match.ctypes.data) == 0
            before = ctx.launch_count
            out["label_match"][label] = timed(gpu, a.calls)
            assert ctx.launch_count - before == WARMUP + a.calls      # one launch per call
            assert np.array_equal(match, want)
            assert np.array_equal(ctx.mdev_label_match(files, NAME), want.astype(bool))

            def cpu():
                return [cpu_rule(f) == "GRID_A100-4C" for f in files]
            out["cpu_rule"][label] = timed(cpu, a.calls)
            assert np.array_equal(np.array(cpu(), dtype=np.uint8), want)
            del keep

        import torch
        rr = np.zeros(16, dtype=kvgpu.PCI_REC)
        for i in range(16):
            rr[i] = (i, 0x10de, 0, i // 2, 1, 0, 0)                    # what BatchRevalidator builds (bench.py)
        hr = torch.from_numpy(np.frombuffer(rr.tobytes(), dtype=np.uint8).copy()).pin_memory()

        def scan():
            res = C.POINTER(kvgpu._lib.PciResultC)()
            assert lib.kvg_scan_pci(ctx.handle, hr.data_ptr(), 16, C.byref(res)) == 0
            assert res.contents.n_survivors == 16
            lib.kvg_result_free(res)
        out["scan_pci_16"] = timed(scan, a.calls)

        for k in GROUP_SIZES:
            recs = rr[:k].copy()
            recs["driver"][::3] = kvgpu._lib.DRV_OTHER                 # ignored by the rule
            recs["device"][1::3] = 0x1b38
            want = np.ascontiguousarray(recs["iommu_group"], dtype=np.uint32)
            first, expect = C.c_size_t(), group_rule(recs, want)

            def check():
                assert lib.kvg_pci_group_check(ctx.handle, recs.ctypes.data, want.ctypes.data, k, C.byref(first)) == 0
                assert first.value == expect
            before = ctx.launch_count
            out["group_check"]["%d" % k] = timed(check, a.calls)
            assert ctx.launch_count - before == WARMUP + a.calls      # one launch per call
            bad = want.copy()
            bad[k - 1] += 1                                            # the last member's link moved
            assert ctx.pci_group_check(recs, bad) == group_rule(recs, bad) == k - 1

        from kvgpu import serve
        for label, n_reqs, n_avail, n_must, n_nodes in PREF_LEGS:
            devs, reqs = pref_call(n_reqs, n_avail, n_must, n_nodes)
            calls = a.calls if n_avail <= 1000 else min(a.calls, 100)
            want = [serve.preferred_allocation(devs, av, m, sz) for av, m, sz in reqs]
            seen = []

            def keep(ids, n_m, n_a, sizes):                         # the arrays NumaPacker builds, for the raw leg
                seen.append((ids, np.zeros(len(sizes), dtype=kvgpu._lib.PREF_REQ)))
                seen[-1][1]["n_must"], seen[-1][1]["n_avail"], seen[-1][1]["size"] = n_m, n_a, sizes
                return ctx.preferred_allocation(ids, n_m, n_a, sizes)
            packer = serve.NumaPacker(keep)
            assert packer(devs, reqs) == want
            ids, rq = seen[0]
            res = np.zeros(n_reqs, dtype=kvgpu._lib.PREF_RES)
            pos = np.zeros(len(ids), dtype=np.uint32)

            def gpu():
                assert lib.kvg_preferred_allocation(ctx.handle, rq.ctypes.data, n_reqs, ids.ctypes.data, len(ids),
                                                    res.ctypes.data, pos.ctypes.data) == 0
            before = ctx.launch_count
            out["preferred_allocation"][label] = timed(gpu, calls)
            assert ctx.launch_count - before == WARMUP + calls         # one launch per call
            assert list(res["n_out"]) == [len(w) for w in want]
            packer = serve.NumaPacker(ctx.preferred_allocation)
            out["numa_packer"][label] = timed(lambda: packer(devs, reqs), calls)
            assert packer(devs, reqs) == want
            out["preferred_cpu_rule"][label] = timed(
                lambda: [serve.preferred_allocation(devs, av, m, sz) for av, m, sz in reqs], calls)

        # (f) the group check and the EGM match of every container request in one call
        egm_devs = [serve.EGMDeviceInfo("/dev/egm0", ["0000:00:00.0", "0000:00:01.0"]),
                    serve.EGMDeviceInfo("/dev/egm1", ["0000:00:02.0", "0000:00:03.0"])]

        def alloc_args(n_reqs, k, n_egm):
            """The arrays AllocateCheck builds for n_reqs requests of k members (the records of (d)) and one DevicesID
            per group; the IDs are the first GPU strings of the EGM devices, then strings no device lists."""
            recs = np.concatenate([rr[:k]] * n_reqs)
            recs["driver"][::3] = kvgpu._lib.DRV_OTHER
            want = np.ascontiguousarray(recs["iommu_group"], dtype=np.uint32)
            n_ids = (k + 1) // 2
            devices_ids = ["0000:00:%02x.0" % i for i in range(n_ids)]
            handle = {serve.egm_key(g): h for h, g in enumerate(g for e in egm_devs[:n_egm] for g in e.gpu_bdfs)}
            ids = np.array([handle.get(serve.egm_key(b), len(handle)) for b in devices_ids] * n_reqs, dtype=np.uint32)
            egm_off = np.array([0, 2, 4][:n_egm + 1] if n_egm else [], dtype=np.uint32)
            egm_gpu = np.arange(2 * n_egm, dtype=np.uint32)
            reqs = np.zeros(n_reqs, dtype=kvgpu._lib.ALLOC_REQ)
            reqs["n_members"], reqs["n_ids"] = k, n_ids
            return recs, want, reqs, ids, egm_off, egm_gpu, len(handle), devices_ids

        def alloc_leg(n_reqs, k, n_egm):
            recs, want, reqs, ids, egm_off, egm_gpu, n_egm_gpus, devices_ids = alloc_args(n_reqs, k, n_egm)
            first = np.zeros(n_reqs, dtype=np.uint32)
            take = np.zeros(max(n_reqs * n_egm, 1), dtype=np.uint8)
            expect_take = [p in egm_paths_for(devices_ids, egm_devs[:n_egm]) for p in
                           [e.dev_path for e in egm_devs[:n_egm]]] * n_reqs
            args = (ctx.handle, reqs.ctypes.data, n_reqs, recs.ctypes.data, want.ctypes.data, len(recs),
                    ids.ctypes.data, len(ids), egm_off.ctypes.data if n_egm else None, egm_gpu.ctypes.data, n_egm,
                    n_egm_gpus, first.ctypes.data, take.ctypes.data)    # the pointers taken once, as a host would

            def gpu():
                assert lib.kvg_pci_allocate_check(*args) == 0
            before = ctx.launch_count
            st = timed(gpu, a.calls)
            assert ctx.launch_count - before == WARMUP + a.calls      # one launch per call
            assert first.tolist() == [group_rule(recs[:k], want[:k])] * n_reqs == [k] * n_reqs
            assert take[:n_reqs * n_egm].astype(bool).tolist() == expect_take
            return st, recs, want, devices_ids
        egm_paths_for = serve.egm_paths_for_allocated_gpus
        for k in GROUP_SIZES:
            for n_egm in (0, 1, 2):
                out["allocate_check"]["1x%d egm%d" % (k, n_egm)] = alloc_leg(1, k, n_egm)[0]
        out["allocate_check_4x4"], recs, want, devices_ids = alloc_leg(4, 4, 2)
        first = C.c_size_t()
        ptrs = [(recs[4 * r:].ctypes.data, want[4 * r:].ctypes.data) for r in range(4)]

        def four_group_checks():
            for rp, wp in ptrs:
                assert lib.kvg_pci_group_check(ctx.handle, rp, wp, 4, C.byref(first)) == 0
                assert first.value == 4
                assert egm_paths_for(devices_ids, egm_devs) == ["/dev/egm0"]
        out["group_check_4x4_egm_cpu"] = timed(four_group_checks, a.calls)

    print("%-28s %10s %10s" % ("call", "p50 us", "p99 us"))
    for label, _ in legs:
        s = out["label_match"][label]
        print("%-28s %10.1f %10.1f" % ("kvg_mdev_label_match " + label, s["p50_us"], s["p99_us"]))
    s = out["scan_pci_16"]
    print("%-28s %10.1f %10.1f" % ("kvg_scan_pci 16 records", s["p50_us"], s["p99_us"]))
    for k in GROUP_SIZES:
        s = out["group_check"]["%d" % k]
        print("%-28s %10.1f %10.1f" % ("kvg_pci_group_check %d" % k, s["p50_us"], s["p99_us"]))
    for label, _ in legs:
        s = out["cpu_rule"][label]
        print("%-28s %10.1f %10.1f" % ("CPU rule " + label, s["p50_us"], s["p99_us"]))
    for key, what in (("preferred_allocation", "kvg_preferred_allocation"), ("numa_packer", "NumaPacker"),
                      ("preferred_cpu_rule", "CPU preferred_allocation")):
        for label, *_ in PREF_LEGS:
            s = out[key][label]
            print("%-40s %10.1f %10.1f" % ("%s %s" % (what, label), s["p50_us"], s["p99_us"]))
    for label, s in out["allocate_check"].items():
        print("%-40s %10.1f %10.1f" % ("kvg_pci_allocate_check " + label, s["p50_us"], s["p99_us"]))
    for label, s in (("kvg_pci_allocate_check 4x4 egm2", out["allocate_check_4x4"]),
                     ("4 x kvg_pci_group_check + CPU EGM", out["group_check_4x4_egm_cpu"])):
        print("%-40s %10.1f %10.1f" % (label, s["p50_us"], s["p99_us"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_allocate.json"), "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
