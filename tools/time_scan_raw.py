#!/usr/bin/env python3
"""Host wall time of kvg_scan_pci_raw (raw sysfs text in, GPU decode + scan) against host packing plus kvg_scan_pci,
and the decode kernel's event time with the raw bytes it reads per second.  Inputs: oracle gen_pci records rendered as
the sysfs text a walk would read, at 8, 1,000, 10,000 and 1,000,000 entries.  The card's name and power limit are read
in the same run.   python tools/time_scan_raw.py [reps]   -> one JSON line per size"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200")]
import kvgpu  # noqa: E402
from kvgpu import _lib as L  # noqa: E402
from oracle import oracle as O  # noqa: E402

DRV = {L.DRV_VFIO_PCI: b"../vfio-pci", L.DRV_NVGRACE: b"../nvgrace_gpu_vfio_pci", L.DRV_OTHER: b"../nvidia",
       L.DRV_NONE: b"../none"}


def render(recs) -> kvgpu.PciRaw:
    """every read made; a flag makes that read fail (what read_pci_tree_raw returns for such a tree)"""
    parts, state = [], np.zeros(len(recs), dtype=np.uint16)
    for i, r in enumerate(recs):
        fl = int(r["flags"])
        row = [kvgpu.format_bdf(int(r["addr"])).encode(), b"0x%04x\n" % int(r["vendor"]), DRV[min(int(r["driver"]), 3)],
               b"../%d" % int(r["iommu_group"]), b"%d\n" % int(r["numa"]), b"0x%04x\n" % int(r["device"])]
        st = 0x3E
        for f, bit in ((1, L.PF_VENDOR_ERR), (2, L.PF_DRIVER_ERR), (3, L.PF_IOMMU_ERR), (4, L.PF_NUMA_ERR),
                       (5, L.PF_DEVICE_ERR)):
            if fl & bit:
                st |= 1 << (8 + f)
                row[f] = b""
        state[i] = st
        parts.extend(row)
    off = np.zeros(len(parts) + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(p) for p in parts], dtype=np.uint64)
    return kvgpu.PciRaw([], off, b"".join(parts), state)


def pack(raw, n):
    """the host's part of the packed path: the numeric decode of the same bytes (vendor, driver, group, numa, device)"""
    recs = np.zeros(n, dtype=L.PCI_REC)
    b, off = raw.bytes, raw.off
    for i in range(n):
        g = lambda f: b[off[6 * i + f]:off[6 * i + f + 1]]
        recs[i] = (kvgpu.parse_bdf(g(0).decode()), int(g(1)[2:].strip(b"\n") or b"ffff", 16),
                   int(g(5)[2:].strip(b"\n") or b"0", 16), int(g(3).rsplit(b"/", 1)[-1] or b"0"),
                   {b"vfio-pci": 1, b"nvgrace_gpu_vfio_pci": 2}.get(g(2).rsplit(b"/", 1)[-1], 3), 0,
                   int(g(4).strip() or b"0"))
    return recs


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    text = open(os.path.join(ROOT, "tests", "golden", "pci.ids.gz"), "rb").read()
    import gzip
    text = gzip.decompress(text)
    ids = O.nv_ids(text)
    with kvgpu.Context(0) as ctx:
        ctx.pciids_load(text)
        for n in (8, 1000, 10_000, 1_000_000):
            recs = O.gen_pci(0, n, ids, 16)
            raw = render(recs)
            raw.names = [kvgpu.format_bdf(int(a)) for a in recs["addr"]]
            ctx.scan_pci_raw(raw)
            ctx.scan_pci(recs)
            t_raw, t_pack = [], []
            for _ in range(reps):
                t0 = time.perf_counter()
                ctx.scan_pci_raw(raw)
                t_raw.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                ctx.scan_pci(pack(raw, n) if n <= 10_000 else recs)
                t_pack.append(time.perf_counter() - t0)
            ctx.set_kernel_timing(True)
            ctx.scan_pci_raw(raw)
            times = ctx.kernel_times()
            ctx.set_kernel_timing(False)
            dec = sum(ms for name, ms in times if name == "raw_decode")
            print(json.dumps({"card": card, "entries": n, "raw_bytes": len(raw.bytes),
                              "scan_pci_raw_ms_median": 1e3 * float(np.median(t_raw)),
                              "pack_plus_scan_pci_ms_median": 1e3 * float(np.median(t_pack)),
                              "host_pack_timed": n <= 10_000, "decode_kernel_ms": dec,
                              "decode_GBps": (len(raw.bytes) / (dec * 1e-3) / 1e9) if dec else None}))


if __name__ == "__main__":
    main()
