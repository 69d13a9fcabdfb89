"""Timing of the re-scan deltas against the plain scans on one GPU: kvg_scan_pci_delta against kvg_scan_pci
(--kind pci, the default), kvg_scan_mdev_delta against kvg_scan_mdev (--kind mdev), and kvg_dev_scan_pci_sharded +
kvg_dev_scan_pci_shard_fetch_delta against kvg_dev_scan_pci_sharded + kvg_dev_scan_pci_shard_fetch (--kind shard:
one rank, world 1, over peer windows; sizes are records per rank), and the same for the sharded mdev scan
(--kind mdev-shard: kvg_dev_scan_mdev_sharded + kvg_dev_scan_mdev_shard_fetch_delta against
kvg_dev_scan_mdev_sharded + kvg_dev_scan_mdev_shard_fetch).

A sequence of snapshots changes about 0.1 % of the records per step (PCI: regroups, NUMA moves, re-binds,
hot-removes and hot-adds in turn; mdev: retypes, NUMA moves, parent moves, destroys and hot-adds).  For each size both
entry points walk the same sequence, alternating in rounds; the host wall time of each C call (it returns with its
result on the host) is recorded.  A separate pass with kernel timing on reports the device time of the delta kernels.
The card name and power limit are read in the same run.

    python tools/time_delta.py [--kind pci|mdev|shard|mdev-shard] [--sizes 10000,1000000] [--steps 200] [--types 256]
                               [--out results.json]
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
    return list(pci_sequence(n, ids, steps, seed))


def pci_sequence(n, ids, steps, seed=1):
    """The PCI snapshots one after the other (steps + 1 of them)."""
    rng = np.random.default_rng(seed)
    recs = O.gen_pci(seed, n, ids, 16)
    recs["addr"] = np.arange(n, dtype=np.uint32) * 4
    yield recs
    for s in range(steps):
        r = recs.copy()
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
            add = add[np.unique(add["addr"], return_index=True)[1]]   # two picks may land on one free address
            r = np.sort(np.concatenate([r, add]), order="addr", kind="stable")
        recs = np.ascontiguousarray(r)
        yield recs


def mdev_snapshots(n, steps, n_types, seed=1):
    """mdev records with canonical UUIDs spaced by 4 in their first word; types of an n_types-entry dictionary."""
    rng = np.random.default_rng(seed)
    recs = O.gen_mdev(seed, n)
    recs["uuid"][:, :4] = (np.arange(n, dtype=np.uint32) * 4).astype(">u4").view(np.uint8).reshape(n, 4)
    recs["type_idx"] = rng.integers(0, n_types, n)
    key = lambda a: np.ascontiguousarray(a["uuid"]).view("V16").ravel()
    out = [recs]
    for s in range(steps):
        r = out[-1].copy()
        k = max(1, n // 1000)
        pick = rng.choice(len(r), k, replace=False)
        kind = s % 5
        if kind == 0:
            r["type_idx"][pick] = rng.integers(0, n_types, k)
        elif kind == 1:
            r["parent_numa"][pick] = (r["parent_numa"][pick] + 1) % 4
        elif kind == 2:
            r["parent"][pick] = r["parent"][rng.choice(len(r), k)]
        elif kind == 3:
            r = np.delete(r, pick)
        else:
            add = r[pick].copy()
            add["uuid"][:, 3] += (1 + rng.integers(0, 3, k)).astype(np.uint8)
            add = add[~np.isin(key(add), key(r))]
            add = add[np.unique(key(add), return_index=True)[1]]
            r = np.concatenate([r, add])
            r = r[np.argsort(key(r), kind="stable")]
        out.append(np.ascontiguousarray(r))
    return out


def time_sequence(ctx, seq, plain, delta, reset, prefix):
    """Warm up, then alternate the two entry points in rounds of ten steps; one more pass with kernel timing on."""
    for r in seq[:10]:                       # warm-up: buffers, pinned blocks, radix hints
        plain(r)
        delta(r)
    reset()
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
            if name.startswith(prefix):
                per.setdefault(name, []).append(t * 1e3)
    ctx.set_kernel_timing(False)
    return tp, td, changes, per


def main_mdev(a, card):
    ctx = kvgpu.Context(0)
    ctx.pciids_load(util.pciids_text())
    lib, h = ctx._lib, ctx.handle
    types = [b"GRID T%05d\n" % k for k in range(a.types)]
    td_c, keep = ctx._type_dict(types)
    out = {"card": card, "kind": "mdev", "steps": a.steps, "types": a.types, "sizes": {}}
    for n in [int(x) for x in a.sizes.split(",")]:
        seq = mdev_snapshots(n, a.steps, a.types)
        res, dl = C.POINTER(L.MdevResultC)(), C.POINTER(L.MdevDeltaC)()

        def plain(r):
            t0 = time.perf_counter()
            rc = lib.kvg_scan_mdev(h, r.ctypes.data, len(r), C.byref(td_c), C.byref(res))
            t1 = time.perf_counter()
            assert rc == 0
            lib.kvg_result_free(res)
            return t1 - t0

        def delta(r):
            t0 = time.perf_counter()
            rc = lib.kvg_scan_mdev_delta(h, r.ctypes.data, len(r), C.byref(td_c), C.byref(res), C.byref(dl))
            t1 = time.perf_counter()
            assert rc == 0
            n_changes = int(dl.contents.n_changes)
            lib.kvg_result_free(res)
            lib.kvg_result_free(dl)
            return t1 - t0, n_changes

        tp, td, changes, per = time_sequence(ctx, seq, plain, delta, ctx.scan_mdev_delta_reset, "mdev_delta_")
        q = lambda v, p: round(float(np.percentile(np.array(v) * 1e6, p)), 1)
        out["sizes"][n] = {
            "scan_mdev_us": {"p50": q(tp, 50), "p90": q(tp, 90)},
            "scan_mdev_delta_us": {"p50": q(td, 50), "p90": q(td, 90)},
            "changes_per_step_median": int(np.median(changes)),
            "kernel_us_median": {k: round(float(np.median(v)), 2) for k, v in per.items()},
        }
        print(n, json.dumps(out["sizes"][n]), flush=True)
    del keep
    ctx.close()
    return out


def main_shard(a, card):
    """Each step: the next snapshot goes to the device untimed, then scan + fetch and scan + fetch_delta on it, in
    turn (the plain fetch leaves the delta's previous result alone)."""
    import torch
    text = util.pciids_text()
    ids = O.nv_ids(text)
    sizes = [int(x) for x in a.sizes.split(",")]
    cap = max(sizes) + max(sizes) // 50 + 64
    ctx = kvgpu.Context(0)
    ctx.pciids_load(text)
    sh = kvgpu.ShardedScan(ctx, 0, 1, lambda b, src: b, lambda b: [b], cap)
    lib, h = ctx._lib, ctx.handle
    buf = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
    out = {"card": card, "kind": "shard", "world": 1, "exchange": sh.mode, "steps": a.steps, "sizes": {}}
    res, dl = C.POINTER(L.PciShardResultC)(), C.POINTER(L.PciDeltaC)()

    def plain(n):
        t0 = time.perf_counter()
        rc = lib.kvg_dev_scan_pci_sharded(h, buf.data_ptr(), n)
        rc = rc or lib.kvg_dev_scan_pci_shard_fetch(h, C.byref(res))
        t1 = time.perf_counter()
        assert rc == 0
        lib.kvg_result_free(res)
        return t1 - t0

    def delta(n):
        t0 = time.perf_counter()
        rc = lib.kvg_dev_scan_pci_sharded(h, buf.data_ptr(), n)
        rc = rc or lib.kvg_dev_scan_pci_shard_fetch_delta(h, C.byref(res), C.byref(dl))
        t1 = time.perf_counter()
        assert rc == 0, (rc, lib.kvg_last_error(h))
        n_changes = int(dl.contents.n_changes)
        lib.kvg_result_free(res)
        lib.kvg_result_free(dl)
        return t1 - t0, n_changes

    for n in sizes:
        tp, td, changes, per = [], [], [], {}
        sh.delta_reset()
        for i, r in enumerate(pci_sequence(n, ids, a.steps + 19)):
            buf[:r.nbytes].copy_(torch.from_numpy(r.view(np.uint8)))
            torch.cuda.synchronize()
            if i < 10:                           # warm-up: buffers, pinned blocks, radix hints
                plain(len(r))
                delta(len(r))
                continue
            if i >= a.steps + 10:                # the last ten steps: kernel times, in a pass of their own
                ctx.set_kernel_timing(True)
                delta(len(r))
                for name, t in ctx.kernel_times():
                    if name.startswith("shard_delta_"):
                        per.setdefault(name, []).append(t * 1e3)
                ctx.set_kernel_timing(False)
                continue
            tp.append(plain(len(r)))
            t, c = delta(len(r))
            td.append(t)
            changes.append(c)
        q = lambda v, p: round(float(np.percentile(np.array(v) * 1e6, p)), 1)
        out["sizes"][n] = {
            "scan_fetch_us": {"p50": q(tp, 50), "p90": q(tp, 90)},
            "scan_fetch_delta_us": {"p50": q(td, 50), "p90": q(td, 90)},
            "changes_per_step_median": int(np.median(changes)),
            "kernel_us_median": {k: round(float(np.median(v)), 2) for k, v in per.items()},
        }
        print(n, json.dumps(out["sizes"][n]), flush=True)
    del buf
    torch.cuda.synchronize()
    sh.close()
    ctx.close()
    return out


def main_mdev_shard(a, card):
    """As main_shard, over the mdev snapshots of main_mdev (an mdev record takes two PCI records of window)."""
    import torch
    sizes = [int(x) for x in a.sizes.split(",")]
    cap = 2 * (max(sizes) + max(sizes) // 50 + 64)
    ctx = kvgpu.Context(0)
    ctx.pciids_load(util.pciids_text())
    sh = kvgpu.ShardedScan(ctx, 0, 1, lambda b, src: b, lambda b: [b], cap)
    lib, h = ctx._lib, ctx.handle
    types = [b"GRID T%05d\n" % k for k in range(a.types)]
    td_c, keep = ctx._type_dict(types)
    buf = torch.empty(cap * 16, dtype=torch.uint8, device="cuda")
    out = {"card": card, "kind": "mdev-shard", "world": 1, "exchange": sh.mode, "steps": a.steps, "types": a.types,
           "sizes": {}}
    res, dl = C.POINTER(L.MdevShardResultC)(), C.POINTER(L.MdevDeltaC)()

    def plain(n):
        t0 = time.perf_counter()
        rc = lib.kvg_dev_scan_mdev_sharded(h, buf.data_ptr(), n, C.byref(td_c))
        rc = rc or lib.kvg_dev_scan_mdev_shard_fetch(h, C.byref(res))
        t1 = time.perf_counter()
        assert rc == 0, (rc, lib.kvg_last_error(h))
        lib.kvg_result_free(res)
        return t1 - t0

    def delta(n):
        t0 = time.perf_counter()
        rc = lib.kvg_dev_scan_mdev_sharded(h, buf.data_ptr(), n, C.byref(td_c))
        rc = rc or lib.kvg_dev_scan_mdev_shard_fetch_delta(h, C.byref(res), C.byref(dl))
        t1 = time.perf_counter()
        assert rc == 0, (rc, lib.kvg_last_error(h))
        n_changes = int(dl.contents.n_changes)
        lib.kvg_result_free(res)
        lib.kvg_result_free(dl)
        return t1 - t0, n_changes

    for n in sizes:
        tp, td, changes, per = [], [], [], {}
        sh.mdev_delta_reset()
        for i, r in enumerate(mdev_snapshots(n, a.steps + 19, a.types)):
            buf[:r.nbytes].copy_(torch.from_numpy(r.view(np.uint8).ravel()))
            torch.cuda.synchronize()
            if i < 10:                           # warm-up: buffers, pinned blocks, radix hints
                plain(len(r))
                delta(len(r))
                continue
            if i >= a.steps + 10:                # the last ten steps: kernel times, in a pass of their own
                ctx.set_kernel_timing(True)
                delta(len(r))
                for name, t in ctx.kernel_times():
                    if name.startswith("shard_mdev_delta_"):
                        per.setdefault(name, []).append(t * 1e3)
                ctx.set_kernel_timing(False)
                continue
            tp.append(plain(len(r)))
            t, c = delta(len(r))
            td.append(t)
            changes.append(c)
        q = lambda v, p: round(float(np.percentile(np.array(v) * 1e6, p)), 1)
        out["sizes"][n] = {
            "scan_fetch_us": {"p50": q(tp, 50), "p90": q(tp, 90)},
            "scan_fetch_delta_us": {"p50": q(td, 50), "p90": q(td, 90)},
            "changes_per_step_median": int(np.median(changes)),
            "kernel_us_median": {k: round(float(np.median(v)), 2) for k, v in per.items()},
        }
        print(n, json.dumps(out["sizes"][n]), flush=True)
    del keep, buf
    torch.cuda.synchronize()
    sh.close()
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,1000000")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", help="also write the JSON result to this file")
    ap.add_argument("--kind", choices=("pci", "mdev", "shard", "mdev-shard"), default="pci")
    ap.add_argument("--types", type=int, default=256, help="--kind mdev / mdev-shard: entries of the type dictionary")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    if a.kind in ("mdev", "shard", "mdev-shard"):
        run = {"mdev": main_mdev, "shard": main_shard, "mdev-shard": main_mdev_shard}[a.kind]
        out = run(a, card[0] if card else "unknown")
        if a.out:
            with open(a.out, "w") as f:
                json.dump(out, f, indent=1)
        print(json.dumps(out))
        return
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

        tp, td, changes, per = time_sequence(ctx, seq, plain, delta, ctx.scan_pci_delta_reset, "delta_")
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
