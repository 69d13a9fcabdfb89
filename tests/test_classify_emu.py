"""K3, the record-classification pipeline (k_classify_ragged -> k_tile_offsets -> k_pack_survivors, and
the one-launch k_compact<PciClassifyOp, 128, 8>), executed on the CPU from its real kernel source under the warp
emulator of tools/emu/: drop rules of device_plugin.go:203-238, NUMA clamp, name join through nv_index,
Walk-order compaction across tiles, the device-side maxima that size the radix plan."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest  # noqa: F401
import kvgpu
import util
from oracle import oracle as O

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_classify())
    L.emu_classify_pci.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L


def expected_survivors(recs, nv_index):
    drop = 1 | 2 | 4 | 8
    keep = (recs["vendor"] == 0x10de) & ((recs["flags"] & drop) == 0) & ((recs["driver"] == 1) | (recs["driver"] == 2))
    r = recs[keep]
    s = np.zeros(len(r), dtype=kvgpu.PCI_SURV)
    s["addr"], s["iommu_group"], s["device"] = r["addr"], r["iommu_group"], r["device"]
    numa = r["numa"].astype(np.int32)
    numa[(numa < 0) | ((r["flags"] & 16) != 0)] = 0          # :227-230, :316-318
    s["numa"] = numa.astype(np.uint16)
    s["name_slot"] = nv_index[r["device"]]
    return s


@pytest.mark.parametrize("variant", [0, 1], ids=["ragged_offsets_pack", "oneshot"])
def test_classify_pipeline_matches_the_drop_rules(emu, variant):
    ids = O.nv_ids(util.pciids_text())
    rng = np.random.default_rng(3)
    nv_index = rng.integers(0, 1 << 20, 65536, dtype=np.uint64).astype(np.uint32)
    for n, gbits in ((0, 0), (1, 0), (1023, 8), (1024, 8), (1025, 8), (3000, 0), (5000, 12)):
        recs = O.gen_pci(11, n, ids, gbits)
        if n >= 1024:
            recs[1023] = (0xabc, 0x10de, int(ids[3]), 0x7fffffff, 2, 0, -1)     # tile edge, widest group, numa -1
        out = np.zeros(n + 1, dtype=kvgpu.PCI_SURV)
        ctrl = np.zeros(3, dtype=np.uint32)
        buf = np.ascontiguousarray(recs) if n else np.zeros(1, dtype=kvgpu.PCI_REC)
        assert emu.emu_classify_pci(buf.ctypes.data, n, nv_index.ctypes.data, variant, out.ctypes.data, ctrl.ctypes.data) == 0
        want = expected_survivors(recs, nv_index)
        assert int(ctrl[0]) == len(want), (n, variant)
        assert np.array_equal(out[:len(want)], want), (n, variant)
        if len(want):
            assert int(ctrl[1]) == int(want["iommu_group"].max()) and int(ctrl[2]) == int(want["device"].max())


def test_health_diff_kernel_reports_transitions_in_record_order(emu):
    """K6 = k_compact<HealthOp<PciHealthRule>, 256, 8> (BASELINE.json config 5): the transition list of every tick, like
    tests/test_gpu_parity.py::test_health_rescan_transitions, from kernel source."""
    emu.emu_health_rescan.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    ids = O.nv_ids(util.pciids_text())
    n = 10_000
    recs = O.gen_pci(0, n, ids, 0)
    alive_prev = np.zeros(n + 1, dtype=np.uint8)
    prev = np.zeros(n, dtype=bool)
    rng = np.random.default_rng(5)
    drop = 1 | 2 | 4 | 8
    for tick in range(5):
        if tick:
            flip = rng.integers(0, n, 10)
            recs["driver"][flip] = rng.integers(0, 5, 10)
            recs["flags"][flip] ^= rng.integers(0, 32, 10).astype(np.uint8)
        changed = np.zeros(n + 1, dtype=np.uint32)
        ctrl = np.zeros(2, dtype=np.uint32)
        assert emu.emu_health_rescan(np.ascontiguousarray(recs).ctypes.data, n, alive_prev.ctypes.data,
                                     changed.ctypes.data, ctrl.ctypes.data) == 0
        now = (recs["vendor"] == 0x10de) & ((recs["flags"] & drop) == 0) & ((recs["driver"] == 1) | (recs["driver"] == 2))
        idx = np.nonzero(now != prev)[0]
        want = (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)
        assert int(ctrl[0]) == len(want) and int(ctrl[1]) == int(now.sum())
        assert np.array_equal(changed[:len(want)], want)
        assert np.array_equal(alive_prev[:n].astype(bool), now)
        prev = now


def test_health_small_kernel_one_cta(emu):
    """K6 at poll-loop sizes = k_health_small (one CTA, the transition list and the counters written where the
    host reads them): same contract as the look-back form, at sizes around the row and CTA boundaries."""
    emu.emu_health_small.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    ids = O.nv_ids(util.pciids_text())
    drop = 1 | 2 | 4 | 8
    rng = np.random.default_rng(6)
    for n in (1, 1023, 1024, 1025, 10_000, 12_288, 12_289, 32_768):
        recs = O.gen_pci(0, n, ids, 0)
        alive_prev = np.zeros(n + 1, dtype=np.uint8)
        prev = np.zeros(n, dtype=bool)
        for tick in range(3):
            if tick:
                flip = rng.integers(0, n, 10)
                recs["driver"][flip] = rng.integers(0, 5, 10)
            changed = np.zeros(n + 1, dtype=np.uint32)
            hdr = np.zeros(3, dtype=np.uint32)
            assert emu.emu_health_small(np.ascontiguousarray(recs).ctypes.data, n, alive_prev.ctypes.data,
                                        changed.ctypes.data, hdr.ctypes.data) == 0
            now = (recs["vendor"] == 0x10de) & ((recs["flags"] & drop) == 0) & ((recs["driver"] == 1) | (recs["driver"] == 2))
            idx = np.nonzero(now != prev)[0]
            want = (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)
            assert int(hdr[0]) == int(now.sum()) and int(hdr[1]) == len(want) and int(hdr[2]) == 7, (n, tick)
            assert np.array_equal(changed[:len(want)], want)
            assert np.array_equal(alive_prev[:n].astype(bool), now)
            prev = now


def test_mdev_dictionary_and_classification_from_kernel_source(emu):
    """K5: label rule (Trim "\\n", \\s+ -> "_", device_plugin.go:341-342), equal labels merge into the
    smallest raw index, drop rules :270-279, NUMA clamp, survivors in Walk order with their source index."""
    import re
    emu.emu_scan_mdev.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]
    raw_types = O.gen_type_names(64) + [b"\n\nGRID  P100X-1B\n", b"GRID P100X-1B", b"GRID\tP100X-1B\n\n", b"", b"\n", b" x \r\n y"]
    nt = len(raw_types)
    blob = np.frombuffer(b"".join(raw_types) + b"\0", dtype=np.uint8).copy()
    off = np.zeros(nt + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(t) for t in raw_types])
    want_labels = [re.sub(rb"[\t\n\f\r ]+", b"_", t.strip(b"\n")) for t in raw_types]
    want_canon = [want_labels.index(l) for l in want_labels]
    for n in (0, 1, 511, 512, 513, 3000):
        recs = O.gen_mdev(5, n)
        if n:
            recs["type_idx"] = recs["type_idx"] % (nt + 3)           # a few out-of-range type indices
        label = np.zeros(len(blob) + 1, dtype=np.uint8)
        label_len = np.zeros(nt, dtype=np.uint32)
        canon = np.zeros(nt, dtype=np.uint16)
        surv = np.zeros(n + 1, dtype=O.MDEV_SURV)
        ctrl = np.zeros(3, dtype=np.uint32)
        buf = np.ascontiguousarray(recs) if n else np.zeros(1, dtype=O.MDEV_REC)
        assert emu.emu_scan_mdev(buf.ctypes.data, n, blob.ctypes.data, off.ctypes.data, nt, label.ctypes.data,
                                 label_len.ctypes.data, canon.ctypes.data, surv.ctypes.data, ctrl.ctypes.data) == 0
        got_labels = [bytes(label[off[k]:off[k] + label_len[k]]) for k in range(nt)]
        assert got_labels == want_labels and list(canon) == want_canon
        keep = ((recs["flags"] & 3) == 0) & (recs["type_idx"] < nt)
        r = recs[keep]
        assert int(ctrl[0]) == len(r)
        s = surv[:len(r)]
        assert np.array_equal(s["uuid"], r["uuid"]) and np.array_equal(s["parent"], r["parent"])
        assert np.array_equal(s["type_key"], np.array(want_canon, dtype=np.uint16)[r["type_idx"]])
        numa = r["parent_numa"].astype(np.int32)
        numa[(numa < 0) | ((r["flags"] & 4) != 0)] = 0
        assert np.array_equal(s["numa"], numa.astype(np.uint16))
        assert np.array_equal(s["src"], np.nonzero(keep)[0].astype(np.uint32))
        if len(r):
            assert int(ctrl[1]) == int(r["parent"].max()) and int(ctrl[2]) == int(s["type_key"].max())
