"""Records for the passthrough plugin's Allocate-time group check (kvg_pci_group_check), and its rule restated in
numpy: record i passes iff its iommu_group link read back (no PF_IOMMU_ERR) as want[i] and its vendor read back (no
PF_VENDOR_ERR) as 10de (generic_device_plugin.go:387-397).  Every other field of the record is noise the rule must
ignore, so the generators fill those fields at random."""
import itertools

import numpy as np

import conftest  # noqa: F401  (sys.path)
from kvgpu import _lib as L

VENDORS = (0x10de, 0x10df, 0x8086, 0xffff)
IGNORED_FLAGS = 0xff & ~(L.PF_IOMMU_ERR | L.PF_VENDOR_ERR)   # DRIVER_ERR, DEVICE_ERR, NUMA_ERR and the spare bits


def passes(recs, want) -> np.ndarray:
    flags = recs["flags"].astype(np.uint32)
    return (((flags & L.PF_IOMMU_ERR) == 0) & (recs["iommu_group"] == np.asarray(want, dtype=np.uint32))
            & ((flags & L.PF_VENDOR_ERR) == 0) & (recs["vendor"] == 0x10de))


def first_bad(recs, want) -> int:
    """The smallest failing index, or len(recs) when every record passes (what the kernel writes)."""
    bad = np.flatnonzero(~passes(recs, want))
    return int(bad[0]) if len(bad) else len(recs)


def noise(n, rng) -> tuple:
    """n records that pass against the returned want, every ignored field random."""
    recs = np.zeros(n, dtype=L.PCI_REC)
    recs["addr"] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    recs["device"] = rng.integers(0, 1 << 16, n)
    recs["driver"] = rng.integers(0, 256, n)
    recs["flags"] = rng.integers(0, 256, n) & IGNORED_FLAGS
    recs["numa"] = rng.integers(-(1 << 15), 1 << 15, n)
    recs["vendor"] = 0x10de
    want = rng.integers(0, 64, n).astype(np.uint32)
    recs["iommu_group"] = want
    return recs, want


def combinations() -> list:
    """(iommu_err, vendor_err, vendor, same_group) for every combination the rule distinguishes: 2 x 2 x 4 x 2."""
    return list(itertools.product((False, True), (False, True), VENDORS, (True, False)))


def apply(recs, want, i, combo):
    """Give record i the combination (its ignored fields stay as they are)."""
    iommu_err, vendor_err, vendor, same = combo
    f = int(recs["flags"][i]) & IGNORED_FLAGS
    recs["flags"][i] = f | (L.PF_IOMMU_ERR if iommu_err else 0) | (L.PF_VENDOR_ERR if vendor_err else 0)
    recs["vendor"][i] = vendor
    recs["iommu_group"][i] = want[i] if same else want[i] ^ (1 + (i % 7))


FAILING = [c for c in combinations() if not (not c[0] and not c[1] and c[2] == 0x10de and c[3])]


def with_failures(n, at, rng) -> tuple:
    """n noisy passing records with a random failing combination at each index of `at`."""
    recs, want = noise(n, rng)
    for i in at:
        apply(recs, want, i, FAILING[int(rng.integers(0, len(FAILING)))])
    return recs, want


def failure_sets(n, rng) -> list:
    """Where the failures go: first at 0, at n-1, nowhere, and several where the smallest must win."""
    sets = [[0], [n - 1], [], sorted({x for x in (31, 32, n // 2, n - 1) if x < n})]
    if n > 2:
        lo = int(rng.integers(1, n - 1))
        sets.append(sorted({lo} | set(int(x) for x in rng.integers(lo, n, 5))))
        sets.append(sorted({0, n - 1} | set(int(x) for x in rng.integers(0, n, 3))))
    return sets
