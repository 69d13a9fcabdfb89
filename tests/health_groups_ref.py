"""numpy restatement of kvg_health_rescan_groups (include/kvgpu.h): the passthrough health state machine by IOMMU
group, independent of the kernels.

Record i carries one bit h from the previous tick.  With G the handles of the IOMMU groups whose VFIO node exists:

    h' = createIommuDeviceMap's filter (util.pci_alive) & (iommu_group in G)
    i is listed iff h' != h, as (i << 1) | h'
"""
from dataclasses import dataclass

import numpy as np

import util


def step(recs, group_nodes, h):
    """One tick: -> (changed words, n_alive, h')."""
    g = np.unique(np.asarray(group_nodes, dtype=np.uint32))
    now = util.pci_alive(recs) & np.isin(recs["iommu_group"], g)
    idx = np.nonzero(h != now)[0]
    changed = (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)
    return changed, int(now.sum()), now


@dataclass
class Delta:
    n_records: int
    n_alive: int
    changed: np.ndarray


class HealthGroupsRef:
    """The per-context state of kvg_health_rescan_groups: a different n re-arms it, as does reset()."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.h = np.zeros(0, dtype=bool)

    def rescan(self, recs, group_nodes=()) -> Delta:
        n = len(recs)
        if n != len(self.h):
            self.h = np.zeros(n, dtype=bool)
        changed, alive, self.h = step(recs, group_nodes, self.h)
        return Delta(n, alive, changed)

    def state_bytes(self):
        return self.h.astype(np.uint8)


def make_recs(n, rng, per_group=4, alive_frac=0.9):
    """n PCI records, `per_group` consecutive functions per IOMMU group (handles from 1); about `alive_frac` of them
    pass the filter, the rest fail it by vendor, driver or a read-error flag."""
    from kvgpu import PCI_REC
    recs = np.zeros(n, dtype=PCI_REC)
    recs["addr"] = np.arange(n, dtype=np.uint32)
    recs["vendor"] = 0x10DE
    recs["device"] = 0x2330
    recs["iommu_group"] = 1 + np.arange(n, dtype=np.uint32) // per_group
    recs["driver"] = 1 + (np.arange(n) % 2)
    dead = np.nonzero(rng.random(n) >= alive_frac)[0]
    kill(recs, dead, rng)
    return recs


def kill(recs, idx, rng):
    """Make records idx fail the filter, each one of three ways."""
    how = rng.integers(0, 3, len(idx))
    recs["vendor"][idx[how == 0]] = 0x8086
    recs["driver"][idx[how == 1]] = 3
    recs["flags"][idx[how == 2]] |= np.uint8(1) << rng.integers(0, 4, int((how == 2).sum())).astype(np.uint8)


def revive(recs, idx):
    recs["vendor"][idx] = 0x10DE
    recs["driver"][idx] = 1
    recs["flags"][idx] &= 0xF0
