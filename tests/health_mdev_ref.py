"""numpy restatement of kvg_health_rescan_mdev (include/kvgpu.h): the vGPU health state machine, independent of the
kernels.

Record i carries two bits from the previous tick, p (present) and m (marked), m => p.  With X the tick's XID parent
handles:

    p' = createVgpuIDMap's keep rule (no type / parent read error, type index inside the dictionary)
    m' = p' & (parent in X | (p & m))
    h = p & ~m, h' = p' & ~m';  i is listed iff h' != h, as (i << 1) | h'
"""
from dataclasses import dataclass

import numpy as np


def mdev_present(recs, n_types):
    return ((recs["flags"] & 3) == 0) & (recs["type_idx"].astype(np.int64) < n_types)


def step(recs, n_types, xid_parents, p, m):
    """One tick: -> (changed words, n_alive, p', m')."""
    now_p = mdev_present(recs, n_types)
    x = np.unique(np.asarray(xid_parents, dtype=np.uint32))
    now_m = now_p & (np.isin(recs["parent"], x) | (p & m))
    h, now_h = p & ~m, now_p & ~now_m
    idx = np.nonzero(h != now_h)[0]
    changed = (idx.astype(np.uint32) << 1) | now_h[idx].astype(np.uint32)
    return changed, int(now_h.sum()), now_p, now_m


@dataclass
class Delta:
    n_records: int
    n_alive: int
    changed: np.ndarray


class HealthMdevRef:
    """The per-context state of kvg_health_rescan_mdev: a different n re-arms it, as does reset()."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.p = self.m = np.zeros(0, dtype=bool)

    def rescan(self, recs, n_types, xid_parents=()) -> Delta:
        n = len(recs)
        if n != len(self.p):
            self.p = np.zeros(n, dtype=bool)
            self.m = np.zeros(n, dtype=bool)
        changed, alive, self.p, self.m = step(recs, n_types, xid_parents, self.p, self.m)
        return Delta(n, alive, changed)

    def state_bytes(self):
        """The state as the kernels keep it: bit 0 healthy (p and not m), bit 1 marked (p and m)."""
        return (self.p & ~self.m).astype(np.uint8) | ((self.p & self.m).astype(np.uint8) << 1)
