"""Dict-keyed restatement of kvg_health_rescan_mdev_keyed and kvg_health_rescan_groups_keyed (include/kvgpu.h),
independent of the kernels.  The rules are those of health_mdev_ref.step and health_groups_ref.step; only the prior
state of a record comes from a dict keyed by its UUID (big-endian bytes) or its address instead of from its index:

    prior_i = state[key_i] if key_i was in the previous call's list, else "nothing" (0)
    s_i     = the rule's next state from record i and prior_i; i is listed iff healthy(s_i) != healthy(prior_i)
    state   = {key_i: s_i}   (keys missing from this call are forgotten)

A call whose keys do not ascend strictly raises KeyError and leaves the state unchanged.
"""
from dataclasses import dataclass

import numpy as np

import health_groups_ref as HG
import health_mdev_ref as HM


@dataclass
class Delta:
    n_records: int
    n_alive: int
    changed: np.ndarray


def mdev_keys(recs):
    return [bytes(u) for u in np.asarray(recs["uuid"], dtype=np.uint8)]


def group_keys(recs):
    return [int(a) for a in recs["addr"]]


def _check_ascending(keys):
    for a, b in zip(keys, keys[1:]):
        if not a < b:
            raise KeyError("keys are not strictly ascending")


class KeyedMdevRef:
    """vGPUs: the state of a key is (p, m), present and marked."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.state = {}

    def rescan(self, recs, n_types, xid_parents=()) -> Delta:
        keys = mdev_keys(recs)
        _check_ascending(keys)
        prior = [self.state.get(k, (False, False)) for k in keys]
        p = np.array([s[0] for s in prior], dtype=bool)
        m = np.array([s[1] for s in prior], dtype=bool)
        changed, alive, p2, m2 = HM.step(recs, n_types, xid_parents, p, m)
        self.state = {k: (bool(a), bool(b)) for k, a, b in zip(keys, p2, m2)}
        return Delta(len(recs), alive, changed)

    def state_bytes(self, keys):
        """The kernels' state bytes of `keys` (bit 0 healthy, bit 1 marked); 0 for a key not in the list."""
        out = np.zeros(len(keys), dtype=np.uint8)
        for i, k in enumerate(keys):
            p, m = self.state.get(k, (False, False))
            out[i] = (1 if p and not m else 0) | (2 if p and m else 0)
        return out


class KeyedGroupsRef:
    """Passthrough GPUs by IOMMU group: the state of a key is the healthy bit."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.state = {}

    def rescan(self, recs, group_nodes=()) -> Delta:
        keys = group_keys(recs)
        _check_ascending(keys)
        h = np.array([self.state.get(k, False) for k in keys], dtype=bool)
        changed, alive, h2 = HG.step(recs, group_nodes, h)
        self.state = {k: bool(v) for k, v in zip(keys, h2)}
        return Delta(len(recs), alive, changed)

    def state_bytes(self, keys):
        return np.array([1 if self.state.get(k, False) else 0 for k in keys], dtype=np.uint8)
