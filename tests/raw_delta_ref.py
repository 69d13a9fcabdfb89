"""A string-level restatement of kvg_scan_pci_raw_delta, independent of the kernels: both sides' entry names, group
strings and device strings go into one sorted space, delta_ref.expect_pci_delta applies the delta's rules there, and
the answer is mapped back to each side's own encoding (address, group and device handles).

A side is a dict of its survivors in Walk order: names / groups / devices (lists of bytes), numa (clamped), and the
side's own encoding of each: addr, grp, dev (handles as the snapshot has them), plus dev_keys / grp_keys (the
result's distinct handles, ascending)."""
import numpy as np

import kvgpu
import delta_ref

NO_INDEX = 0xFFFFFFFF


def side_of(res, snap):
    """A side from a PciResult and its PciSnapshot: the strings behind every survivor's handles."""
    s = res.survivors
    if snap.packed_addr:
        names = [kvgpu.format_bdf(int(a)).encode() for a in s["addr"]]
    else:
        names = [snap.names[int(a)].encode("latin-1") if isinstance(snap.names[int(a)], str) else snap.names[int(a)]
                 for a in s["addr"]]
    groups = [str(int(g)).encode() if snap.group_names is None else snap.group_names[int(g)].encode("latin-1")
              for g in s["iommu_group"]]
    devices = ["%04x" % int(d) for d in s["device"]] if snap.device_names is None else \
        [snap.device_names[int(d)] for d in s["device"]]
    return dict(names=names, groups=groups, devices=[d.encode("latin-1") for d in devices],
                numa=s["numa"].astype(np.uint16), addr=s["addr"].astype(np.uint32),
                grp=s["iommu_group"].astype(np.uint32), dev=s["device"].astype(np.uint32),
                dev_keys=np.asarray(res.dev_keys, dtype=np.uint32), grp_keys=np.asarray(res.grp_keys, dtype=np.uint32))


def empty_side():
    """the previous side of a first call or a call after a reset"""
    z = np.zeros(0, np.uint32)
    return dict(names=[], groups=[], devices=[], numa=z.astype(np.uint16), addr=z, grp=z, dev=z, dev_keys=z,
                grp_keys=z)


def expect(prev, now):
    """The delta of two sides (names strictly ascending on both), as kvgpu.h kvg_scan_pci_raw_delta states it."""
    space = {}
    for col in ("names", "groups", "devices"):
        u = sorted(set(prev[col]) | set(now[col]))
        space[col] = {v: k for k, v in enumerate(u)}

    def common(side):
        s = np.zeros(len(side["names"]), dtype=kvgpu.PCI_SURV)
        s["addr"] = [space["names"][v] for v in side["names"]]
        s["iommu_group"] = [space["groups"][v] for v in side["groups"]]
        s["device"] = [space["devices"][v] for v in side["devices"]]
        s["numa"] = side["numa"]
        return s

    assert len(space["devices"]) < 65536
    P, N = common(prev), common(now)
    want = delta_ref.expect_pci_delta(P, N, kvgpu.PCI_CHANGE)
    ch = want["changes"]
    out = np.zeros(len(ch), dtype=kvgpu.PCI_CHANGE)
    out["what"] = ch["what"]
    out["prev_index"], out["now_index"] = ch["prev_index"], ch["now_index"]
    out["prev_numa"], out["now_numa"] = ch["prev_numa"], ch["now_numa"]
    hp, hn = ch["prev_index"] != NO_INDEX, ch["now_index"] != NO_INDEX
    for tag, has, side in (("prev", hp, prev), ("now", hn, now)):
        idx = ch[tag + "_index"][has]
        out[tag + "_group"][has] = side["grp"][idx]
        out[tag + "_device"][has] = side["dev"][idx]
    out["addr"] = np.where(hn, now["addr"][np.where(hn, ch["now_index"], 0)] if len(now["addr"]) else 0,
                           prev["addr"][np.where(hp, ch["prev_index"], 0)] if len(prev["addr"]) else 0)

    def back(col, handles, field, dirty, gone):
        """dirty: indices into the new common keys -> indices into the new side's keys; gone: common -> previous
        handles, ascending"""
        to_now = {space[col][v]: int(h) for v, h in zip(now[col], now[handles])}
        to_prev = {space[col][v]: int(h) for v, h in zip(prev[col], prev[handles])}
        keys_common = np.unique(N[field])
        nk = now[handles + "_keys"]
        d = np.sort(np.searchsorted(nk, [to_now[int(keys_common[i])] for i in dirty])).astype(np.uint32)
        g = np.sort(np.array([to_prev[int(c)] for c in gone], dtype=np.uint32))
        return d, g

    dev_dirty, dev_gone = back("devices", "dev", "device", want["dev_dirty"], want["dev_gone"])
    grp_dirty, grp_gone = back("groups", "grp", "iommu_group", want["grp_dirty"], want["grp_gone"])
    return dict(changes=out, dev_dirty=dev_dirty, dev_gone=dev_gone.astype(np.uint16), grp_dirty=grp_dirty,
                grp_gone=grp_gone)
