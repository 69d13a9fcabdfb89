"""An exact numpy restatement of the re-scan delta (kvg_scan_pci_delta) on two PCI survivor lists, independent of
the kernels: the changes keyed by address and the dirty / gone keys of deviceMap and iommuMap."""
import numpy as np

CH_ADDED, CH_REMOVED, CH_GROUP, CH_DEVICE, CH_NUMA = 1, 2, 4, 8, 16


def _members_changed(pk, pa, pn, nk, na, nn):
    """Masks of the previous and the new members (key, addr, numa) that have no equal member on the other side."""
    cp = (pk.astype(np.uint64) << np.uint64(32)) | pa.astype(np.uint64)
    cn = (nk.astype(np.uint64) << np.uint64(32)) | na.astype(np.uint64)
    _, ip, jn = np.intersect1d(cp, cn, assume_unique=True, return_indices=True)
    bad_p = np.ones(len(cp), dtype=bool)
    bad_n = np.ones(len(cn), dtype=bool)
    same = pn[ip] == nn[jn]
    bad_p[ip] = ~same
    bad_n[jn] = ~same
    return bad_p, bad_n


def _key_lists(prev, now, field):
    """(dirty, gone) of one group-by map: dirty = indices into the new distinct keys whose (addr, numa) member
    sequence in Walk order differs (new keys included), gone = previous keys absent now."""
    pk, nk = prev[field].astype(np.int64), now[field].astype(np.int64)
    bad_p, bad_n = _members_changed(pk, prev["addr"], prev["numa"], nk, now["addr"], now["numa"])
    keys_now, keys_prev = np.unique(nk), np.unique(pk)
    touched = np.union1d(pk[bad_p], nk[bad_n])
    dirty = np.searchsorted(keys_now, np.intersect1d(touched, keys_now)).astype(np.uint32)
    return dirty, np.setdiff1d(keys_prev, keys_now)


def expect_pci_delta(prev, now, change_dtype):
    """The delta of two PCI survivor lists (PCI_SURV, strictly ascending addr), as kvgpu.h kvg_pci_delta
    states it: one change per address whose survivor differs (ascending), and the dirty / gone keys of deviceMap
    and iommuMap.  Returns a dict of changes / dev_dirty / dev_gone / grp_dirty / grp_gone."""
    pa, na = prev["addr"], now["addr"]
    u = np.union1d(pa, na).astype(np.uint32)
    ip = np.minimum(np.searchsorted(pa, u), max(len(pa) - 1, 0))
    jn = np.minimum(np.searchsorted(na, u), max(len(na) - 1, 0))
    inp = (pa[ip] == u) if len(pa) else np.zeros(len(u), dtype=bool)
    inn = (na[jn] == u) if len(na) else np.zeros(len(u), dtype=bool)
    what = np.zeros(len(u), dtype=np.uint32)
    what[inn & ~inp] = CH_ADDED
    what[inp & ~inn] = CH_REMOVED
    both = inp & inn
    P, N = prev[ip[both]], now[jn[both]]
    what[both] = ((P["iommu_group"] != N["iommu_group"]) * CH_GROUP | (P["device"] != N["device"]) * CH_DEVICE |
                  (P["numa"] != N["numa"]) * CH_NUMA).astype(np.uint32)
    sel = what != 0
    ch = np.zeros(int(sel.sum()), dtype=change_dtype)
    ch["addr"], ch["what"] = u[sel], what[sel]
    hp, hn = inp[sel], inn[sel]
    for side, has, idx, lst in (("prev", hp, ip[sel], prev), ("now", hn, jn[sel], now)):
        r = lst[idx[has]] if has.any() else lst[:0]
        ch[side + "_group"][has] = r["iommu_group"]
        ch[side + "_device"][has] = r["device"]
        ch[side + "_numa"][has] = r["numa"]
        ch[side + "_index"] = np.where(has, idx, 0xFFFFFFFF).astype(np.uint32)
    dev_dirty, dev_gone = _key_lists(prev, now, "device")
    grp_dirty, grp_gone = _key_lists(prev, now, "iommu_group")
    return dict(changes=ch, dev_dirty=dev_dirty, dev_gone=dev_gone.astype(np.uint16),
                grp_dirty=grp_dirty, grp_gone=grp_gone.astype(np.uint32))
