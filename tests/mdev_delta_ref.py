"""An exact numpy restatement of the mdev re-scan delta (kvg_scan_mdev_delta) on two mdev survivor lists, independent
of the kernels: the changes keyed by UUID, with type identity by sanitised label, and the dirty / gone keys of vGpuMap
and gpuVgpuMap.  The PCI form is delta_ref.expect_pci_delta."""
import numpy as np

from delta_ref import CH_ADDED, CH_NUMA, CH_REMOVED  # noqa: F401  (the bits both deltas share)

CH_TYPE, CH_PARENT = 32, 64


def _uuid_words(s):
    """The UUID of each MDEV_SURV as two big-endian u64: (high, low) sort like the bytes."""
    w = np.ascontiguousarray(s["uuid"]).reshape(-1, 16).view(">u8").astype(np.uint64)
    return w[:, 0], w[:, 1]


def expect_mdev_delta(prev, now, prev_labels, now_labels, change_dtype):
    """The delta of two mdev survivor lists (MDEV_SURV, strictly ascending UUID bytes) as kvgpu.h kvg_mdev_delta
    states it.  prev_labels / now_labels: the sanitised label (bytes) of each canonical id of the two results'
    dictionaries (MdevResult.labels); a type is the same type in both iff its label is.  Returns a dict of
    changes / type_dirty / type_gone (labels) / par_dirty / par_gone."""
    ph, pl = _uuid_words(prev)
    nh, nl = _uuid_words(now)
    np_, nn = len(prev), len(now)
    hi, lo = np.concatenate([ph, nh]), np.concatenate([pl, nl])
    side = np.r_[np.zeros(np_, np.int64), np.ones(nn, np.int64)]
    order = np.lexsort((side, lo, hi))
    hs, ls, ss = hi[order], lo[order], side[order]
    idx = order - side[order] * np_
    start = np.r_[True, (hs[1:] != hs[:-1]) | (ls[1:] != ls[:-1])] if len(order) else np.zeros(0, bool)
    g = np.cumsum(start) - 1
    G = int(start.sum())
    pi, ni = np.full(G, -1, np.int64), np.full(G, -1, np.int64)
    pi[g[ss == 0]] = idx[ss == 0]
    ni[g[ss == 1]] = idx[ss == 1]
    inp, inn = pi >= 0, ni >= 0
    # label identity: one integer per distinct label over both dictionaries
    lid_of = {}
    plid = np.array([lid_of.setdefault(bytes(b), len(lid_of)) for b in prev_labels] + [0], np.int64)
    nlid = np.array([lid_of.setdefault(bytes(b), len(lid_of)) for b in now_labels] + [0], np.int64)
    p_lab = plid[prev["type_key"].astype(np.int64)] if np_ else np.zeros(0, np.int64)
    n_lab = nlid[now["type_key"].astype(np.int64)] if nn else np.zeros(0, np.int64)

    what = np.zeros(G, np.uint32)
    what[inn & ~inp] = CH_ADDED
    what[inp & ~inn] = CH_REMOVED
    both = inp & inn
    a, b = pi[both], ni[both]
    what[both] = ((p_lab[a] != n_lab[b]) * CH_TYPE | (prev["parent"][a] != now["parent"][b]) * CH_PARENT |
                  (prev["numa"][a] != now["numa"][b]) * CH_NUMA).astype(np.uint32)
    sel = what != 0
    ch = np.zeros(int(sel.sum()), dtype=change_dtype)
    ch["what"] = what[sel]
    hp, hn = inp[sel], inn[sel]
    for side_name, has, ix, lst in (("prev", hp, pi[sel], prev), ("now", hn, ni[sel], now)):
        r = lst[ix[has]]
        ch["uuid"][has] = r["uuid"]
        ch[side_name + "_parent"][has] = r["parent"]
        ch[side_name + "_type"][has] = r["type_key"]
        ch[side_name + "_numa"][has] = r["numa"]
        ch[side_name + "_index"] = np.where(has, ix, 0xFFFFFFFF).astype(np.uint32)

    # members with no equal member on the other side: vGpuMap compares (label, uuid, numa), gpuVgpuMap (parent, uuid)
    bad_pt, bad_nt = np.ones(np_, bool), np.ones(nn, bool)
    bad_pp, bad_np = np.ones(np_, bool), np.ones(nn, bool)
    same_t = (p_lab[a] == n_lab[b]) & (prev["numa"][a] == now["numa"][b])
    same_p = prev["parent"][a] == now["parent"][b]
    bad_pt[a], bad_nt[b] = ~same_t, ~same_t
    bad_pp[a], bad_np[b] = ~same_p, ~same_p

    keys_now = np.unique(now["type_key"])
    keys_prev = np.unique(prev["type_key"])
    touched = set(p_lab[bad_pt].tolist()) | set(n_lab[bad_nt].tolist())
    now_key_lab = nlid[keys_now.astype(np.int64)]
    type_dirty = np.nonzero(np.isin(now_key_lab, list(touched)))[0].astype(np.uint32)
    live = set(now_key_lab.tolist())
    type_gone = [bytes(prev_labels[int(c)]) for c in keys_prev if plid[int(c)] not in live]

    pk, nk = prev["parent"].astype(np.int64), now["parent"].astype(np.int64)
    par_now, par_prev = np.unique(nk), np.unique(pk)
    ptouched = np.union1d(pk[bad_pp], nk[bad_np])
    par_dirty = np.searchsorted(par_now, np.intersect1d(ptouched, par_now)).astype(np.uint32)
    par_gone = np.setdiff1d(par_prev, par_now).astype(np.uint32)
    return dict(changes=ch, type_dirty=type_dirty, type_gone=type_gone, par_dirty=par_dirty, par_gone=par_gone)
