"""Shared helpers for the test-suite: fixtures, synthetic sysfs trees, pci.ids text, exact numpy references."""
import gzip
import json
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def ginkgo():
    with open(os.path.join(GOLDEN, "ginkgo_vectors.json")) as f:
        return json.load(f)


def pciids_text() -> bytes:
    with gzip.open(os.path.join(GOLDEN, "pci.ids.gz"), "rb") as f:
        return f.read()


def pciids_names():
    with open(os.path.join(GOLDEN, "pciids_names.json")) as f:
        return json.load(f)


def make_pci_tree(root, entries, via_symlink=True):
    """Build <root>/devices/<addr> like the Ginkgo test does (device_plugin_test.go:281-301):
    every device entry is a SYMLINK to a real directory elsewhere, so filepath.Walk (Lstat) sees a
    non-directory and visits it.  entries: addr -> dict(vendor, device, driver, iommu_group,
    numa_node) where a missing/None value means "that sysfs read fails"."""
    base = os.path.join(root, "devices")
    real = os.path.join(root, "real")
    links = os.path.join(root, "targets")
    os.makedirs(base, exist_ok=True)
    os.makedirs(real, exist_ok=True)
    for addr, e in entries.items():
        d = os.path.join(real, addr) if via_symlink else os.path.join(base, addr)
        os.makedirs(d, exist_ok=True)
        for prop in ("vendor", "device"):
            if e.get(prop) is not None:
                v = e[prop]
                with open(os.path.join(d, prop), "w") as f:
                    f.write(v if v.startswith("0x") else "0x" + v + e.get("nl", "\n"))
        if e.get("numa_node") is not None:
            with open(os.path.join(d, "numa_node"), "w") as f:
                f.write(e["numa_node"])
        for link, sub in (("driver", "drivers"), ("iommu_group", "iommu_groups")):
            if e.get(link) is not None:
                tgt = os.path.join(links, sub, e[link])
                os.makedirs(tgt, exist_ok=True)
                os.symlink(tgt, os.path.join(d, link))
        if via_symlink:
            os.symlink(d, os.path.join(base, addr))
    return base


def make_mdev_tree(root, parents, mdevs):
    """<root>/mdev/<uuid> -> symlink to <root>/pci/<parent>/<uuid> (real dir holding
    mdev_type/name); <root>/pci/<parent>/numa_node.  mdevs: uuid -> dict(type, parent) with None
    meaning the read fails.  parents: bdf -> numa_node content or None."""
    pci = os.path.join(root, "pci")
    mdev = os.path.join(root, "mdev")
    os.makedirs(pci, exist_ok=True)
    os.makedirs(mdev, exist_ok=True)
    for p, numa in parents.items():
        os.makedirs(os.path.join(pci, p), exist_ok=True)
        if numa is not None:
            with open(os.path.join(pci, p, "numa_node"), "w") as f:
                f.write(numa)
    for uuid, e in mdevs.items():
        if e.get("parent") is not None:
            d = os.path.join(pci, e["parent"], uuid)
            os.makedirs(d, exist_ok=True)
            if e.get("type") is not None:
                os.makedirs(os.path.join(d, "mdev_type"), exist_ok=True)
                with open(os.path.join(d, "mdev_type", "name"), "w") as f:
                    f.write(e["type"])
            os.symlink(d, os.path.join(mdev, uuid))
        else:
            # a plain file: Readlink fails -> readGpuIDForVgpu error
            d = os.path.join(mdev, uuid)
            if e.get("type") is not None:
                os.makedirs(os.path.join(root, "orphans", uuid, "mdev_type"), exist_ok=True)
                with open(os.path.join(root, "orphans", uuid, "mdev_type", "name"), "w") as f:
                    f.write(e["type"])
            with open(d, "w") as f:
                f.write("")
    return mdev, pci


def c1_tree_entries():
    """BASELINE.json config 1: 8 vfio-pci Tesla P40 entries plus decoys (SURVEY.md 8d)."""
    ent = {}
    for k, bus in enumerate(["04", "05", "06", "07", "84", "85", "86", "87"]):
        ent["0000:%s:00.0" % bus] = dict(vendor="10de", device="1b38", driver="vfio-pci",
                                         iommu_group=str(40 + k),
                                         numa_node="0\n" if k < 4 else "1\n")
    ent["0000:01:00.0"] = dict(vendor="8086", device="1572", driver="i40e", iommu_group="3",
                               numa_node="0\n")
    ent["0000:08:00.0"] = dict(vendor="10de", device="1b38", driver="nvidia", iommu_group="48",
                               numa_node="0\n")
    ent["0000:04:00.1"] = dict(vendor="10de", device="10f0", driver="vfio-pci", iommu_group="40",
                               numa_node="-1\n")
    ent["0000:09:00.0"] = dict(vendor="10de", device="1b38", iommu_group="49", numa_node="0\n")
    return ent


# ------------------------------------------------------------------------------------------------
# exact numpy restatements of the scans (independent of the kernels; fast at tens of millions of records)
# ------------------------------------------------------------------------------------------------
def pci_alive(recs):
    """createIommuDeviceMap's drop rules (device_plugin.go:201-238) as a mask: dropped are records with any of
    the vendor / driver / iommu / device read errors (flags & 15), a vendor other than 10de, or a driver other
    than vfio-pci (1) or nvgrace (2)."""
    return ((recs["flags"] & 15) == 0) & (recs["vendor"] == 0x10DE) & ((recs["driver"] == 1) | (recs["driver"] == 2))


def expect_pci(recs):
    """The surviving records (pci_alive) in Walk order as a dict of addr / iommu_group / device / numa.  NUMA is
    0 when it could not be read (flags & 16) or is negative (device_plugin.go:227-230, :316-318)."""
    s = recs[pci_alive(recs)]
    numa = np.where(((s["flags"] & 16) != 0) | (s["numa"] < 0), 0, s["numa"]).astype(np.uint16)
    return dict(addr=s["addr"], iommu_group=s["iommu_group"], device=s["device"], numa=numa)


def check_ordering(values, keys, off, perm, what=""):
    """A stable ordering of `values`: distinct keys ascending, bucket offsets, and the stable permutation."""
    v = np.asarray(values).astype(np.int64)
    order = np.argsort(v, kind="stable")
    uk, first = np.unique(v[order], return_index=True)
    assert np.array_equal(np.asarray(keys).astype(np.int64), uk), what + ": keys"
    assert len(off) == len(uk) + 1, what + ": offsets length"
    assert np.array_equal(np.asarray(off[:-1]).astype(np.int64), first) and int(off[-1]) == len(v), what + ": offsets"
    assert np.array_equal(np.asarray(perm).astype(np.int64), order), what + ": permutation"


def check_pci_result(res, recs, names):
    """Compare a PciResult with the restatement in full.  `names`: Context.name_table() of the loaded
    pci.ids; name slots are offsets into the result's pool, so the join is compared through the names."""
    want = expect_pci(recs)
    s = res.survivors
    assert len(s) == len(want["addr"]), "survivor count %d, want %d" % (len(s), len(want["addr"]))
    for f in ("addr", "iommu_group", "device", "numa"):
        assert np.array_equal(s[f], want[f]), "survivors." + f
    check_ordering(want["device"], res.dev_keys, res.dev_off, res.dev_perm, "device ordering")
    check_ordering(want["iommu_group"], res.grp_keys, res.grp_off, res.grp_perm, "group ordering")
    got = [res.name_at(int(x)) for x in res.dev_name_slot]
    assert got == [names[int(k)] for k in res.dev_keys], "device-id names"
    # every survivor carries the slot of its device id (dev_keys are the distinct ids, checked above)
    assert np.array_equal(s["name_slot"], res.dev_name_slot[np.searchsorted(res.dev_keys, s["device"])]), \
        "survivor name slots"


def mdev_labels(raw_types):
    """The vGPU label of each raw mdev_type/name (device_plugin.go:341-342: Trim "\\n", then white-space runs
    to "_") and its canonical id: the index of the first equal label."""
    labels = [re.sub(rb"[\t\n\f\r ]+", b"_", t.strip(b"\n")) for t in raw_types]
    first = {}
    canon = [first.setdefault(lb, k) for k, lb in enumerate(labels)]
    return labels, np.array(canon, dtype=np.int64)


def expect_mdev(recs, raw_types):
    """createVgpuIDMap's classification (device_plugin.go:255-291): surviving mdevs in Walk order as a dict of
    uuid / parent / type_key / numa / src.  Dropped: a type or parent read error (flags & 3) or a type index
    outside the dictionary.  NUMA is 0 when it could not be read (flags & 4) or is negative."""
    _, canon = mdev_labels(raw_types)
    keep = ((recs["flags"] & 3) == 0) & (recs["type_idx"] < len(raw_types))
    r = recs[keep]
    numa = r["parent_numa"].astype(np.int32)
    numa[(numa < 0) | ((r["flags"] & 4) != 0)] = 0
    type_key = canon[r["type_idx"]] if len(r) else np.zeros(0, np.int64)
    return dict(uuid=r["uuid"], parent=r["parent"], type_key=type_key.astype(np.uint16),
                numa=numa.astype(np.uint16), src=np.nonzero(keep)[0].astype(np.uint32))


def check_mdev_result(res, recs, raw_types):
    """Compare an MdevResult with the restatement in full (survivors, both orderings, labels, canonical ids)."""
    want = expect_mdev(recs, raw_types)
    s = res.survivors
    assert len(s) == len(want["src"]), "survivor count %d, want %d" % (len(s), len(want["src"]))
    for f in ("uuid", "parent", "type_key", "numa", "src"):
        assert np.array_equal(s[f], want[f]), "survivors." + f
    check_ordering(want["type_key"], res.type_keys, res.type_off, res.type_perm, "type ordering")
    check_ordering(want["parent"], res.par_keys, res.par_off, res.par_perm, "parent ordering")
    labels, canon = mdev_labels(raw_types)
    assert res.labels == labels, "labels"
    assert np.array_equal(res.type_canon.astype(np.int64), canon), "canonical type ids"


# vGPU resource names longer than any fixed slot: a 10de section whose device lines carry sanitised names of
# these lengths (the last one near the 64 KiB line limit of bufio.Scanner)
LONG_NAME_LENGTHS = (255, 256, 257, 4096, 60_000)


def long_name_pciids() -> bytes:
    """A small pci.ids: another vendor, then 10de with device lines `\\tab0<k>  <name>` whose names sanitise to
    LONG_NAME_LENGTHS bytes, plus one short name, then a vendor after the section."""
    lines = [b"# long names", b"8086  Intel", b"\tab00  not this vendor", b"10de  NVIDIA Corporation"]
    for k, n in enumerate(LONG_NAME_LENGTHS):
        body = (b"gpu.%d/" % k + b"x" * n)[:n - 1] + b"z"    # '.' and '/' sanitise to '_': same length
        lines.append(b"\tab0%d  " % k + body)
        lines.append(b"\t\t10de %04x  a subsystem line" % k)
    lines += [b"\t1b38  GP102GL [Tesla P40]", b"10df  next vendor", b"\tab09  not this vendor", b""]
    return b"\n".join(lines)


def long_name_types() -> list:
    """vGPU type names that prefix-match the long device lines: exact ids, a shorter prefix (matches the first
    line, keeps the id's tail in the name), whitespace variants that merge, and labels that match nothing."""
    t = [b"ab0%d\n" % k for k in range(len(LONG_NAME_LENGTHS))]
    t += [b"ab\n", b"ab0\n\n", b"\nab04", b"ab03  ", b"1b38\n", b"GRID P40-1Q\n", b"GRID  P40-1Q\n", b"ab09\n"]
    return t
