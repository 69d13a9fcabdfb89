"""A Go-exact restatement of kvg_pci_allocate_response (include/kvgpu.h) over raw reads, and the named edge matrix its
tests share.

The rules restated, from generic_device_plugin.go:352-444 and :702-716: per visited DevicesID its members in map
order, each re-checked (allocate_raw_cases.member), then dev.addr == bdf, then readVFIODev (os.ReadDir sorts names as
bytes; the first entry whose DirEntry.IsDir(), links not followed, and whose name has the prefix "vfio"); the ID's
"not found" after its members; the specs through appendDeviceSpec with filepath.Join's cleaning; envList outliving
the request loop; the EGM rule of allocate_raw_cases.  A request is (ids, visits, lookup_error), visits = per visited
ID [(addr, link, vendor, group, listing)], a listing [(name, is_dir)], None (failed) or NOT_READ."""
import posixpath

import allocate_raw_cases as AR
from kvgpu import NOT_READ

OK, UNKNOWN_ID, UNKNOWN_MEMBER, PANIC, VFIO_READ, VFIO_NONE = range(6)   # KVG_ARESP_*


def _egm(egm_entries):
    """discoverEGMDevicesFunc: the kept fields per entry, raising the lowest missing read; the key cap's entry"""
    kept, keys, order = [], {}, []
    for e, (name, gpus, stat) in enumerate(egm_entries):
        fs, miss = AR.egm_entry(name, gpus, stat)
        if miss:
            raise AR.RawError("miss", ("egm", e, miss))
        kept.append(fs)
        for f in fs or []:
            if AR.key(f) not in keys:
                keys[AR.key(f)] = len(keys)
                order.append(e)
    return kept, (order[AR.MAX_EGM_KEYS] if len(keys) > AR.MAX_EGM_KEYS else None)


def _request(ids, visits, lookup_error, iommufd):
    """one request in the reference's order -> (kind, at, paths, listing miss position or None)"""
    specs, seen, p = [], set(), 0

    def append(path):
        if path not in seen:
            seen.add(path)
            specs.append(path)
    for k, visit in enumerate(visits):
        found = False
        for addr, link, vendor, group, listing in visit:
            v = AR.member(link, vendor, group)
            if v != AR.PASS:
                return (PANIC if v == AR.PANIC else UNKNOWN_MEMBER), p, [], None
            found = found or addr == ids[k]
            if iommufd:
                if listing is NOT_READ:
                    return None, p, [], p
                if listing is None:
                    return VFIO_READ, p, [], None
                names = sorted(n for n, d in listing if d and n.startswith(b"vfio"))
                if not names:
                    return VFIO_NONE, p, [], None
                append(b"/dev/vfio/devices/" + names[0])
            p += 1
        if not found:
            return UNKNOWN_ID, k, [], None
        append(b"/dev/vfio/vfio")
        append(posixpath.normpath(b"/dev/vfio/" + visit[0][3]))   # filepath.Join cleans: "", ".", ".."
        if iommufd:
            append(b"/dev/iommu")
    if lookup_error:
        return UNKNOWN_ID, len(visits), [], None
    return OK, 0, specs, None


def allocate_response(requests, egm_entries, iommufd):
    """-> [(kind, at, paths, env or None)] as Context.pci_allocate_response returns them, or raises AR.RawError:
    "group" / "order" (the plan's group strings, the EGM names' order), then "miss" (EGM first, then request by
    request the raw member miss or a reached listing not made), then "range"."""
    i = 0
    for ids, visits, _ in requests:
        for visit in visits:
            for _, _, _, group, _ in visit:
                if group != visit[0][3] or b"/" in group:
                    raise AR.RawError("group", i)
                i += 1
    names = [e[0] for e in egm_entries]
    for e in range(1, len(names)):
        if not names[e - 1] < names[e]:
            raise AR.RawError("order", e)
    kept, range_at = _egm(egm_entries)
    out, addrs, n_vis = [], [], 0
    for r, (ids, visits, lookup_error) in enumerate(requests):
        members = [m for visit in visits for m in visit]
        for p, m in enumerate(members):
            v = AR.member(*m[1:4])
            if v == AR.MISS:
                raise AR.RawError("miss", ("member", r, p))
            if v != AR.PASS:
                break
        kind, at, paths, miss = _request(ids, visits, lookup_error, iommufd)
        if miss is not None:
            raise AR.RawError("miss", ("listing", r, miss))
        if kind == OK:
            have = {AR.key(x) for x in ids}
            paths += [b"/dev/" + egm_entries[e][0] for e, fs in enumerate(kept)
                      if fs is not None and all(AR.key(f) in have for f in fs)]
        addrs += [m[0] for m in members]
        n_vis += len(visits)
        out.append((kind, at, paths, b",".join(addrs) if n_vis else None))
    if range_at is not None:
        raise AR.RawError("range", ("egm", range_at))
    return out


# ---- the named edge matrix --------------------------------------------------------------------------------------
G = b"42"
A = [b"0000:01:00.0", b"0000:01:00.1", b"0000:02:00.0", b"0000:03:00.0"]
DIR = [(b"vfio3", True)]


def mem(addr, group=G, listing=DIR, link=None, vendor=b"0x10de\n"):
    return (addr, link if link is not None else b"../../../kernel/iommu_groups/" + group, vendor, group, listing)


def one(visits, ids=None, lookup_error=False):
    """one request visiting `visits`, its IDs the first member of each visit unless given"""
    return (ids if ids is not None else [v[0][0] for v in visits], visits, lookup_error)


def edge_calls():
    """[(name, requests, egm, iommufd)] of the matrix, each also run with iommufd off"""
    egm = [(b"egm0", b"0000:01:00.0\n", True), (b"egm\x80", b"0000:01:00.0 0000:01:00.1", True),
           (b"egm\xff", b"0000:02:00.0", True)]
    L = lambda *e: list(e)   # noqa: E731
    cases = [
        ("plain", [one([[mem(A[0])]])], []),
        ("vfio10_before_vfio3", [one([[mem(A[0], listing=L((b"vfio3", True), (b"vfio10", True)))]])], []),
        ("file_before_dir", [one([[mem(A[0], listing=L((b"vfio0", False), (b"vfio1", True)))]])], []),
        ("symlink_to_dir", [one([[mem(A[0], listing=L((b"vfio0", False), (b"vfio7", True)))]])], []),
        ("symlink_only", [one([[mem(A[0], listing=L((b"vfio0", False)))]])], []),
        ("upper_and_short", [one([[mem(A[0], listing=L((b"VFIO3", True), (b"vfi", True), (b"vfio", True)))]])], []),
        ("empty_listing", [one([[mem(A[0], listing=[])]])], []),
        ("failed_listing", [one([[mem(A[0], listing=None)]])], []),
        ("unreached_missing", [one([[mem(A[0], vendor=b"0x8086\n", listing=NOT_READ)]])], []),
        ("unreached_after_error", [one([[mem(A[0], listing=[]), mem(A[1], listing=NOT_READ)]])], []),
        ("group_vfio", [one([[mem(A[0], group=b"vfio")]])], []),
        ("group_empty", [one([[mem(A[0], group=b"", link=b"../")]])], []),
        ("group_dot", [one([[mem(A[0], group=b".")]])], []),
        ("group_dotdot", [one([[mem(A[0], group=b"..")]])], []),
        ("group_042_vs_42", [one([[mem(A[0], group=b"042")], [mem(A[2])]])], []),
        ("id_twice", [one([[mem(A[0]), mem(A[1], listing=L((b"vfio4", True)))]] * 2, ids=[A[0], A[0]])], []),
        ("two_ids_one_group", [one([[mem(A[0]), mem(A[1], listing=L((b"vfio4", True)))]] * 2, ids=[A[0], A[1]])],
         []),
        ("id_absent", [one([[mem(A[1]), mem(A[2])]], ids=[A[0]])], []),
        ("id_absent_vs_vfio_none", [one([[mem(A[1]), mem(A[2], listing=[])]], ids=[A[0]])], []),
        ("lookup_after_visits", [one([[mem(A[0])]], ids=[A[0], b"nope"], lookup_error=True)], []),
        ("lookup_first", [one([], ids=[b"nope"], lookup_error=True)], []),
        ("panic_before_listing_error", [one([[mem(A[0], vendor=b"x"), mem(A[1], listing=None)]])], []),
        ("env_empty_then_full", [one([], ids=[]), one([[mem(A[0])]])], []),
        ("env_full_then_empty", [one([[mem(A[0])]]), one([], ids=[])], []),
        ("three_requests", [one([[mem(A[0])]]), one([[mem(A[2], listing=L((b"vfio9", True)))]]),
                            one([[mem(A[3])]])], egm),
        ("egm_high_bytes", [one([[mem(A[0]), mem(A[1])]] * 2, ids=[A[0], A[1]]), one([[mem(A[2])]])], egm),
    ]
    return [(n, r, e, f) for n, r, e in cases for f in (True, False)]


def edge_refusals():
    """[(name, requests, egm, iommufd)] that must be refused"""
    return [
        ("listing_not_made", [one([[mem(A[0], listing=NOT_READ)]])], [], True),
        ("listing_not_made_second_request", [one([[mem(A[0])]]), one([[mem(A[2], listing=NOT_READ)]])], [], True),
        ("group_differs", [one([[mem(A[0]), mem(A[1], group=b"43")]])], [], False),
        ("group_slash", [one([[mem(A[0], group=b"4/2")]])], [], True),
        ("egm_order", [one([[mem(A[0])]])], [(b"egm1", b"x", True), (b"egm0", b"x", True)], True),
        ("egm_twice", [one([[mem(A[0])]])], [(b"egm1", b"x", True), (b"egm1", b"x", True)], False),
        ("member_not_made", [one([[mem(A[0], vendor=NOT_READ)]])], [], True),
    ]


def random_call(rng, n_reqs=None):
    """a seeded call mixing every case: (requests, egm, iommufd)"""
    n_reqs = int(rng.integers(0, 5)) if n_reqs is None else n_reqs
    names = [b"vfio0", b"vfio1", b"vfio10", b"vfio3", b"VFIO2", b"vfi", b"vfio", b"x", b"vfio\xff"]
    groups = [G, b"43", b"vfio", b"", b".", b"..", b"042"]
    bdfs = A + [b"0000:04:00.0", b"0000:04:00.1"]
    reqs = []
    for _ in range(n_reqs):
        visits, ids = [], []
        for _ in range(int(rng.integers(0, 4))):
            g = groups[rng.integers(len(groups))]
            visit = []
            for _ in range(int(rng.integers(1, 4))):
                listing = [(names[k], bool(rng.random() < 0.7)) for k in rng.integers(0, len(names),
                                                                                     size=int(rng.integers(0, 4)))]
                u = rng.random()
                if u < 0.04:
                    listing = None
                elif u < 0.06:
                    listing = []
                link = b"../" + g if rng.random() < 0.93 else b"../zz"
                vendor = b"0x10de\n" if rng.random() < 0.95 else [b"x", None, b"0x8086"][rng.integers(3)]
                visit.append((bdfs[rng.integers(len(bdfs))], link, vendor, g, listing))
            visits.append(visit)
            ids.append(visit[rng.integers(len(visit))][0] if rng.random() < 0.9 else bdfs[rng.integers(len(bdfs))])
        lookup = rng.random() < 0.1
        if lookup:
            ids.append(b"nope")
        reqs.append((ids, visits, lookup))
    egm = []
    for e in range(int(rng.integers(0, 4))):
        gpus = b" ".join(bdfs[k] for k in rng.integers(0, len(bdfs), size=int(rng.integers(1, 3))))
        egm.append((b"egm%d" % e, gpus, bool(rng.random() < 0.9)))
    return reqs, egm, bool(rng.random() < 0.7)
