"""A Go-exact restatement of kvg_pci_allocate_raw (include/kvgpu.h) and the named edge matrix its tests share.

The rules restated, from generic_device_plugin.go and device_plugin.go:
  member     readLinkFunc (filepath.Split of os.Readlink) compared with bdfToIommu[bdf] as strings, then
             readIDFromFileFunc (data[2:], Trim "\\n") compared with "10de" (:387-399)
  EGM entry  discoverEGMDevicesFunc (:120-157): the "egm" prefix, the gpu_devices read, strings.Fields, the Stat
  keys       egmPathsForAllocatedGPUs (:159-184): strings.ToLower(strings.TrimSpace(s))
utf8.DecodeRune / DecodeLastRune, unicode.IsSpace and unicode.ToLower are written out here from the Go definitions;
ToLower is built from unicodedata, independently of tools/gen_case_table.py.  A read is bytes, None (failed) or
kvgpu.NOT_READ; a stat is True, False or NOT_READ (kvgpu.pack_alloc_raw's convention)."""
import unicodedata

import numpy as np

from kvgpu import NOT_READ

RUNE_ERROR = 0xFFFD
SPACE = {0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0, 0x1680, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000,
         *range(0x2000, 0x200B)}
MAX_EGM_KEYS = 65535


def go_lower(r: int) -> int:
    """unicode.ToLower: the simple mapping; U+0130's is U+0069 (Python's full mapping has two code points)."""
    if r == 0x130:
        return 0x69
    if 0xD800 <= r <= 0xDFFF:
        return r
    low = chr(r).lower()
    return ord(low) if len(low) == 1 else r


_LOWER = {}


def lower(r: int) -> int:
    if r not in _LOWER:
        _LOWER[r] = go_lower(r)
    return _LOWER[r]


def decode_rune(b: bytes, i: int):
    """utf8.DecodeRune(b[i:]) -> (rune, width)"""
    n = len(b) - i
    if n <= 0:
        return RUNE_ERROR, 0
    c = b[i]
    if c < 0x80:
        return c, 1
    if 0xC2 <= c <= 0xDF:
        need, lo, hi, r = 1, 0x80, 0xBF, c & 0x1F
    elif 0xE0 <= c <= 0xEF:
        need, lo, hi, r = 2, 0xA0 if c == 0xE0 else 0x80, 0x9F if c == 0xED else 0xBF, c & 0x0F
    elif 0xF0 <= c <= 0xF4:
        need, lo, hi, r = 3, 0x90 if c == 0xF0 else 0x80, 0x8F if c == 0xF4 else 0xBF, c & 0x07
    else:
        return RUNE_ERROR, 1
    if n < need + 1 or not lo <= b[i + 1] <= hi:
        return RUNE_ERROR, 1
    r = (r << 6) | (b[i + 1] & 0x3F)
    for k in range(2, need + 1):
        if b[i + k] & 0xC0 != 0x80:
            return RUNE_ERROR, 1
        r = (r << 6) | (b[i + k] & 0x3F)
    return r, need + 1


def decode_last_rune(b: bytes):
    """utf8.DecodeLastRune(b) -> (rune, width)"""
    end = len(b)
    if end == 0:
        return RUNE_ERROR, 0
    if b[end - 1] < 0x80:
        return b[end - 1], 1
    lim, start = max(end - 4, 0), end - 1
    start -= 1
    while start >= lim and b[start] & 0xC0 == 0x80:
        start -= 1
    start = max(start, 0)
    r, w = decode_rune(b[:end], start)
    return (r, w) if start + w == end else (RUNE_ERROR, 1)


def runes(b: bytes) -> list:
    out, i = [], 0
    while i < len(b):
        r, w = decode_rune(b, i)
        out.append(r)
        i += w
    return out


def trim_space(b: bytes) -> bytes:
    """strings.TrimSpace"""
    i = 0
    while i < len(b):
        r, w = decode_rune(b, i)
        if r not in SPACE:
            break
        i += w
    b = b[i:]
    while b:
        r, w = decode_last_rune(b)
        if r not in SPACE:
            break
        b = b[:-w]
    return b


def fields(b: bytes) -> list:
    """strings.Fields (unicode.IsSpace over UTF-8; an invalid byte is RuneError, not a space)"""
    out, i, start = [], 0, None
    while i < len(b):
        r, w = decode_rune(b, i)
        if r in SPACE:
            if start is not None:
                out.append(b[start:i])
                start = None
        elif start is None:
            start = i
        i += w
    if start is not None:
        out.append(b[start:])
    return out


def key(b: bytes) -> tuple:
    """strings.ToLower(strings.TrimSpace(s)) as its runes (each invalid byte U+FFFD)"""
    return tuple(lower(r) for r in runes(trim_space(b)))


class RawError(Exception):
    """A refusal: kind "miss" (KVG_EINVAL) or "range" (KVG_ERANGE), and where."""

    def __init__(self, kind, where):
        super().__init__("%s at %s" % (kind, where))
        self.kind, self.where = kind, where


PASS, FAIL, PANIC, MISS = "pass", "fail", "panic", "miss"


def member(link, vendor, group) -> str:
    """:387-399 for one member"""
    if link is NOT_READ:
        return MISS
    if link is None or link.rsplit(b"/", 1)[-1] != group:
        return FAIL
    if vendor is NOT_READ:
        return MISS
    if vendor is None:
        return FAIL
    if len(vendor) < 2:
        return PANIC
    return PASS if vendor[2:].strip(b"\n") == b"10de" else FAIL


def egm_entry(name, gpus, stat):
    """discoverEGMDevicesFunc for one entry -> (kept fields or None, the missing read or None)"""
    if not name.startswith(b"egm"):
        return None, None
    if gpus is NOT_READ:
        return None, "gpu_devices"
    if gpus is None:
        return None, None
    fs = fields(gpus)
    if not fs:
        return None, None
    if stat is NOT_READ:
        return None, "stat"
    return (fs if stat else None), None


def allocate_raw(requests, egm_entries):
    """requests: [(members, ids)], members = [(link, vendor, group)]; egm_entries: [(name, gpu_devices, stat)].
    -> (first_bad, panic, kept, take) as Context.pci_allocate_raw returns them, or raises RawError."""
    kept, keys, order = [], {}, []
    for e, (name, gpus, stat) in enumerate(egm_entries):
        fs, miss = egm_entry(name, gpus, stat)
        if miss:
            raise RawError("miss", ("egm", e, miss))
        kept.append(fs)
        for f in fs or []:
            if key(f) not in keys:
                keys[key(f)] = len(keys)
                order.append(e)
    first_bad, panic = [], []
    for r, (members, ids) in enumerate(requests):
        bad, p = len(members), False
        for i, m in enumerate(members):
            v = member(*m)
            if v == MISS:
                raise RawError("miss", ("member", r, i))
            if v != PASS:
                bad, p = i, v == PANIC
                break
        first_bad.append(bad)
        panic.append(p)
    if len(keys) > MAX_EGM_KEYS:
        raise RawError("range", ("egm", order[MAX_EGM_KEYS]))
    take = np.zeros((len(requests), len(egm_entries)), dtype=bool)
    for r, (_, ids) in enumerate(requests):
        have = {key(x) for x in ids}
        for e, fs in enumerate(kept):
            take[r, e] = fs is not None and all(key(f) in have for f in fs)
    return (np.array(first_bad, dtype=np.uint32), np.array(panic, dtype=bool), np.array([k is not None for k in kept],
            dtype=bool), take)


def egm_paths(egm_entries, kept, take_r) -> list:
    """the mounts of one request: /dev/<name> of the kept and taken entries, sorted"""
    return ["/dev/" + n.decode("utf-8", "surrogateescape")
            for n in sorted(e[0] for e, k, t in zip(egm_entries, kept, take_r) if k and t)]


# ---- the named edge matrix --------------------------------------------------------------------------------------
G = b"42"
LINK_OK = b"../../../kernel/iommu_groups/42"
VENDORS = {"empty": b"", "x": b"x", "0x": b"0x", "0x10de": b"0x10de", "0x10de_nl": b"0x10de\n\n",
           "0x10DE": b"0x10DE", "failed": None, "0x10de\\n": b"0x10de\n", "nl_0x10de": b"\n\n10de"}
LINKS = {"path": LINK_OK, "bare": b"42", "trailing_slash": LINK_OK + b"/", "zero_padded": b"../iommu_groups/042",
         "failed": None, "other": b"../iommu_groups/43", "nl": b"../iommu_groups/42\n"}
BDF = [b"0000:01:00.0", b"0000:02:00.0", b"0000:03:00.0", b"0000:04:00.0"]
GPU_DEVICES = {
    "x1c": b"0000:01:00.0\x1c0000:02:00.0",
    "raw_x85": b"0000:01:00.0\x850000:02:00.0",
    "u0085": b"0000:01:00.0\xc2\x850000:02:00.0",
    "nbsp": b"0000:01:00.0\xc2\xa00000:02:00.0",
    "ideographic": b"0000:01:00.0\xe3\x80\x800000:02:00.0\n",
    "invalid": b"0000:01:00.0\xe2\x82 0000:02:00.0",
    "kelvin": b"0000:01:00.0 \xe2\x84\xaa",
    "dotted_i": b"\xc4\xb0d 0000:02:00.0",
    "upper": b"0000:0A:00.0\n0000:02:00.0\n",
    "whitespace": b" \n\t\xe3\x80\x80 ",
    "ff": b"\xff",
    "plain": b"0000:01:00.0\n0000:02:00.0\n",
    "one": b"0000:03:00.0\n",
}
IDS = [b"0000:01:00.0", b" 0000:02:00.0\n", b"k", b"id", b"\xfe", b"0000:0a:00.0", b"0000:01:00.0\x1c0000:02:00.0",
       b"0000:01:00.0\xc2\x850000:02:00.0"]


def ok_member(group=G):
    return (LINK_OK, b"0x10de\n", group)


def edge_requests():
    """[(name, requests)] of the member matrix: one request per link / vendor case behind a passing member, and the
    precedence cases"""
    out = []
    for k, v in VENDORS.items():
        out.append(("vendor_" + k, [([ok_member(), (LINK_OK, v, G)], [BDF[0]])]))
    for k, v in LINKS.items():
        out.append(("link_" + k, [([ok_member(), (v, b"0x10de\n", G)], [BDF[0]])]))
    out.append(("panic_behind_failure", [([ok_member(), (LINK_OK, b"0x8086", G), (LINK_OK, b"x", G)], [])]))
    out.append(("panic_behind_failed_link", [([(None, b"x", G), ok_member()], [])]))
    out.append(("panic_behind_moved_link", [([(b"../43", b"x", G)], [])]))
    out.append(("later_request_panics", [([(LINK_OK, None, G)], []), ([(LINK_OK, b"", G)], []), ([ok_member()], [])]))
    out.append(("unreached_not_made", [([(None, NOT_READ, G), (NOT_READ, NOT_READ, G)], []),
                                       ([(b"../41", NOT_READ, G)], [])]))
    out.append(("empty_requests", [([], []), ([], [BDF[0]]), ([ok_member()], [])]))
    return out


def edge_refusals():
    """[(name, requests, egm)] that must be refused: reached reads that were not made"""
    return [
        ("link_not_made", [([ok_member(), (NOT_READ, b"0x10de", G)], [])], []),
        ("vendor_not_made", [([(LINK_OK, NOT_READ, G)], [])], []),
        ("second_request", [([ok_member()], []), ([ok_member(), (LINK_OK, NOT_READ, G)], [])], []),
        ("gpu_devices_not_made", [([ok_member()], [])], [(b"egm0", b"0000:01:00.0", True), (b"egm1", NOT_READ, True)]),
        ("stat_not_made", [], [(b"egm0", b"0000:01:00.0", NOT_READ)]),
        ("egm_before_members", [([(LINK_OK, NOT_READ, G)], [])], [(b"egm3", b"a", NOT_READ)]),
    ]


def edge_egm():
    """EGM class entries covering every gpu_devices case, failed reads, missing nodes and non-egm names"""
    out = [(b"egm_" + k.encode(), v, True) for k, v in GPU_DEVICES.items()]
    out += [(b"egm_failed", None, True), (b"egm_nonode", b"0000:01:00.0", False), (b"gpu0", NOT_READ, NOT_READ),
            (b"eg", b"0000:01:00.0", True), (b"Egm1", b"0000:01:00.0", True), (b"egm_notread_nofields", b" ", NOT_READ),
            (b"egm", b"0000:03:00.0", True)]
    return out


def edge_id_sets():
    """DevicesID lists, one request each, that take different subsets of edge_egm()"""
    return [[], [BDF[0]], [BDF[0], BDF[1]], IDS, [b"0000:0a:00.0", b"0000:02:00.0"], [b"\xfe"], [b"K", BDF[0]],
            [b"\t0000:01:00.0 ", b"ID", b"0000:02:00.0"], [BDF[2]], [b"0000:01:00.0\x1c0000:02:00.0"]]


def random_call(rng, n_reqs=None):
    """a seeded call mixing every case: (requests, egm)"""
    n_reqs = int(rng.integers(0, 6)) if n_reqs is None else n_reqs
    vend, links = list(VENDORS.values()), list(LINKS.values())
    reqs = []
    for _ in range(n_reqs):
        members = []
        for _ in range(int(rng.integers(0, 7))):
            if rng.random() < 0.7:
                members.append(ok_member())
            else:
                members.append((links[rng.integers(len(links))], vend[rng.integers(len(vend))], G))
        ids = [IDS[k] for k in rng.integers(0, len(IDS), size=int(rng.integers(0, 5)))]
        ids += [BDF[k] for k in rng.integers(0, len(BDF), size=int(rng.integers(0, 3)))]
        reqs.append((members, ids))
    gd = list(GPU_DEVICES.values())
    egm = []
    for e in range(int(rng.integers(0, 6))):
        name = b"egm%d" % e if rng.random() < 0.85 else b"x%d" % e
        gpus = gd[rng.integers(len(gd))] if rng.random() < 0.9 else None
        if rng.random() < 0.4:
            gpus = b" ".join(BDF[k] for k in rng.integers(0, len(BDF), size=int(rng.integers(1, 3))))
        egm.append((name, gpus, bool(rng.random() < 0.9)))
    return reqs, egm


def unpack(raw):
    """kvgpu.AllocRaw -> (requests, egm_entries) in allocate_raw's form"""
    def field(off, blob, k):
        return blob[int(off[k]):int(off[k + 1])]

    def read(st, f, value):
        if not st >> f & 1:
            return NOT_READ
        return None if st >> (8 + f) & 1 else value
    requests, m, i = [], 0, 0
    for n, k in zip(raw.n_members, raw.n_ids):
        members = []
        for _ in range(int(n)):
            st = int(raw.member_state[m])
            members.append((read(st, 0, field(raw.member_off, raw.member_bytes, 3 * m)),
                            read(st, 1, field(raw.member_off, raw.member_bytes, 3 * m + 1)),
                            field(raw.member_off, raw.member_bytes, 3 * m + 2)))
            m += 1
        requests.append((members, [field(raw.id_off, raw.id_bytes, i + j) for j in range(int(k))]))
        i += int(k)
    egm = []
    for e, st in enumerate(int(s) for s in raw.egm_state):
        stat = read(st, 2, True)
        egm.append((field(raw.egm_off, raw.egm_bytes, 2 * e), read(st, 1, field(raw.egm_off, raw.egm_bytes, 2 * e + 1)),
                    stat if stat is not None else False))
    return requests, egm


def contract(raw):
    """allocate_raw on a packed call: the C-ABI contract as Context.pci_allocate_raw returns it"""
    return allocate_raw(*unpack(raw))
