"""Deterministic pci.ids texts that put bytes and lines on the edges of K1's geometry, and the reference they are
checked against.  Shared by tests/test_gpu_parse_edges.py (the H100) and tests/test_parse_edges_emu.py (the kernel
source under the CPU warp emulator).  No GPU, no torch.

K1 (csrc/kvg_parse_k1.cuh) hands a warp 4 KiB spans read with a 16-byte halo; a span is 4 rows of 1 KiB, and lane l
owns bytes [l*16, l*16 + 16) of both 512-byte halves of a row, as eight 32-bit words.  Newlines are first found on
the low seven bits of each byte, a test that also fires for 0x8A (the second byte of UTF-8 "Ê" C3 8A and "Ċ" C4 8A,
the last byte of U+200A E2 80 8A); bytes >= 0x80 are excluded afterwards.  0x89, 0xA3 and 0x8D are '\\t', '#' and
'\\r' with bit 7 set.  A span's device lines in front of its first header take their vendor from the nearest earlier
span that has a header (the resolve pass); the last span of a file is patched at EOF, where a final '\\n' starts
no line.

The reference is the one the repository already pins: tools/span_model.py (checked against the C oracle by
tests/test_span_model.py) for the section bounds and the id -> first line table, and the oracle's getDeviceName
for each id's name, derived from its one matched line."""
import os
import re
import sys

from oracle import oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import span_model as M  # noqa: E402

NONE = 0xFFFFFFFF
SPAN, ROW = M.SPAN, 1024
# span edges the geometry cases sit on: multiples of 4 KiB that are not multiples of 8 KiB among them
EDGES = (4096, 8192, 12288, 20480)

# ------------------------------------------------------------------------------------------------------------------
# reference
# ------------------------------------------------------------------------------------------------------------------


def reference(text: bytes):
    """(span model of the text, {device id: name}) — the name table a parse of `text` must publish: every id the
    model records inside the first 10de section, named by the oracle from the one line the id matched."""
    model = M.parse(text)
    v, e = model["v_off"], model["sec_end"]
    names = {}
    for dev, off in model["table"].items():
        if v != NONE and v < off < e:
            end = text.find(b"\n", off)
            line = text[off:end if end >= 0 else len(text)]
            names[dev] = O.get_device_name(b"10de\n" + line + b"\n", b"%04x" % dev)
    return model, names


def ids_in(text: bytes) -> list:
    """Every 4-lower-hex key that follows a '\\t' anywhere in the text (device lines, ghosts, subsystem lines)."""
    return sorted({m.decode() for m in re.findall(rb"\t([0-9a-f]{4})", text)})


# ------------------------------------------------------------------------------------------------------------------
# byte builders
# ------------------------------------------------------------------------------------------------------------------
class _Text:
    """A text grown line by line; fill_to() reaches an exact offset with device lines of fresh ids."""

    def __init__(self, first_id: int = 0x4000):
        self.b = bytearray()
        self.next_id = first_id

    def add(self, line: bytes):
        self.b += line
        return self

    def _dev(self, n: int) -> bytes:       # a device line of exactly n >= 8 bytes, '\n' included
        self.next_id = (self.next_id + 1) & 0xFFFF
        return b"\t%04x  " % self.next_id + b"f" * (n - 8) + b"\n"

    def fill_to(self, target: int):
        gap = target - len(self.b)
        assert gap >= 0, (target, len(self.b))
        while gap > 80:
            self.b += self._dev(40)
            gap -= 40
        if gap >= 18:
            self.b += self._dev(gap // 2) + self._dev(gap - gap // 2)
        elif gap >= 8:
            self.b += self._dev(gap)
        elif gap:
            assert gap >= 2, "no line is one byte long"
            self.b += b"#" + b"c" * (gap - 2) + b"\n"
        return self

    def pad_to(self, n: int):
        """Comment lines up to exactly n bytes: texts of one length parse as the images of one batch."""
        gap = n - len(self.b)
        assert gap >= 2, (n, len(self.b))
        while gap > 80:
            self.b += b"#" + b"c" * 38 + b"\n"
            gap -= 40
        self.b += b"#" + b"c" * (gap - 2) + b"\n"
        return self

    def bytes(self) -> bytes:
        return bytes(self.b)


# ---- 0x8A inside device lines, on every offset of a row -----------------------------------------------------------
UNIT = 97              # bytes per line of alias_text: odd, so the 0x8A of 1024 consecutive lines covers a row
ALIAS_AT = 48          # offset of the 0x8A inside its line
ALIASES = (b"\xc3", b"\xc4", b"\xe2\x80", b"")   # + 0x8A: U+00CA, U+010A, U+200A (a space), a lone byte
AFTER_KEY = (0x89, 0xA3, 0x8D, 0x8A)             # '\t', '#', '\r', '\n' with bit 7 set, right after a device key
GHOST = 0x9000         # ghost id of line k: GHOST + k (a device line only if 0x8A were a newline)
REAL = 0x1000          # id of device line k: REAL + k
N_UNITS = 1100
VENDOR_AT = 40         # line 40 is the 10de header; lines 0..39 are vendor 8086, lines from NEXT_AT vendor 10df
NEXT_AT = 1060


def _follower(k: int) -> bytes:
    """What follows the 0x8A of line k: a line of each kind, if 0x8A counted as a newline."""
    return (b"\t%04x  ghost" % (GHOST + k),      # a device line: a ghost id
            b"10de  ghost vendor",               # moves v_off (before the section) or ends it (inside)
            b"1af4  ghost vendor",               # ends the section early
            b"# ghost comment")[(k // 4) % 4]    # one more line


def _alias_line(k: int) -> bytes:
    if k == 0:
        head = b"8086  Intel Corporation "
    elif k == VENDOR_AT:
        head = b"10de  NVIDIA Corporation "
    elif k == NEXT_AT:
        head = b"10df  next vendor "
    elif k % 11 == 5:
        head = b"# comment %d " % k
    elif k % 7 == 3:
        head = b"\t\t10de %04x  subsystem " % (REAL + k)
    elif k % 5 == 2:
        head = b"\t%04x" % (REAL + k) + bytes([AFTER_KEY[(k // 5) % 4]]) + b" n%d " % k
    else:
        head = b"\t%04x  n%d " % (REAL + k, k)
    prefix = ALIASES[k % 4]
    pad = ALIAS_AT - len(head) - len(prefix)
    body = head + b"x" * pad + prefix + b"\x8a" + _follower(k)
    assert pad >= 0 and len(body) < UNIT
    return body + b"y" * (UNIT - 1 - len(body)) + b"\n"


def alias_text() -> bytes:
    """N_UNITS lines of UNIT bytes, each with one 0x8A at ALIAS_AT: line k's 0x8A sits at row offset
    (48 + 97 k) % 1024, so the 1,100 lines put one on every lane, both halves, all 8 words and all 4 byte positions,
    in every row of a span.  Vendor 8086 first (a ghost "10de" there would move v_off), then the 10de section, then
    10df.  Every ghost id is distinct."""
    text = b"".join(_alias_line(k) for k in range(N_UNITS))
    offs = {(ALIAS_AT + UNIT * k) % ROW for k in range(N_UNITS)}
    assert len(offs) == ROW and {(ALIAS_AT + UNIT * k) // ROW % 4 for k in range(N_UNITS)} == {0, 1, 2, 3}
    return text


def alias_keys() -> list:
    """Arbitrary (general-path) keys that contain 0x8A or one of its relatives."""
    keys = [b"\x8a", b"\x8a\t", b"\xc3\x8a", b"5678\x8a", b"%04x\x89" % (REAL + 42), b"%04x\x8d" % (REAL + 62)]
    for k in (41, 42, 43, 44, 45, 47, 62, 82, 1059):
        line = _alias_line(k)[1:-1]
        cut = line.index(b"\x8a")
        keys += [line[:cut + 1], line[:cut + 6], line]
    return keys


# ---- bytes >= 0x80 at line starts ----------------------------------------------------------------------------------
def line_start_texts() -> list:
    """A line that starts with 0x89 / 0xA3 / 0x8D / 0x8A inside the 10de section: a header-type line to getDeviceName
    (neither '\\t' nor '#'), so it ends the section; the bytes behind it form a device line only if the special
    byte were taken for its low seven bits.  Placed around row, lane and span edges."""
    out = []
    for b in AFTER_KEY:
        for p in (1023, 1024, 1040, 1535, 1536, SPAN - 1, SPAN, SPAN + 1, 2 * SPAN + 15, 3 * SPAN + 16):
            t = _Text(0x2000).add(b"10de  NVIDIA\n\t0001  first\n").fill_to(p)
            t.add(bytes([b]) + b"\t0002  behind\n\t0003  after\n").fill_to(p + 600).add(b"\t0004  last\n")
            out.append(t.bytes())
    return out


# ---- span geometry at 4 KiB ----------------------------------------------------------------------------------------
def span_edge_texts() -> list:
    """For each span edge S of EDGES and each d in -2..2, texts of S + 6144 bytes with:
      - a 10de device line starting at S + d (a line on a span's last byte has its first bytes in the halo;
        at S - 1 the '\\t' is the span's last byte and the id is in the next span), the lines of its span in front
        of the span's first header resolved from the 10de header 1 to 5 spans back;
      - a 10de header starting at S + d (straddling the edge for d < 0), its device lines running into the next
        span, which resolves them from the span just before it;
      - a non-10de header at S + d whose device lines run into the next span (resolved, not recorded)."""
    out = []
    for S in EDGES:
        for d in range(-2, 3):
            t = _Text(0x0100).add(b"10de  NVIDIA\n").fill_to(S + d)
            t.add(b"\tedfe  on the edge\n").fill_to(S + d + 3000).add(b"8086  Intel\n\t7777  other\n")
            out.append(t.pad_to(S + 6144).bytes())
            t = _Text(0x0200).add(b"8086  Intel\n").fill_to(S + d)
            t.add(b"10de  NVIDIA\n\t1111  first\n").fill_to(S + d + 5000).add(b"10df  next\n\t2222  other\n")
            out.append(t.pad_to(S + 6144).bytes())
            t = _Text(0x0300).add(b"10de  NVIDIA\n\t0001  a\n").fill_to(S + d)
            t.add(b"8086  Intel\n").fill_to(S + d + 5000).add(b"10de  again\n\t3333  second section\n")
            out.append(t.pad_to(S + 6144).bytes())
    return out


def resolve_texts() -> list:
    """Device lines in front of a span's first header whose vendor context is 1, 2 and 33 spans back (the resolve
    warp looks back 32 spans per step), behind a 10de header and behind a non-10de one (nothing may be recorded),
    and with a run of two spans that hold no newline at all in between."""
    out = []
    for back in (1, 2, 33):
        n = (back + 4) * SPAN
        for vendor in (b"10de  NVIDIA", b"8086  Intel"):
            t = _Text(0x0400).add(b"# head\n" + vendor + b"\n").fill_to(back * SPAN + 100)
            out.append(t.add(b"1002  AMD\n\t5555  amd\n").pad_to(n).bytes())
        t = _Text(0x0500).add(b"10de  NVIDIA\n\t0001  a\n#" + b"c" * (2 * SPAN + 7) + b"\n").fill_to((back + 2) * SPAN + 9)
        out.append(t.add(b"1002  AMD\n\t5555  amd\n").pad_to(n).bytes())
    return out


# ---- EOF -----------------------------------------------------------------------------------------------------------
EOF_DELTAS = (-1, 0, 1, 15, 16, 17)
EOF_KINDS = {"device": (1, 2), "header": (1, 2), "10de_header": (1, 2), "long_line": (1, 2, 16, 17)}   # kind -> k


def eof_text(k: int, delta: int, newline: bool, kind: str) -> bytes:
    """A text of exactly k * 4096 + delta bytes, ending in '\\n' or not, whose last line is a 10de device line, a
    non-10de header, the 10de header itself (an empty section), or a device line that runs from near the start of
    the file (the last line is just under 64 KiB at k = 16 and over it at k = 17: the bufio.Scanner token limit)."""
    n = k * SPAN + delta
    end = b"\n" if newline else b""
    if kind == "device":
        t = _Text(0x0600).add(b"10de  NVIDIA\n").fill_to(n - 12 - len(end)).add(b"\tcafe  last!" + end)
    elif kind == "header":
        t = _Text(0x0700).add(b"10de  NVIDIA\n").fill_to(n - 12 - len(end)).add(b"8086  last v" + end)
    elif kind == "10de_header":
        t = _Text(0x0800).add(b"8086  Intel\n").fill_to(n - 12 - len(end)).add(b"10de  NVIDIA" + end)
    else:
        head = b"10de  NVIDIA\n\t0001  first\n"
        t = _Text().add(head + b"\tbeef  " + b"y" * (n - len(head) - 7 - len(end)) + end)
    text = t.bytes()
    assert len(text) == n, (k, delta, newline, kind, len(text))
    return text


def eof_cases() -> list:
    """(k, delta, newline, kind) of every EOF text."""
    return [(k, d, nl, kind) for kind, ks in EOF_KINDS.items() for k in ks for d in EOF_DELTAS for nl in (True, False)]
