"""K1 (csrc/kvg_parse_k1.cuh) from its kernel source under the CPU warp emulator on the texts of tests/parse_edges.py:
0x8A and its relatives on every offset of a row, lines on both sides of 4 KiB span edges, vendor context resolved
from 1 to 33 spans back, and every way a file can end around a span edge.  The scan kernel runs at several grid
sizes (scan_ctas), so that warps also stream many spans through their ring.  Per text: the section bounds, line count
and the whole device-id table against tools/span_model.py, and the names the library sequence returns (table path
and k_lookup_general) against the oracle's getDeviceName."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import parse_edges as E
from parse_edges import M
from oracle import oracle as O

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402
from test_names_emu import device_names  # noqa: E402
from test_parse_k1_emu import pad  # noqa: E402

NONE = E.NONE


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_names())
    L.emu_parse_k1.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    L.emu_get_device_names.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                       C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                       C.c_void_p]
    return L


def check_batch(emu, texts, scan_ctas, what=""):
    """Texts of one length parsed as the images of one batch: per image the section bounds, the line count and the
    whole device-id table against the span model."""
    n = len(texts[0])
    assert all(len(t) == n for t in texts)
    images = np.concatenate([pad(t) for t in texts])
    stride = len(images) // len(texts)
    info = np.zeros((len(texts), 8), dtype=np.uint32)
    tables = np.zeros((len(texts), 65536), dtype=np.uint32)
    assert emu.emu_parse_k1(images.ctypes.data, stride, n, len(texts), scan_ctas, info.ctypes.data,
                            tables.ctypes.data) == 0
    for f, text in enumerate(texts):
        model = M.parse(text)
        assert model["n_lines"] == text.count(b"\n")
        v_off, sec_end, _, n_lines, limit, overflow = (int(x) for x in info[f][:6])
        assert (v_off, sec_end, limit, n_lines, overflow) == \
            (model["v_off"], model["sec_end"], model["limit"], model["n_lines"], 0), (what, f, scan_ctas)
        want = np.full(65536, NONE, dtype=np.uint32)
        for dev, off in model["table"].items():
            want[dev] = off
        bad = np.nonzero(tables[f] != want)[0]
        assert len(bad) == 0, (what, f, scan_ctas, ["%04x: %x want %x" % (i, tables[f][i], want[i]) for i in bad[:8]])


def by_length(texts):
    groups = {}
    for t in texts:
        groups.setdefault(len(t), []).append(t)
    return [groups[n] for n in sorted(groups)]


def check_names(emu, text, extra=(), what=""):
    """Every id in the text through the table path and `extra` keys through the general path, against the oracle;
    the reference's names (tests/parse_edges.py) are checked against the oracle on the way."""
    _, names = E.reference(text)
    ids = E.ids_in(text)
    keys = [k.encode() for k in ids] + list(extra)
    for k, g in zip(keys, device_names(emu, text, keys)):
        assert g == O.get_device_name(text, k), (what, k)
    for k in ids:
        assert names.get(int(k, 16), "") == O.get_device_name(text, k.encode()), (what, k)


def test_alias_bytes_on_every_row_offset(emu):
    """0x8A inside valid UTF-8 and alone, on all 1,024 offsets of a row in all four rows, each followed by a ghost
    device line, a ghost 10de header, a ghost header and a ghost comment; 0x89 / 0xA3 / 0x8D / 0x8A right after
    device keys.  Grids of one warp per span, and of 1, 2 and 5 CTAs (the ring wraps)."""
    text = E.alias_text()
    model = M.parse(text)
    assert model["v_off"] == E.VENDOR_AT * E.UNIT and len(model["table"]) > 700
    assert not any(E.GHOST <= d < E.GHOST + E.N_UNITS for d in model["table"])
    for scan_ctas in (0, 1, 2, 5):
        check_batch(emu, [text], scan_ctas, "alias")
    check_names(emu, text, E.alias_keys(), "alias")


def test_high_bytes_at_line_starts(emu):
    for i, group in enumerate(by_length(E.line_start_texts())):
        check_batch(emu, group, i % 3, ("line start", len(group[0])))
    text = E.line_start_texts()[5]
    check_names(emu, text, (b"0002", b"\x89\t0002", b"\x8a"), "line start")


def test_span_edges(emu):
    for i, group in enumerate(by_length(E.span_edge_texts())):
        check_batch(emu, group, i % 3, ("span edge", len(group[0])))
    texts = E.span_edge_texts()
    for i in (3, 4, 5, 22):
        check_names(emu, texts[i], (), ("span edge", i))


def test_resolve_from_spans_back(emu):
    for i, group in enumerate(by_length(E.resolve_texts())):
        check_batch(emu, group, 2 - i, ("resolve", len(group[0])))


def test_file_ends_around_span_edges(emu):
    cases = E.eof_cases()
    for k, d in sorted({(c[0], c[1]) for c in cases}):
        texts = [E.eof_text(*c) for c in cases if c[:2] == (k, d)]
        check_batch(emu, texts, (k + d) % 3, ("eof", k, d))
    for c in cases:
        if c[0] == 1 and c[1] in (0, 16) and c[3] != "long_line":   # long names exceed the harness's name buffer
            check_names(emu, E.eof_text(*c), (), c)
