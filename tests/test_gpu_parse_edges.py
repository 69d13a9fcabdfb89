"""K1, the pci.ids parse (csrc/kvg_parse_k1.cuh), on the H100 at its own geometry: the texts of tests/parse_edges.py
(0x8A and its relatives on every offset of a row, lines on both sides of 4 KiB span edges, vendor context resolved
from 1 to 33 spans back, every way a file can end around a span edge), a batch large enough that every warp of the
persistent scan grid streams several spans through its ring, and the self-cleaning table across parses.

Per text: pciids_info() and the whole name_table() against tools/span_model.py with names from the oracle, and
name_lookup() against the oracle's getDeviceName for every id in the text (ghost ids included), random ids and
arbitrary keys (k_lookup_general).  Every test here needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

import parse_edges as E
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

# CTAs of k_pciids_scan per SM: what cudaOccupancyMaxActiveBlocksPerMultiprocessor returns for it (the query of
# kvg_api_pciids.inc that sizes the persistent grid, k1_grid = SMs x this).  Measured on an H100 80GB HBM3 (132 SMs,
# 400 W power limit): 10, so k1_grid = 1,320 CTAs = 5,280 warps.  The kernel uses 42 registers per thread (10 CTAs of
# 128 threads fill the register file) and 16,448 + 128 bytes of shared memory per CTA.
K1_CTAS_PER_SM = 10


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


@pytest.fixture(scope="module")
def ctx(kv):
    c = kv.Context(0)
    yield c
    c.close()


def check_parsed(ctx, text, extra_keys=(), lookups=None, what=""):
    """The table published for `text` against the reference, in full; name_lookup for every id in the text (or the
    ids given as `lookups`), 40 random ids and `extra_keys` against the oracle."""
    model, names = E.reference(text)
    info = ctx.pciids_info()
    assert model["n_lines"] == text.count(b"\n")
    assert (info["vendor_off"], info["section_end"], info["n_lines"], info["n_entries"]) == \
        (model["v_off"], model["sec_end"], model["n_lines"], len(model["table"])), what
    want = [""] * 65536
    for dev, name in names.items():
        want[dev] = name
    got = ctx.name_table(0, 65536)
    if got != want:
        bad = [i for i in range(65536) if got[i] != want[i]]
        raise AssertionError("%s: %d ids differ, first %s" % (what, len(bad), [("%04x" % i, got[i], want[i]) for i in bad[:4]]))
    rng = np.random.default_rng(len(text))
    keys = [k.encode() for k in (E.ids_in(text) if lookups is None else lookups)]
    keys += [b"%04x" % int(i) for i in rng.integers(0, 65536, 40)] + list(extra_keys)
    for k in keys:
        assert ctx.name_lookup(k) == O.get_device_name(text, k), (what, k)


def test_alias_bytes_on_every_row_offset(ctx):
    """0x8A inside valid UTF-8 and alone on all 1,024 offsets of a row, in all four rows, each followed by what would
    be a device line, a 10de header, another header or a comment if it were a newline; 0x89 / 0xA3 / 0x8D / 0x8A right
    after device keys, looked up as arbitrary keys too."""
    text = E.alias_text()
    ctx.pciids_load(text)
    check_parsed(ctx, text, E.alias_keys(), what="alias")


def test_high_bytes_at_line_starts(ctx):
    for i, text in enumerate(E.line_start_texts()):
        ctx.pciids_load(text)
        check_parsed(ctx, text, (b"\x89\t0002", b"\xa3\t0002", b"\x8a", b"0002 "), what=("line start", i))


def test_span_edges(ctx):
    for i, text in enumerate(E.span_edge_texts()):
        ctx.pciids_load(text)
        check_parsed(ctx, text, what=("span edge", i))


def test_resolve_from_spans_back(ctx):
    for i, text in enumerate(E.resolve_texts()):
        ctx.pciids_load(text)
        check_parsed(ctx, text, what=("resolve", i))


def test_file_ends_around_span_edges(ctx):
    for c in E.eof_cases():
        text = E.eof_text(*c)
        ctx.pciids_load(text)
        check_parsed(ctx, text, (b"cafe  last", b"beef  yyy", b"\x8a"), what=c)


def test_ring_cycles_on_the_h100(kv):
    """A batch of distinct images of one length whose span count is 4 x (4 warps x k1_grid): every warp of the
    persistent scan grid streams at least four spans through its ring, crossing from one image into the next.
    Image 0 holds the 0x8A sweep, a 10de header straddling a span edge and context resolved 33 spans back; the others are slices of the
    shipped pci.ids.  Image 0's table and info are checked in full.  Then the same context parses a single text with
    disjoint ids: no slot of the batch may survive into its table."""
    import torch
    k1_grid = torch.cuda.get_device_properties(0).multi_processor_count * K1_CTAS_PER_SM
    alias = E.alias_text()
    gap = -len(alias) % E.SPAN    # the span edge case stays on span edges
    image0 = alias + b"#" + b"c" * (gap - 2) + b"\n" + E.span_edge_texts()[40] + E.resolve_texts()[6]
    n = len(image0)
    spf = (n + E.SPAN - 1) // E.SPAN
    n_files = -(-4 * 4 * k1_grid // spf)
    shipped = util.pciids_text()
    step = (len(shipped) - n) // n_files
    assert step > 0
    c = kv.Context(0)
    try:
        stride = c.text_pad(n) + 16
        host = np.full(stride * n_files, 10, dtype=np.uint8)
        host[:n] = np.frombuffer(image0, dtype=np.uint8)
        src = np.frombuffer(shipped, dtype=np.uint8)
        for f in range(1, n_files):
            host[f * stride:f * stride + n] = src[f * step:f * step + n]
        dev = torch.from_numpy(host).cuda()
        torch.cuda.synchronize()
        assert spf * n_files >= 16 * k1_grid
        c.dev_pciids_parse(dev.data_ptr(), n, stride, n_files)
        model = E.M.parse(image0)
        check_parsed(c, image0, lookups=[k for k in E.ids_in(image0) if int(k, 16) in model["table"]][::3],
                     what="ring image 0")
        c.dev_pciids_parse(dev.data_ptr(), n, stride, n_files)   # the same batch again, from the table it left
        check_parsed(c, image0, lookups=(), what="ring image 0, re-parse")
        other = b"10de  NVIDIA\n" + b"".join(b"\t%04x  disjoint %d\n" % (0xd000 + i, i) for i in range(3000))
        c.pciids_load(other)
        check_parsed(c, other, lookups=(), what="single parse after the batch")
        del dev
    finally:
        torch.cuda.synchronize()
        c.close()


def test_table_cleans_itself_between_texts(kv):
    """Every id of the table named, then a text without any 10de header: the whole table must read empty.  Then the
    other way round."""
    c = kv.Context(0)
    try:
        full = b"10de  NVIDIA\n" + b"".join(b"\t%04x  d%04x\n" % (i, i) for i in range(65536))
        c.pciids_load(full)
        check_parsed(c, full, lookups=["0000", "1b38", "8a8a", "ffff"], what="full table")
        none = b"8086  Intel\n\t0000  a\n\t1b38  b\n1002  AMD\n\tffff  c\n# 10de  in a comment\n\t10de  not a vendor\n"
        c.pciids_load(none)
        check_parsed(c, none, what="no 10de")
        assert c.pciids_info()["vendor_off"] == E.NONE
        c.pciids_load(full)
        check_parsed(c, full, lookups=["0001", "fffe"], what="full table again")
    finally:
        c.close()
