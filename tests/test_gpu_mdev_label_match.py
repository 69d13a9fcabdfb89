"""kvg_mdev_label_match on the H100: the vGPU plugin's Allocate-time label check, one launch per call, against the label
rule of the plugin's CPU path (tests/label_match_cases.py) at 0 to 100,000 files and over 1 MiB of bytes; every refusal
(KVG_EINVAL, nothing launched); and isolation: a call between a device scan and its fetch, between two mdev delta
scans, or between two keyed vGPU health ticks changes none of their results."""
import ctypes as C

import numpy as np
import pytest

import label_match_cases as LM
import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

KVG_EINVAL = -1


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


@pytest.fixture(scope="module")
def ctx(kv):
    c = kv.Context(0)
    c.pciids_load(util.pciids_text())
    yield c
    c.close()


def checked(ctx, files, name):
    before = ctx.launch_count
    got = ctx.mdev_label_match(files, name)
    assert ctx.launch_count - before == (1 if files else 0)
    assert got.dtype == bool and len(got) == len(files)
    assert np.array_equal(got, LM.want(files, name)), (len(files), name[:40])
    return got


def test_edges(ctx):
    for name in LM.edge_names():
        checked(ctx, LM.EDGES, name)
    for raw in LM.EDGES:
        assert checked(ctx, [raw], LM.ref_label(raw))[0]


def test_str_names_are_latin1(ctx):
    files = [b"GRID\xa0A100\n", b"GRID A100"]
    assert list(ctx.mdev_label_match(files, "GRID\xa0A100")) == [True, False]
    assert list(ctx.mdev_label_match(files, "GRID_A100")) == [False, True]


@pytest.mark.parametrize("n", [0, 1, 16, 4096, 100_000])
def test_sizes(ctx, n):
    rng = np.random.default_rng(n)
    files = LM.random_files(n, rng)
    for name in (LM.NAME, b"GRID_A100-4Q", b"", LM.NAME + b"_"):
        checked(ctx, files, name)
    if n >= 16:
        assert 0 < LM.want(files, LM.NAME).sum() < n


def test_more_than_a_mebibyte(ctx):
    files = LM.random_files(3000, np.random.default_rng(5), big_every=150)
    assert sum(len(f) for f in files) > 1 << 20
    got = checked(ctx, files, LM.NAME)
    assert got[::150].all()
    checked(ctx, files, LM.NAME[:-1])


def _raw_call(kv, ctx, handle, files, name, name_len, match):
    lib = kv.load()
    return lib.kvg_mdev_label_match(handle, files, name, name_len, match)


def test_refusals_launch_nothing(kv, ctx):
    off = np.array([0, 3, 5], dtype=np.uint32)
    raw = np.frombuffer(b"abcde\0", dtype=np.uint8)
    match = np.zeros(4, dtype=np.uint8)
    P32, P8 = C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)

    def td(n, o, b):
        return C.byref(kv._lib.TypeDict(n, C.cast(o, P32) if o is not None else None,
                                        C.cast(b, P8) if b is not None else None))
    good = (td(2, off.ctypes.data, raw.ctypes.data), b"abc", 3, match.ctypes.data)
    h = ctx.handle
    before = ctx.launch_count
    assert _raw_call(kv, ctx, h, *good) == 0
    assert ctx.launch_count == before + 1 and list(match[:2]) == [1, 0]
    before = ctx.launch_count
    bad_off0 = np.array([1, 3, 5], dtype=np.uint32)
    bad_desc = np.array([0, 4, 3], dtype=np.uint32)
    cases = [
        (None,) + good,                                                        # ctx NULL
        (h, None) + good[1:],                                                  # files NULL
        (h,) + good[:3] + (None,),                                             # match NULL
        (h, td(2, None, raw.ctypes.data)) + good[1:],                          # off NULL
        (h, td(2, off.ctypes.data, None)) + good[1:],                          # bytes NULL
        (h, good[0], None, 3, match.ctypes.data),                              # name NULL, name_len > 0
        (h, td(2, bad_off0.ctypes.data, raw.ctypes.data)) + good[1:],          # off[0] != 0
        (h, td(2, bad_desc.ctypes.data, raw.ctypes.data)) + good[1:],          # decreasing offsets
    ]
    for i, args in enumerate(cases):
        match[:] = 0xee
        assert _raw_call(kv, ctx, *args) == KVG_EINVAL, i
        assert (match == 0xee).all(), i
    assert ctx.launch_count == before
    # n = 0: nothing to check, nothing launched, with or without arrays; a NULL name of length 0 is fine
    assert _raw_call(kv, ctx, h, td(0, None, None), None, 0, match.ctypes.data) == 0
    assert _raw_call(kv, ctx, h, td(0, off.ctypes.data, raw.ctypes.data), b"x", 1, match.ctypes.data) == 0
    assert ctx.launch_count == before
    assert _raw_call(kv, ctx, h, td(2, off.ctypes.data, raw.ctypes.data), None, 0, match.ctypes.data) == 0
    assert list(match[:2]) == [0, 0] and ctx.launch_count == before + 1


def _same(a, b):
    for f in a.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f


def _match_in_between(ctx):
    files = LM.random_files(5000, np.random.default_rng(11), big_every=1000)
    checked(ctx, files, LM.NAME)


def test_device_scan_and_fetch_are_untouched(kv, ctx):
    import torch
    recs, types = O.gen_mdev(3, 50_000), O.gen_type_names(300)
    buf = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    try:
        ctx.dev_scan_mdev(buf.data_ptr(), len(recs), types)
        want = ctx.dev_scan_mdev_fetch()
        ctx.dev_scan_mdev(buf.data_ptr(), len(recs), types)
        _match_in_between(ctx)
        _same(ctx.dev_scan_mdev_fetch(), want)
    finally:
        torch.cuda.synchronize()
        del buf


def test_mdev_delta_is_untouched(kv, ctx):
    a, b, types = O.gen_mdev(4, 20_000), O.gen_mdev(4, 20_000), O.gen_type_names(256)
    b["type_idx"][::97] = (b["type_idx"][::97] + 1) % 256
    b["flags"][::301] ^= 1
    ctx.scan_mdev_delta_reset()
    ctx.scan_mdev_delta(a, types)
    want_res, want = ctx.scan_mdev_delta(b, types)
    ctx.scan_mdev_delta_reset()
    ctx.scan_mdev_delta(a, types)
    _match_in_between(ctx)
    got_res, got = ctx.scan_mdev_delta(b, types)
    _same(got_res, want_res)
    _same(got, want)
    assert len(want.changes) > 0


@pytest.mark.parametrize("n", [1000, 40_000])
def test_keyed_health_is_untouched(kv, ctx, n):
    recs = O.gen_mdev(6, n)
    order = np.argsort(np.ascontiguousarray(recs["uuid"]).view("V16").ravel(), kind="stable")
    recs = recs[order]
    parents = np.unique(recs["parent"])
    ticks = [(recs, [int(parents[0])]), (recs[1:], []), (recs, [int(parents[-1])])]

    def run(between):
        ctx.health_rescan_mdev_keyed(recs[:0], 200)          # an empty list resets
        out = []
        for r, x in ticks:
            if between:
                _match_in_between(ctx)
            d = ctx.health_rescan_mdev_keyed(r, 200, x)
            out.append((d.n_records, d.n_alive, d.changed.tobytes()))
        return out
    assert run(True) == run(False)
