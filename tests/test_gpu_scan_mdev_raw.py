"""kvg_scan_mdev_raw on the H100: the decoded snapshot against the Go-exact restatement (tests/mdev_raw_cases.py), the
result against kvg_scan_mdev on the decoded records and dictionary, canonical dumps against the oracle's tree walk,
refusals, launch counts and isolation from the mdev delta and health state."""
import numpy as np
import pytest

import mdev_raw_cases as MC
import util
import kvgpu
from kvgpu import _lib as L
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = kvgpu.Context(0)
    c.pciids_load(util.pciids_text())
    yield c
    c.close()


def same_result(a, b):
    assert a.n_records == b.n_records
    assert (a.labels, a.type_names) == (b.labels, b.type_names)
    for f in ("survivors", "type_keys", "type_off", "type_perm", "type_canon", "par_keys", "par_off", "par_perm"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def check(ctx, raw):
    try:
        want = MC.go_mdev_snapshot(raw)
    except MC.RawError as e:
        exc = kvgpu.ReferencePanic if e.kind == "panic" else L.KvgError
        with pytest.raises(exc) as got:
            ctx.scan_mdev_raw(raw)
        if e.kind != "panic":
            assert got.value.rc == (L.KVG_EINVAL if e.kind == "miss" else L.KVG_ERANGE)
        assert ("entry %d " % e.entry) in str(got.value)
        return None
    res, snap = ctx.scan_mdev_raw(raw)
    assert snap.recs.tobytes() == want[0].tobytes()
    assert (snap.uuid_ok, snap.parent_names is None, snap.raw_types, snap.parent_names) == want[1:]
    assert snap.names == list(raw.names)
    same_result(res, ctx.scan_mdev(snap.recs, snap.raw_types))
    return res, snap


@pytest.mark.parametrize("n", [0, 1, 257, 1025, 5000, 70000])
@pytest.mark.parametrize("names,parents", [("canonical", "packed"), ("mixed", "mixed"), ("canonical", "mixed"),
                                           ("mixed", "packed")])
def test_random_matrix(ctx, n, names, parents):
    got = check(ctx, MC.raw_of(MC.gen_entries(np.random.default_rng(n + len(names) + 5 * len(parents)), n,
                                              names=names, parents=parents)))
    if got is not None and n >= 1025:
        assert got[1].uuid_ok == (names == "canonical") and (got[1].parent_names is None) == (parents == "packed")


@pytest.mark.parametrize("seed", range(4))
def test_panic_precedence(ctx, seed):
    # targets without '/' where they are reached: the lowest entry wins, and any panic beats a range error
    check(ctx, MC.raw_of(MC.gen_entries(np.random.default_rng(200 + seed), 4000, panic=True, parents="mixed")))


U = [MC.uuid_name(bytes([k]) * 16) for k in range(1, 4)]


def one(u, **kw):
    e = {"type": b"GRID P40-1Q\n", "link": MC.link_to(MC.PARENT, u), "numa_node": b"0\n"}
    e.update(kw)
    return e


def test_panic_beats_range(ctx):
    raw = MC.raw_of([(U[0], one(U[0], numa_node=b"40000")), (U[1], one(U[1], link=b"nolash"))])
    with pytest.raises(kvgpu.ReferencePanic, match="entry 1 .*link"):
        ctx.scan_mdev_raw(raw)


@pytest.mark.parametrize("k", [65535, 65536])
def test_type_cap(ctx, k):
    names = MC.canonical_names(np.random.default_rng(k), k)
    got = check(ctx, MC.raw_of([(u, one(u, type=b"T%d" % j)) for j, u in enumerate(names)]))
    assert (got is None) == (k == 65536)


def test_trees(ctx, tmp_path):
    text = util.pciids_text()
    for name, vbase, pbase, plain in MC.trees(tmp_path):
        res, snap = ctx.scan_mdev_raw(kvgpu.read_mdev_tree_raw(vbase, pbase))
        same_result(res, ctx.scan_mdev(snap.recs, snap.raw_types))
        om = O.Maps()
        assert om.create_vgpu_id_map_tree(vbase, pbase) == 0
        got = kvgpu.canonical_dump(kvgpu.mdev_maps_from_result(res, snap))
        assert got == om.dump(text), name
        if plain:
            want = kvgpu.snapshot_mdev_tree(vbase, pbase)
            assert snap.recs.tobytes() == want.recs.tobytes(), name
            assert (snap.uuid_ok, snap.raw_types, snap.parent_names) == (
                want.uuid_ok, want.raw_types, want.parent_names), name
        else:
            assert "" in kvgpu.mdev_maps_from_result(res, snap).gpuVgpuMap, name


def test_million_numeric(ctx):
    types = O.gen_type_names(256)
    recs = O.gen_mdev(0, 1_000_000)
    res, snap = ctx.scan_mdev_raw(MC.render_records(recs, types))
    assert snap.uuid_ok and snap.parent_names is None
    kept = (recs["flags"] & L.MF_TYPE_ERR) == 0
    assert np.array_equal(snap.recs["uuid"], recs["uuid"])
    assert [snap.raw_types[t] for t in snap.recs["type_idx"][kept]] == [types[t] for t in recs["type_idx"][kept]]
    linked = kept & ((recs["flags"] & L.MF_PARENT_ERR) == 0)
    assert np.array_equal(snap.recs["parent"][linked], recs["parent"][linked])
    want_flags = np.where(~kept, L.MF_TYPE_ERR, np.where(~linked, L.MF_PARENT_ERR, recs["flags"] & L.MF_NUMA_ERR))
    assert np.array_equal(snap.recs["flags"], want_flags.astype(np.uint8))
    same_result(res, ctx.scan_mdev(snap.recs, snap.raw_types))


def raw_arg(raw):
    import ctypes as C
    off = np.ascontiguousarray(raw.off, dtype=np.uint32)
    state = np.ascontiguousarray(raw.state, dtype=np.uint16)
    blob = np.frombuffer(raw.bytes + b"\0", dtype=np.uint8)
    a = L.MdevRawC(len(state), off.ctypes.data, blob.ctypes.data, state.ctypes.data)
    return C.byref(a), (a, off, state, blob)


def test_refusals(ctx):
    import ctypes as C
    lib, h = ctx._lib, ctx.handle
    raw = MC.raw_of([(U[0], one(U[0]))])
    res, snap = C.byref(C.POINTER(L.MdevResultC)()), C.byref(C.POINTER(L.MdevSnapC)())
    base = ctx.launch_count
    assert lib.kvg_scan_mdev_raw(None, None, None, None) == L.KVG_EINVAL
    assert lib.kvg_scan_mdev_raw(h, None, res, snap) == L.KVG_EINVAL
    arg = raw_arg(raw)
    assert lib.kvg_scan_mdev_raw(h, arg[0], None, snap) == L.KVG_EINVAL
    assert lib.kvg_scan_mdev_raw(h, arg[0], res, None) == L.KVG_EINVAL
    bad = raw.off.copy()
    bad[2] = 0  # decreasing
    assert lib.kvg_scan_mdev_raw(h, raw_arg(kvgpu.MdevRaw(raw.names, bad, raw.bytes, raw.state))[0], res,
                                 snap) == L.KVG_EINVAL
    bad = raw.off.copy() + 1
    assert lib.kvg_scan_mdev_raw(h, raw_arg(kvgpu.MdevRaw(raw.names, bad, raw.bytes, raw.state))[0], res,
                                 snap) == L.KVG_EINVAL
    nul = L.MdevRawC(1, None, None, None)
    assert lib.kvg_scan_mdev_raw(h, C.byref(nul), res, snap) == L.KVG_EINVAL
    assert ctx.launch_count == base and not res._obj and not snap._obj
    fresh = kvgpu.Context(0)
    try:
        with pytest.raises(L.KvgError) as e:
            fresh.scan_mdev_raw(raw)
        assert e.value.rc == L.KVG_ESTATE and fresh.launch_count == 0
    finally:
        fresh.close()


def test_launch_counts(ctx):
    """decode + type probe + type compaction + pack + the scan's; + a probe and a compaction for parents in index
    mode; none for n = 0"""
    names = MC.canonical_names(np.random.default_rng(3), 19)
    numeric = MC.raw_of([(u, one(u, type=b"T%d\n" % (k % 3))) for k, u in enumerate(names)])
    _, snap = ctx.scan_mdev_raw(numeric)
    ctx.scan_mdev(snap.recs, snap.raw_types)
    b0 = ctx.launch_count
    ctx.scan_mdev(snap.recs, snap.raw_types)
    scan = ctx.launch_count - b0
    b0 = ctx.launch_count
    ctx.scan_mdev_raw(numeric)
    assert ctx.launch_count - b0 == 1 + 2 + 1 + scan
    index = MC.raw_of([(b"%d" % k, one(b"%d" % k, type=b"T%d\n" % (k % 3), link=b"x/gpu%d/u" % (k % 2)))
                       for k in range(19)])
    ctx.scan_mdev_raw(index)
    b0 = ctx.launch_count
    ctx.scan_mdev_raw(index)
    assert ctx.launch_count - b0 == 1 + 2 + 2 + 1 + scan
    b0 = ctx.launch_count
    res, snap = ctx.scan_mdev_raw(MC.raw_of([]))
    assert ctx.launch_count == b0 and len(res.survivors) == 0 and len(snap.recs) == 0 and snap.raw_types == []


def test_isolation(ctx):
    """the mdev delta and mdev health state are untouched: the next delta / health call sees only its own history"""
    recs, types = O.gen_mdev(0, 5000), O.gen_type_names(256)
    ctx.scan_mdev_delta_reset()
    ctx.health_mdev_reset()
    r1, d1 = ctx.scan_mdev_delta(recs, types)
    h1 = ctx.health_rescan_mdev(recs, len(types))
    k1 = ctx.health_rescan_mdev_keyed(recs, len(types))
    check(ctx, MC.raw_of(MC.gen_entries(np.random.default_rng(9), 3000, names="mixed", parents="mixed")))
    r2, d2 = ctx.scan_mdev_delta(recs, types)
    h2 = ctx.health_rescan_mdev(recs, len(types))
    k2 = ctx.health_rescan_mdev_keyed(recs, len(types))
    assert len(d2.changes) == 0 and d2.n_prev == len(r1.survivors)
    assert len(h2.changed) == 0 and h2.n_alive == h1.n_alive
    assert len(k2.changed) == 0 and k2.n_alive == k1.n_alive
