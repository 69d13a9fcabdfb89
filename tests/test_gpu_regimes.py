"""Every size regime of the scans against an exact reference, on both sides of each threshold the host uses to
pick a kernel variant.

The host chooses among kernel variants by record count, key width and the kind of caller memory
(kvg_api_scan.inc, kvg_api_mdev.inc, kvg_api_health.inc, kvg_api_shard.inc).  Each group below runs one of
those decisions on both sides and compares the whole result with the numpy restatements of tests/util.py
(exact at any size), and with the CPU oracle's canonical dump where the oracle finishes in seconds.  Where a
launch label shows which variant ran, a separate call with kernel timing on asserts it, so that no case can
pass on the wrong side of its threshold.  Every test here needs an H100 (`-m gpu`).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import util
from oracle import oracle as O

pytestmark = pytest.mark.gpu

Mi = 1 << 20
# kvg_api_scan.inc enqueue_classify: `if (n < (2u << 20))` one k_compact<PciClassifyOp, 128, 8> launch, else k_classify_ragged ->
# k_tile_offsets -> k_pack_survivors
CLASSIFY_SPLIT = 2 * Mi
# kvg_api_scan.inc enqueue_orderings: `if (expect < (2u << 20))` k_order_final, else k_order_heads<false> ->
# k_tile_offsets -> k_order_heads<true>
FINAL_SPLIT = 2 * Mi
# kvg_order.cuh C_TILE (2048 items per tile); enqueue_orderings: Te = ceil(n / C_TILE),
# `tile_major = !big && Te <= 1024` (k_order_tilescan_cols), `else if (Te > 2048)` k_order_tilescan_long
C_TILE = 2048
TILE_MAJOR_MAX = 1024 * C_TILE
TILESCAN_LONG_ABOVE = 2048 * C_TILE
# kvg_api_scan.inc enqueue_orderings: `const bool big = expect >= (8u << 20)`: 8-bit digits instead of 11
DIGITS8_MIN = 8 * Mi
# kvg_api_scan.inc PIPE_MIN_RECORDS / PIPE_MAX_RECORDS: kvg_scan_pci pipelines its copies in between
PIPE_MAX = 16 * Mi
# kvg_scan.cuh HEALTH_STAGE_ROWS x HEALTH_SMALL_THREADS records per TMA round of k_health_small, and
# HEALTH_SMALL_MAX = 32 rows of 1024: above it (or with kernel timing on) k_compact<HealthOp<PciHealthRule>, 256, 8>
HEALTH_ROUND = 12 * 1024
HEALTH_SMALL_MAX = 32 * 1024
# kvg_api_shard.inc FUSED_SEND_MAX: shards from this size on classify, then send with k_shard_send
FUSED_SEND_MAX = 2 * Mi
# kvg_api_mdev.inc load_type_dict: at most 65535 types
MAX_TYPES = 65535
# where the oracle's canonical dump finishes in seconds
ORACLE_PCI_MAX = 2_500_000
ORACLE_MDEV_MAX = 1_100_000


@pytest.fixture(scope="module")
def kv():
    import kvgpu
    return kvgpu


@pytest.fixture(scope="module")
def pciids():
    return util.pciids_text()


@pytest.fixture(scope="module")
def ids(pciids):
    return O.nv_ids(pciids)


@pytest.fixture(scope="module")
def loaded(kv, pciids):
    c = kv.Context(0)
    c.pciids_load(pciids)
    yield c
    c.close()


@pytest.fixture(scope="module")
def names(loaded):
    return loaded.name_table(0, 65536)


def _to_device(recs):
    import torch
    return torch.from_numpy(np.frombuffer(recs.tobytes(), dtype=np.uint8).copy()).cuda()


def _from_device(buf, dtype):
    return np.frombuffer(buf.cpu().numpy().tobytes(), dtype=dtype)


def _pci_on_device(kv, ctx, n, ids, bits, seed):
    """dev_gen_pci records whose iommu groups are rewritten to `bits`-bit keys; record 0 is a certain survivor
    carrying the widest key.  Returns the device buffer and its host copy."""
    import torch
    buf = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    ctx.dev_gen_pci(buf.data_ptr(), seed, n, ids, 0)
    torch.cuda.synchronize()     # the generator ran on the context's stream
    words = buf.view(torch.int32).view(n, 4)
    grp = np.random.default_rng(seed + bits).integers(0, 1 << bits, n, dtype=np.uint64).astype(np.uint32)
    words[:, 2] = torch.from_numpy(grp.view(np.int32)).cuda()
    first = np.zeros(1, dtype=kv.PCI_REC)
    first[0] = (0x0100, 0x10de, int(ids[0]), (1 << bits) - 1, 1, 0, 0)
    words[0] = torch.from_numpy(first.view(np.int32).copy()).cuda()
    torch.cuda.synchronize()
    return buf, _from_device(buf, kv.PCI_REC)


def _pci_dump_oracle(recs, text):
    m = O.Maps()
    m.create_iommu_device_map_flat(np.ascontiguousarray(recs))
    return m.dump(text)


def _launch_labels(ctx, scan):
    """the launch labels of one call of `scan`, with kernel timing on only for it"""
    ctx.set_kernel_timing(True)
    try:
        scan()
        return {name for name, _ in ctx.kernel_times(1 << 16)}
    finally:
        ctx.set_kernel_timing(False)


# ------------------------------------------------------------------------------------------------
# PCI classify, histogram layout / tile scan, digit width, final step (device-resident)
# ------------------------------------------------------------------------------------------------
SIZES_11BIT = [CLASSIFY_SPLIT - 1, CLASSIFY_SPLIT, CLASSIFY_SPLIT + 1, TILESCAN_LONG_ABOVE - 1, TILESCAN_LONG_ABOVE,
               TILESCAN_LONG_ABOVE + 1, 6_000_000, DIGITS8_MIN - 1]
assert TILE_MAJOR_MAX == CLASSIFY_SPLIT   # the first three sizes also straddle the tile-major histogram layout
PCI_POINTS = ([(n, bits) for n in SIZES_11BIT for bits in (22, 32)] +            # 2 and 3 pass sets of 11 bits
              [(n, bits) for n in (DIGITS8_MIN, PIPE_MAX + 3) for bits in (24, 25, 32)])  # 3, 4, 4 sets of 8 bits


@pytest.mark.parametrize("n,bits", PCI_POINTS)
def test_pci_regimes_match_reference(kv, loaded, ids, names, pciids, n, bits):
    buf, recs = _pci_on_device(kv, loaded, n, ids, bits, seed=n % 997)
    loaded.dev_scan_pci(buf.data_ptr(), n)
    res = loaded.dev_scan_pci_fetch()
    assert res.n_records == n
    assert int(res.grp_keys[-1]) == (1 << bits) - 1
    util.check_pci_result(res, recs, names)
    if n <= ORACLE_PCI_MAX and bits == 22:
        assert kv.canonical_dump(kv.pci_maps_from_result(res)) == _pci_dump_oracle(recs, pciids)


@pytest.mark.parametrize("n", [CLASSIFY_SPLIT - 1, CLASSIFY_SPLIT])
def test_pci_split_paths_launch_where_expected(kv, loaded, ids, n):
    """pack_survivors / tile_offsets come only from the split classify, order_count / order_emit only from the
    split final step; order_final only from the chained-scan final step."""
    assert CLASSIFY_SPLIT == FINAL_SPLIT
    buf, _ = _pci_on_device(kv, loaded, n, ids, 22, seed=3)
    labels = _launch_labels(loaded, lambda: loaded.dev_scan_pci(buf.data_ptr(), n))
    split = n >= CLASSIFY_SPLIT
    for lb in ("pack_survivors", "tile_offsets", "order_count", "order_emit"):
        assert (lb in labels) == split, (lb, sorted(labels))
    assert ("order_final" in labels) == (not split), sorted(labels)
    loaded.dev_scan_pci_fetch()


def test_speculated_pass_sets_at_8bit_digits(kv, loaded, ids, names):
    """The wide ordering's pass-set count is speculated from the previous scan's largest key: 8-bit groups,
    then 32-bit groups (4 sets needed, 2 launched: re-run on fetch), then 8-bit groups again, through the fetch
    and through count + fetch."""
    n = DIGITS8_MIN
    for counted in (False, True):
        for bits in (8, 32, 8):
            buf, recs = _pci_on_device(kv, loaded, n, ids, bits, seed=bits + counted)
            loaded.dev_scan_pci(buf.data_ptr(), n)
            if counted:
                s, k, g = loaded.dev_scan_pci_count()
                want = util.expect_pci(recs)
                assert (s, k, g) == (len(want["addr"]), len(np.unique(want["device"])),
                                     len(np.unique(want["iommu_group"]))), bits
            util.check_pci_result(loaded.dev_scan_pci_fetch(), recs, names)
            del buf


def test_deferred_join_on_the_large_paths(kv, ids, pciids):
    """A re-parse on the side stream right before the scan: the split paths join the names late."""
    import torch
    ctx = kv.Context(0)
    try:
        pad = ctx.text_pad(len(pciids))
        h = np.full(pad + 16, 10, dtype=np.uint8)
        h[:len(pciids)] = np.frombuffer(pciids, dtype=np.uint8)
        d_text = torch.from_numpy(h).cuda()
        ctx.dev_pciids_parse(d_text.data_ptr(), len(pciids), pad + 16, 1)          # publishes (synchronous)
        names = ctx.name_table(0, 65536)
        for n in (CLASSIFY_SPLIT + 1, DIGITS8_MIN):
            buf, recs = _pci_on_device(kv, ctx, n, ids, 22, seed=11)
            ctx.dev_pciids_parse(d_text.data_ptr(), len(pciids), pad + 16, 1)      # re-parse: side stream
            ctx.dev_scan_pci(buf.data_ptr(), n)
            res = ctx.dev_scan_pci_fetch()
            util.check_pci_result(res, recs, names)
            assert int((res.survivors["name_slot"] != 0xffffffff).sum()) > 0
            del buf
    finally:
        torch.cuda.synchronize()
        ctx.close()


def test_host_entry_above_the_pipeline(kv, loaded, ids, names):
    """kvg_scan_pci runs the plain path again above PIPE_MAX records: equal to the device-resident scan of the
    same records and to the reference."""
    n = PIPE_MAX + 1
    recs = O.gen_pci(5, n, ids, 24)
    res = loaded.scan_pci(recs)
    util.check_pci_result(res, recs, names)
    buf = _to_device(recs)
    loaded.dev_scan_pci(buf.data_ptr(), n)
    dev = loaded.dev_scan_pci_fetch()
    assert np.array_equal(res.survivors, dev.survivors)
    for f in ("dev_keys", "dev_off", "dev_perm", "dev_name_slot", "grp_keys", "grp_off", "grp_perm"):
        assert np.array_equal(getattr(res, f), getattr(dev, f)), f


def test_pinned_pciids_load(kv, loaded, pciids, ids, names):
    """kvg_pciids_load reads pinned caller memory in place (it only enqueues the parse): lookups, the name table
    and a scan must equal those of the pageable load, with the buffer alive until they return."""
    import ctypes as C
    import torch
    lib = kv.load()
    ctx = kv.Context(0)
    try:
        pinned = torch.empty(len(pciids), dtype=torch.uint8, pin_memory=True)
        pinned.numpy()[:] = np.frombuffer(pciids, dtype=np.uint8)
        assert lib.kvg_pciids_load(ctx.handle, C.c_void_p(pinned.data_ptr()), len(pciids)) == 0
        for k in ("1b38", "2901", "1b3", "", "ffff", "10de", "0008  NV1"):
            assert ctx.name_lookup(k) == loaded.name_lookup(k), k
        assert ctx.name_table(0, 65536) == names
        recs = O.gen_pci(9, 300_001, ids, 18)
        got, want = ctx.scan_pci(recs), loaded.scan_pci(recs)
        util.check_pci_result(got, recs, names)
        assert kv.canonical_dump(kv.pci_maps_from_result(got)) == kv.canonical_dump(kv.pci_maps_from_result(want))
        del pinned
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------
# mdev: type ordering (16-bit keys), parent ordering (32-bit keys), dictionary sizes
# ------------------------------------------------------------------------------------------------
def _types(nt):
    """nt raw type names: even entries distinct, each odd entry a white-space variant of the one before (merges)"""
    out = []
    for k in range(nt):
        sep = b" \t " if k & 1 else b" "
        out.append(b"NVIDIA%sV%05d-%dQ\n" % (sep, k >> 1, 1 << ((k >> 1) % 5)))
    return out


def _mdev_records(kv, n, parent_bits, nt, seed):
    """gen_mdev records rewritten: parents of `parent_bits` bits, type indices past the dictionary, every flag
    combination.  Record 0 is a certain survivor with the widest parent and the largest type index."""
    recs = O.gen_mdev(seed, n)
    rng = np.random.default_rng(seed)
    recs["parent"] = rng.integers(0, 1 << parent_bits, n, dtype=np.uint64).astype(np.uint32)
    recs["type_idx"] = rng.integers(0, min(nt + max(2, nt // 16), 1 << 16), n).astype(np.uint16)
    recs["flags"] = np.where(rng.integers(0, 2, n) == 0, 0, rng.integers(0, 8, n)).astype(np.uint8)
    recs["parent_numa"] = rng.integers(-2, 4, n).astype(np.int16)
    recs["parent"][0], recs["type_idx"][0], recs["flags"][0] = (1 << parent_bits) - 1, nt - 1, 0
    if n > 1:   # a packed BDF with a domain
        recs["parent"][1], recs["flags"][1] = (0x0001 << 16 | 0x3b << 8 | 0x1f << 3 | 7) & ((1 << parent_bits) - 1), 0
    return recs


MDEV_CASES = [  # n, parent bits, dictionary size
    (1_000, 1, 1), (65_536, 11, 2048), (70_001, 12, 2049), (1_048_577, 32, 2049),
    (CLASSIFY_SPLIT - 1, 22, 2048), (CLASSIFY_SPLIT, 23, MAX_TYPES), (CLASSIFY_SPLIT + 1, 25, 2049),
    (TILESCAN_LONG_ABOVE - 1, 32, 2049), (TILESCAN_LONG_ABOVE, 12, 1), (TILESCAN_LONG_ABOVE + 1, 23, MAX_TYPES),
    (6_000_000, 22, 2049), (DIGITS8_MIN - 1, 25, 2048), (DIGITS8_MIN + 5, 32, MAX_TYPES), (DIGITS8_MIN + 5, 11, 2049),
]


@pytest.mark.parametrize("n,parent_bits,nt", MDEV_CASES)
def test_mdev_regimes_match_reference(kv, loaded, pciids, n, parent_bits, nt):
    types = _types(nt)
    labels, canon = util.mdev_labels(types)
    assert len(set(labels)) == (nt + 1) // 2 and (nt < 2 or canon[1] == 0)   # the pairs merge
    recs = _mdev_records(kv, n, parent_bits, nt, seed=n % 1009 + nt)
    if MDEV_CASES.index((n, parent_bits, nt)) & 1:   # host entry point
        res = loaded.scan_mdev(recs, types)
    else:                                             # device-resident entry point
        buf = _to_device(recs)
        loaded.dev_scan_mdev(buf.data_ptr(), n, types)
        res = loaded.dev_scan_mdev_fetch()
        del buf
    assert res.n_records == n
    assert int(res.par_keys[-1]) == (1 << parent_bits) - 1
    util.check_mdev_result(res, recs, types)
    assert int(res.type_keys[-1]) == canon[nt - 1]
    if n <= ORACLE_MDEV_MAX:
        m = O.Maps()
        m.create_vgpu_id_map_flat(recs, types)
        assert kv.canonical_dump(kv.mdev_maps_from_result(res)) == m.dump(pciids)


@pytest.mark.parametrize("n", [CLASSIFY_SPLIT - 1, CLASSIFY_SPLIT])
def test_mdev_final_step_launches_where_expected(kv, loaded, n):
    recs = _mdev_records(kv, n, 22, 2049, seed=4)
    buf = _to_device(recs)
    labels = _launch_labels(loaded, lambda: loaded.dev_scan_mdev(buf.data_ptr(), n, _types(2049)))
    split = n >= FINAL_SPLIT
    assert ("order_count" in labels) == split and ("order_emit" in labels) == split, sorted(labels)
    assert ("order_final" in labels) == (not split), sorted(labels)
    loaded.dev_scan_mdev_fetch()


def test_mdev_dictionary_limit(kv, loaded):
    recs = O.gen_mdev(0, 16)
    with pytest.raises(kv.KvgError) as e:
        loaded.scan_mdev(recs, [b"t\n"] * (MAX_TYPES + 1))
    assert e.value.rc == -6      # KVG_ERANGE
    res = loaded.scan_mdev(recs, [b"t\n"] * MAX_TYPES)      # the context is still usable
    util.check_mdev_result(res, recs, [b"t\n"] * MAX_TYPES)


# ------------------------------------------------------------------------------------------------
# vGPU resource names longer than 256 bytes
# ------------------------------------------------------------------------------------------------
def test_long_vgpu_names_are_whole(kv, pciids):
    """getDeviceName(label) returns the whole sanitised rest of the first matching line, however long."""
    import torch
    text, types = util.long_name_pciids(), util.long_name_types()
    recs = O.gen_mdev(0, 4096)
    recs["type_idx"] %= len(types)
    m = O.Maps()
    m.create_vgpu_id_map_flat(recs, types)
    want_dump = m.dump(text)
    ctx = kv.Context(0)
    try:
        ctx.pciids_load(text)
        for rep in range(2):
            res = ctx.scan_mdev(recs, types)
            want = [O.get_device_name(text, lb) for lb in res.labels]
            assert [len(x) for x in res.type_names] == [len(x) for x in want], rep
            assert res.type_names == want
            assert max(len(x) for x in want) == max(util.LONG_NAME_LENGTHS)
            assert kv.canonical_dump(kv.mdev_maps_from_result(res)) == want_dump
            # short names again in the same context: slots of the first size
            short = ctx.scan_mdev(recs, [b"1b38\n", b"ab09\n"])
            assert short.type_names == [O.get_device_name(text, b"1b38"), ""]
        buf = _to_device(recs)
        ctx.dev_scan_mdev(buf.data_ptr(), len(recs), types)
        res = ctx.dev_scan_mdev_fetch()
        assert res.type_names == want
        util.check_mdev_result(res, recs, types)
        del buf
    finally:
        torch.cuda.synchronize()
        ctx.close()
    # the shipped pci.ids: every name fits the first slot size
    with kv.Context(0) as c:
        c.pciids_load(pciids)
        res = c.scan_mdev(recs, [b"1b38\n", b"2901\n", b"GRID P40-1Q\n"])
        assert res.type_names == [O.get_device_name(pciids, k) for k in (b"1b38", b"2901", b"GRID_P40-1Q")]


def _run_worker(args, port, timeout):
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(here, "_nccl_worker.py")] + args
    env = dict(os.environ, KVG_WORKER_STALL_S=str(timeout - 30))
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return r.stdout


def test_long_vgpu_names_sharded():
    """The sharded mdev fetch at world 1 (its own name area) against the oracle on the long-name table."""
    out = _run_worker(["5", "p2p", "4096", "long-names"], 29650, 300)
    assert "nccl-ok world=1 n=5" in out and "exchange=p2p" in out, out[-2000:]


def test_sharded_standalone_send_over_peer_windows():
    """A shard of FUSED_SEND_MAX + 5 records in p2p mode: classify, then k_shard_send into a peer window."""
    n = FUSED_SEND_MAX + 5
    out = _run_worker([str(n), "p2p"], 29651, 600)
    assert "nccl-ok world=1 n=%d" % n in out and "exchange=p2p" in out, out[-2000:]


# ------------------------------------------------------------------------------------------------
# health re-scan
# ------------------------------------------------------------------------------------------------
HEALTH_SIZES = [1, HEALTH_ROUND, HEALTH_ROUND + 1, 2 * HEALTH_ROUND + 1, HEALTH_SMALL_MAX, HEALTH_SMALL_MAX + 1,
                100_000]


def _flip_points(n, rng):
    edges = [0, n - 1]
    for b in (1024, HEALTH_ROUND, 2 * HEALTH_ROUND, HEALTH_SMALL_MAX):   # row and round boundaries
        edges += [b - 1, b, b + 1]
    pts = [p for p in edges if 0 <= p < n] + list(rng.integers(0, n, 8))
    return np.unique(np.array(pts, dtype=np.int64))


@pytest.mark.parametrize("pinned", [False, True])
def test_health_regimes(kv, ids, pinned):
    """Ticks with flips on row / round boundaries at every size regime, pageable and pinned snapshots (pinned:
    changed in place), sizes changed between calls (the state re-arms), and kernel timing switched on for one
    tick (k_compact<HealthOp<PciHealthRule>, 256, 8> on the same state) and off again."""
    import torch
    ctx = kv.Context(0)
    rng = np.random.default_rng(17 + pinned)
    keep = []
    try:
        ctx.health_reset()
        for n in HEALTH_SIZES + [HEALTH_ROUND, 1]:
            if pinned:
                t = torch.empty(n * 16, dtype=torch.uint8, pin_memory=True)
                keep.append(t)
                recs = t.numpy().view(kv.PCI_REC)
                recs[:] = O.gen_pci(n, n, ids, 0)
            else:
                recs = O.gen_pci(n, n, ids, 0)
            prev = np.zeros(n, dtype=bool)      # a new size re-arms: everything alive is a transition
            for tick in range(5):
                if tick:
                    f = _flip_points(n, rng)
                    recs["driver"][f] = rng.integers(0, 5, len(f))
                    recs["flags"][f] ^= rng.integers(0, 32, len(f)).astype(np.uint8)
                timed = tick == 2
                if timed:
                    ctx.set_kernel_timing(True)
                d = ctx.health_rescan(recs)
                if timed:
                    labels = {name for name, _ in ctx.kernel_times(1 << 16)}
                    ctx.set_kernel_timing(False)
                    # timing moves every size to k_compact<HealthOp<PciHealthRule>, 256, 8>; the untimed ticks
                    # around it run k_health_small up to HEALTH_SMALL_MAX records, on the same alive-set
                    assert "health_compact" in labels and "health_small" not in labels, sorted(labels)
                now = util.pci_alive(recs)
                idx = np.nonzero(now != prev)[0]
                want = (idx.astype(np.uint32) << 1) | now[idx].astype(np.uint32)
                assert d.n_records == n and d.n_alive == int(now.sum()), (n, tick)
                assert np.array_equal(d.changed, want), (n, tick, len(d.changed), len(want))
                prev = now
        ctx.health_reset()
        d = ctx.health_rescan(np.zeros(0, dtype=kv.PCI_REC))
        assert (d.n_records, d.n_alive, len(d.changed)) == (0, 0, 0)
    finally:
        torch.cuda.synchronize()
        ctx.close()
        del keep
