"""k_mdev_label_match (kvg_mdev_label_match's kernel) executed on the CPU from its real source under the warp emulator of
tools/emu/, in its launch shape (one CTA, one thread per file, striding), against the label rule of the vGPU plugin's
CPU path (serve._read_vgpu_label) on files written to disk and on generated ones."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import conftest
import label_match_cases as LM

sys.path.insert(0, os.path.join(conftest.ROOT, "tools", "emu"))
import build as emu_build  # noqa: E402

THREADS = 1024  # LABEL_MATCH_THREADS


@pytest.fixture(scope="module")
def emu():
    L = C.CDLL(emu_build.build_classify())
    L.emu_mdev_label_match.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint64, C.c_void_p,
                                       C.c_void_p]
    return L


def run(emu, files, name):
    """What the host stages: the offsets, the raw bytes and at most as many name bytes as there are raw bytes."""
    off = np.zeros(len(files) + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(f) for f in files])
    raw = np.frombuffer(b"".join(files) + b"\0", dtype=np.uint8)
    match = np.full(len(files), 0xee, dtype=np.uint8)
    seq = np.zeros(1, dtype=np.uint32)
    assert emu.emu_mdev_label_match(raw.ctypes.data, off.ctypes.data, len(files), name[:int(off[-1])], len(name),
                                    match.ctypes.data, seq.ctypes.data) == 0
    assert int(seq[0]) == 7
    assert set(np.unique(match)) <= {0, 1}
    return match.astype(bool)


def test_reference_rule_is_the_plugins(tmp_path):
    """ref_label (used for the large generated sets) is exactly what the plugin's CPU reader returns."""
    from kvgpu import serve
    for i, raw in enumerate(LM.EDGES):
        d = tmp_path / str(i) / "mdev_type"
        d.mkdir(parents=True)
        (d / "name").write_bytes(raw)
        label, err = serve._read_vgpu_label(str(tmp_path), str(i), "mdev_type/name")
        assert not err and label.encode("latin-1") == LM.ref_label(raw), raw[:40]
    assert LM.ref_label(b"\r\nX\r\n") == b"_X_"
    assert LM.ref_label(LM.BIG) == LM.NAME and len(LM.BIG) > 64 * 1024


@pytest.mark.parametrize("name", LM.edge_names())
def test_edges(emu, name):
    assert np.array_equal(run(emu, LM.EDGES, name), LM.want(LM.EDGES, name)), name


def test_one_file(emu):
    for raw in LM.EDGES:
        lb = LM.ref_label(raw)
        assert run(emu, [raw], lb)[0]
        assert not run(emu, [raw], lb + b"_")[0]


@pytest.mark.parametrize("n", [THREADS - 1, THREADS + 1, 2 * THREADS + 517])
def test_threads_stride_over_more_files_than_the_cta_has(emu, n):
    rng = np.random.default_rng(n)
    files = LM.random_files(n, rng, big_every=997)
    for name in (LM.NAME, b"GRID_A100-4Q", b""):
        got, want = run(emu, files, name), LM.want(files, name)
        assert np.array_equal(got, want), name
    assert 0 < LM.want(files, LM.NAME).sum() < n
