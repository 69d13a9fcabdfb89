"""Raw mdev_type/name contents for the vGPU plugin's Allocate-time label check (kvg_mdev_label_match), and the
label rule as the plugin's CPU path applies it (serve._read_vgpu_label)."""
import re

import numpy as np

NAME = b"GRID_A100-4C"
RE2_SPACE = (b" ", b"\t", b"\n", b"\f", b"\r")

# > 64 KiB of raw text that collapses to NAME: newline runs on both ends, one long run of all five spaces inside
BIG = b"\n" * 7 + b"GRID" + b" \t\r\f\n" * 14_000 + b"A100-4C" + b"\n" * 9

EDGES = [
    b"\n\n\nGRID A100-4C\n\n",          # leading and trailing \n runs
    b"GRID A100-4C\n",
    b"\r\nX\r\n",                        # a \r before the trailing \n: "_X_"
    b"GRID \t\n\f\r A100-4C",           # one run of all five RE2 spaces
    b"GRID\r\n\tA100-4C\f",
    b"GRID\vA100-4C",                   # \v, 0x85, 0xA0 and NUL are not RE2 \s: kept verbatim
    b"GRID\x85A100-4C",
    b"GRID\xa0A100-4C",
    b"GRID\x00A100-4C",
    b"",                                 # empty file
    b"\n",
    b"\n\n\n\n",                         # only newlines
    b"GRID__A100-4C",                   # a literal __ stays two bytes
    b"GRID_ A100-4C",
    b"GRID A100-4",                      # the label is a prefix of NAME
    b"GRID A100-4C-x",                   # NAME is a prefix of the label
    b" GRID A100-4C",
    b"GRID A100-4C \n",
    BIG,
]


def ref_label(raw: bytes) -> bytes:
    """Trim(raw, "\\n") then every RE2 \\s+ run -> "_" (device_plugin.go:341-342), as serve._read_vgpu_label does."""
    return re.sub(rb"[\t\n\f\r ]+", b"_", raw.strip(b"\n"))


def edge_names():
    """Every label of EDGES, each one byte shorter and one byte longer, and the empty name."""
    out = {b"", b"_", NAME, NAME + b"x"}
    for raw in EDGES:
        lb = ref_label(raw)
        out |= {lb, lb[:-1], lb + b"C"}
    return sorted(out)


def random_files(n, rng, big_every=0):
    """n raw files, most of which are NAME written with other space runs, others near misses or noise; every
    big_every-th file (if > 0) is BIG."""
    noise = [b"A", b"G", b"_", b"-", b"\v", b"\x85", b"\xa0", b"\x00"] + list(RE2_SPACE)
    out = []
    for i in range(n):
        if big_every and i % big_every == 0:
            out.append(BIG)
            continue
        k = int(rng.integers(0, 8))
        if k == 0:
            out.append(b"".join(noise[j] for j in rng.integers(0, len(noise), int(rng.integers(0, 24)))))
            continue
        run = b"".join(RE2_SPACE[j] for j in rng.integers(0, 5, int(rng.integers(1, 4))))
        raw = b"\n" * int(rng.integers(0, 3)) + b"GRID" + run + b"A100-4C" + b"\n" * int(rng.integers(0, 3))
        if k == 1:
            raw = raw.replace(b"4C", b"4Q")
        elif k == 2:
            raw += b"\r"
        out.append(raw)
    return out


def want(files, name):
    return np.array([ref_label(f) == name for f in files], dtype=bool)
