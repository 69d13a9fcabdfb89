#!/usr/bin/env python3
"""Build the CPU twins of the CUDA kernels (tools/emu/_build/lib*_emu.so): each harness <name>_emu.cpp includes
warp_emu.h and then the kernel headers of csrc/ whole, so the emulator compiles the same text nvcc compiles."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200", "csrc")
OUT = os.path.join(HERE, "_build")


def build(name: str, force: bool = False) -> str:
    """lib<name>_emu.so from <name>_emu.cpp; rebuilt when older than any header it may include (every
    csrc/*.cuh, as the Makefile's HDRS rule does), the emulator, the harness or this script."""
    os.makedirs(OUT, exist_ok=True)
    lib = os.path.join(OUT, "lib%s_emu.so" % name)
    cpp = os.path.join(HERE, "%s_emu.cpp" % name)
    srcs = glob.glob(os.path.join(CSRC, "*.cuh")) + [
        os.path.join(ROOT, "include", "kvgpu.h"), os.path.join(HERE, "warp_emu.h"), cpp, __file__]
    if not force and os.path.exists(lib) and all(os.path.getmtime(lib) >= os.path.getmtime(s) for s in srcs):
        return lib
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
           "-Wno-unknown-pragmas", "-I", HERE, cpp, "-o", lib]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stderr)
        raise RuntimeError("emulation build failed")
    return lib


def build_radix(force: bool = False) -> str:
    return build("radix", force)


def build_shard(force: bool = False) -> str:
    return build("shard", force)


def build_classify(force: bool = False) -> str:
    return build("classify", force)


def build_names(force: bool = False) -> str:
    return build("names", force)


def build_delta(force: bool = False) -> str:
    return build("delta", force)


if __name__ == "__main__":
    for name in ("radix", "shard", "classify", "names", "delta", "health_raw"):
        print(build(name, force=True))
