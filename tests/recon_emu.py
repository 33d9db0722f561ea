"""TEST INFRASTRUCTURE: the host-emulator build of the mesh-extraction unit, tests/cuda_emu/_build/libpnr_emu_recon.so.

It is tests/cuda_emu/build_emu.py's library (the same rewrite of the launches, the same translation units and
stubs) plus csrc/pnr_recon.cu, compiled with a prelude that gives the emulator the float64 round-to-nearest
intrinsics pnr_recon.cu uses.  On x86-64 with -ffp-contract=off each is one IEEE operation, as on the GPU.
"""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import emu_util as eu

sys.path.insert(0, os.path.join(eu.ROOT, "tests", "cuda_emu"))
import build_emu  # noqa: E402

UNITS = build_emu.UNITS + ["pnr_recon.cu"]
PRELUDE = """#pragma once
#include "cuda_runtime.h"
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline float __double2float_rn(double x) { return (float)x; }
"""

_lib = None


def build():
    out = build_emu.OUT
    os.makedirs(out, exist_ok=True)
    h = hashlib.sha256(PRELUDE.encode())
    for d in (build_emu.CSRC, build_emu.HERE):
        for name in sorted(os.listdir(d)):
            if name.split(".")[-1] in ("cu", "cuh", "h", "cpp", "py"):
                h.update(open(os.path.join(d, name), "rb").read())
    h.update(open(os.path.join(eu.ROOT, "include", "pnr.h"), "rb").read())
    lib = os.path.join(out, "libpnr_emu_recon.so")
    stamp = os.path.join(out, "stamp_recon")
    if os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest():
        return lib
    prelude = os.path.join(out, "recon_prelude.h")
    with open(prelude, "w") as f:
        f.write(PRELUDE)
    texts = {u: open(os.path.join(build_emu.CSRC, u)).read() for u in UNITS}
    modes = build_emu.classify(texts.values())
    srcs = []
    for u in UNITS:
        dst = os.path.join(out, u.replace(".cu", "_recon_emu.cpp"))
        with open(dst, "w") as f:
            f.write(build_emu.rewrite(texts[u], modes))
        srcs.append(dst)
    srcs.append(os.path.join(build_emu.HERE, "emu_stubs.cpp"))
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fno-omit-frame-pointer", "-ffp-contract=off",
                    "-w", "-I", build_emu.HERE, "-I", build_emu.CSRC, "-include", prelude, "-o", lib] + srcs,
                   check=True)
    with open(stamp, "w") as f:
        f.write(h.hexdigest())
    return lib


def lib():
    global _lib
    if _lib is None:
        _lib = eu.pn.declare(C.CDLL(build()))
    return _lib
