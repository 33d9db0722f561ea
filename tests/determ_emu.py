"""TEST INFRASTRUCTURE: the host-emulator build with deterministic mode, tests/cuda_emu/_build/libpnr_emu_determ.so.

It is tests/cuda_emu/build_emu.py's library (the same rewrite of the launches, the same translation units and
stubs) plus csrc/pnr_determ.cu, compiled with a prelude that gives the emulator the bit casts, the 32- and 64-bit
integer atomics and the rounding conversions that unit uses.  The emulator runs one thread at a time, so an atomic is
a plain read-modify-write; each conversion is one IEEE operation in round-to-nearest-even, as on the GPU.

The library also reports every chunk the fixed-point latent scatter receives: `latent_scatter_fixed` calls the hook
`pnr_emu_chunk_hook(g0, n, d_lat, count)` first when a test has set it, so that a test can replay the chunks through
oracle/pnr_determinism.py.  The hook only reads the chunk's inputs.
"""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import numpy as np

import emu_util as eu

sys.path.insert(0, os.path.join(eu.ROOT, "tests", "cuda_emu"))
import build_emu  # noqa: E402

UNITS = build_emu.UNITS + ["pnr_determ.cu"]
PRELUDE = """#pragma once
#include <cmath>
#include <cstring>
#include "cuda_runtime.h"
static inline unsigned __float_as_uint(float x) { unsigned u; memcpy(&u, &x, 4); return u; }
static inline float __uint_as_float(unsigned u) { float x; memcpy(&x, &u, 4); return x; }
static inline float __int_as_float(int i) { float x; memcpy(&x, &i, 4); return x; }
static inline unsigned atomicMax(unsigned* p, unsigned v) { const unsigned old = *p; if (v > old) *p = v; return old; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) {
  const unsigned long long old = *p;
  *p = old + v;
  return old;
}
static inline long long __double2ll_rn(double x) { return std::llrint(x); }
static inline double __ll2double_rn(long long a) { return (double)a; }
static inline float __double2float_rn(double x) { return (float)x; }
"""

HOOK_DECL = "int latent_scatter_fixed("
HOOK_CALL = "  if (pnr_emu_chunk_hook) pnr_emu_chunk_hook(g0, n, d_lat, n * sc.NS * sc.C);\n"
PRELUDE += """#include <cstdint>
extern "C" __attribute__((weak)) void (*pnr_emu_chunk_hook)(int64_t, int64_t, const float*, int64_t) = nullptr;
"""
HOOK_TYPE = C.CFUNCTYPE(None, C.c_int64, C.c_int64, C.POINTER(C.c_float), C.c_int64)


def _with_hook(text):
    i = text.index(HOOK_DECL)
    j = text.index("{\n", i) + 2
    return text[:j] + HOOK_CALL + text[j:]


_lib = None


def build():
    out = build_emu.OUT
    os.makedirs(out, exist_ok=True)
    h = hashlib.sha256((PRELUDE + HOOK_CALL).encode())
    for d in (build_emu.CSRC, build_emu.HERE):
        for name in sorted(os.listdir(d)):
            if name.split(".")[-1] in ("cu", "cuh", "h", "cpp", "py"):
                h.update(open(os.path.join(d, name), "rb").read())
    h.update(open(os.path.join(eu.ROOT, "include", "pnr.h"), "rb").read())
    lib = os.path.join(out, "libpnr_emu_determ.so")
    stamp = os.path.join(out, "stamp_determ")
    if os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest():
        return lib
    prelude = os.path.join(out, "determ_prelude.h")
    with open(prelude, "w") as f:
        f.write(PRELUDE)
    texts = {u: open(os.path.join(build_emu.CSRC, u)).read() for u in UNITS}
    texts["pnr_determ.cu"] = _with_hook(texts["pnr_determ.cu"])
    modes = build_emu.classify(texts.values())
    srcs = []
    for u in UNITS:
        dst = os.path.join(out, u.replace(".cu", "_determ_emu.cpp"))
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


def set_chunk_hook(fn):
    """fn(g0, n, d_lat float32 array [count]) for every chunk of the fixed-point scatter, or None.  Returns the ctypes
    callback, which the caller keeps alive while it is set."""
    cb = HOOK_TYPE(lambda g0, n, p, count: fn(g0, n, np.ctypeslib.as_array(p, (count,)).copy())) if fn else None
    C.c_void_p.in_dll(lib(), "pnr_emu_chunk_hook").value = C.cast(cb, C.c_void_p).value if cb else None
    return cb
