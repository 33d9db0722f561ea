"""TEST INFRASTRUCTURE: the host-emulator build of the mesh-components unit, tests/cuda_emu/_build/libpnr_emu_mesh.so.

It is tests/recon_emu.py's library (the same rewrite of the launches, the same translation units, stubs and
float64 intrinsics) plus csrc/pnr_mesh.cu, whose prelude also gives the emulator the 64-bit integer atomics that unit
uses.  The emulator runs one thread at a time, so an atomic is a plain read-modify-write there; the union-find then
hooks in one fixed order, and only the GPU runs it concurrently.
"""
import ctypes as C
import hashlib
import os
import subprocess

import emu_util as eu
import recon_emu
from recon_emu import build_emu

UNITS = recon_emu.UNITS + ["pnr_mesh.cu"]
PRELUDE = recon_emu.PRELUDE + """static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) {
  const unsigned long long old = *p;
  *p = old + v;
  return old;
}
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  const unsigned long long old = *p;
  if (old == cmp) *p = v;
  return old;
}
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
    lib = os.path.join(out, "libpnr_emu_mesh.so")
    stamp = os.path.join(out, "stamp_mesh")
    if os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest():
        return lib
    prelude = os.path.join(out, "mesh_prelude.h")
    with open(prelude, "w") as f:
        f.write(PRELUDE)
    texts = {u: open(os.path.join(build_emu.CSRC, u)).read() for u in UNITS}
    modes = build_emu.classify(texts.values())
    srcs = []
    for u in UNITS:
        dst = os.path.join(out, u.replace(".cu", "_mesh_emu.cpp"))
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
