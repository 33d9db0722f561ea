"""pnr_mgpu_field_eval (csrc/pnr_mgpu_field.cu, the sharded field evaluation behind `util.recon.marching_cubes(...,
gpus=...)`) on the host emulator with the SIMT engine: for grid, band-lattice, band-refinement (apron 0 and 1) and
point-list sources, 1 to 4 shards on emulated devices -- repeated devices, ragged last chunks, more shards than chunks,
no points -- the stored channels are bit for bit those of ONE pnr_field_eval loop over the same chunks.  The emulator
gives a repeated device no peer access to device 0, so `[0, 0]` takes the staging path and `[0, 1]` the peer stores.
Also the error codes and a gcc probe of the new structs against their ctypes mirrors."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest
import torch

import emu_util as eu
import golden_util as gu
import recon_emu

pn = eu.pn
build_emu = recon_emu.build_emu

PNR_ERR_INVALID, PNR_ERR_WORKSPACE = -1, -2
UNITS = recon_emu.UNITS + ["pnr_mgpu_field.cu"]
LO, HI = (-0.4, -0.35, -0.3), (0.45, 0.4, 0.5)

_lib = None


def lib():
    """tests/cuda_emu/_build/libpnr_emu_mgpu_recon.so: the mesh-extraction emulator build plus the sharded field."""
    global _lib
    if _lib is not None:
        return _lib
    out = build_emu.OUT
    os.makedirs(out, exist_ok=True)
    h = hashlib.sha256(recon_emu.PRELUDE.encode())
    for d in (build_emu.CSRC, build_emu.HERE):
        for name in sorted(os.listdir(d)):
            if name.split(".")[-1] in ("cu", "cuh", "h", "cpp", "py"):
                h.update(open(os.path.join(d, name), "rb").read())
    h.update(open(os.path.join(eu.ROOT, "include", "pnr.h"), "rb").read())
    path = os.path.join(out, "libpnr_emu_mgpu_recon.so")
    stamp = os.path.join(out, "stamp_mgpu_recon")
    if not (os.path.exists(path) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest()):
        prelude = os.path.join(out, "mgpu_recon_prelude.h")
        with open(prelude, "w") as f:
            f.write(recon_emu.PRELUDE)
        texts = {u: open(os.path.join(build_emu.CSRC, u)).read() for u in UNITS}
        modes = build_emu.classify(texts.values())
        srcs = []
        for u in UNITS:
            dst = os.path.join(out, u.replace(".cu", "_mgpu_recon_emu.cpp"))
            with open(dst, "w") as f:
                f.write(build_emu.rewrite(texts[u], modes))
            srcs.append(dst)
        srcs.append(os.path.join(build_emu.HERE, "emu_stubs.cpp"))
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fno-omit-frame-pointer", "-ffp-contract=off",
                        "-w", "-I", build_emu.HERE, "-I", build_emu.CSRC, "-include", prelude, "-o", path] + srcs,
                       check=True)
        with open(stamp, "w") as f:
            f.write(h.hexdigest())
    _lib = pn.declare(C.CDLL(path))
    return _lib


def ok(rc):
    assert rc == 0, lib().pnr_last_error().decode()


def r3(reso):
    return (C.c_int32 * 3)(*reso)


def b3():
    return (C.c_double * 3)(*LO), (C.c_double * 3)(*HI)


class Scene:
    """The SB = 1 golden case "tiny" as a PnrScene / coarse PnrMlp over CPU tensors."""

    def __init__(self):
        case = gu.load_case("tiny")
        self.keep = []
        self.scene = eu.scene_struct(case, gu.oracle_state(case), self.keep)
        self.mlp = eu.mlp_struct(case["wc"], case["cfg"]["d_hidden"])
        self.keep.append(case)


_SCENE = None


def scene():
    global _SCENE
    if _SCENE is None:
        _SCENE = Scene()
    return _SCENE


def band_plan(reso, block, apron):
    """A plan whose lattice sigma is inside at the first lattice point only: block 0 is seeded and it and its
    neighbours are refined -> (plan tensor, bytes, refinement points)."""
    L = lib()
    m = [(n - 1 + block - 1) // block + 1 for n in reso]
    coarse = torch.full((int(np.prod(m)),), -1.0)
    coarse[0] = 1.0
    nbytes = int(L.pnr_band_plan_bytes(r3(reso), block, apron))
    plan = torch.zeros(nbytes, dtype=torch.uint8)
    counts = torch.zeros(2, dtype=torch.int64)
    ok(L.pnr_band_plan(eu.ptr(coarse), r3(reso), block, 0.0, apron, C.c_void_p(counts.data_ptr()),
                       C.c_void_p(plan.data_ptr()), nbytes, None))
    return plan, nbytes, int(counts[1])


def make_source(kind, reso=(4, 3, 5), block=2, apron=0, count=None):
    """-> (PnrPointSource, count, points(first, n, xyz, vd) for the one-GPU loop, plan or None, kept tensors)"""
    L = lib()
    lo, hi = b3()
    if kind == pn.POINTS_GRID:
        src = pn.point_source(kind, LO, HI, reso)
        n = int(np.prod(reso))
        return src, n if count is None else count, lambda f, k, x, d: ok(
            L.pnr_grid_points(lo, hi, r3(reso), f, k, eu.ptr(x), eu.ptr(d), None)), None, []
    if kind == pn.POINTS_LATTICE:
        src = pn.point_source(kind, LO, HI, reso, block)
        n = int(np.prod([(r - 1 + block - 1) // block + 1 for r in reso]))
        return src, n if count is None else count, lambda f, k, x, d: ok(
            L.pnr_band_lattice_points(lo, hi, r3(reso), block, f, k, eu.ptr(x), eu.ptr(d), None)), None, []
    if kind == pn.POINTS_BAND:
        plan, nbytes, M = band_plan(reso, block, apron)
        src = pn.point_source(kind, LO, HI, reso, block, apron, M)
        pp = C.c_void_p(plan.data_ptr())
        return src, M, lambda f, k, x, d: ok(L.pnr_band_points(lo, hi, r3(reso), block, apron, pp, nbytes, M, f, k,
                                                               eu.ptr(x), eu.ptr(d), None)), (plan, nbytes), []
    n = 29 if count is None else count                  # POINTS_LIST: points and unit view directions on "device 0"
    g = torch.Generator().manual_seed(3)
    xyz = (torch.rand(n, 3, generator=g) - 0.5) * 0.8
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=1).contiguous()
    src = pn.PnrPointSource()
    src.kind, src.xyz0, src.viewdirs0 = kind, eu.ptr(xyz), eu.ptr(vd)

    def points(f, k, x, d):
        x[:k] = xyz[f:f + k]
        d[:k] = vd[f:f + k]
    return src, n, points, None, [xyz, vd]


def one_gpu(points, count, chunk, channel, nc):
    """the one-GPU loop: pnr_field_eval per chunk of `chunk` points from 0 -> [count, nc]"""
    L, sc = lib(), scene()
    out = torch.full((count, nc), float("nan"))
    xyz, vd, field = torch.empty(chunk, 3), torch.empty(chunk, 3), torch.empty(chunk, 4)
    nbytes = L.pnr_field_workspace_bytes(sc.scene, sc.mlp, chunk, pn.ENGINE_SIMT)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8)
    for first in range(0, count, chunk):
        n = min(chunk, count - first)
        points(first, n, xyz, vd)
        ok(L.pnr_field_eval(sc.scene, sc.mlp, eu.ptr(xyz), eu.ptr(vd), eu.ptr(field), n, pn.ENGINE_SIMT,
                            ws.data_ptr(), nbytes, None))
        out[first:first + n] = field[:n, channel:channel + nc]
    return out


def sharded(devices, src, count, chunk, channel, nc, plan=None, ws_bytes=None, fill=-7.0):
    """pnr_mgpu_field_eval over `devices` -> (rc, out [count, nc])"""
    L, sc = lib(), scene()
    n = len(devices)
    h = C.c_void_p()
    ok(L.pnr_mgpu_create((C.c_int32 * n)(*devices), n, C.byref(h)))
    shards = (pn.PnrFieldShard * n)()
    need = L.pnr_mgpu_field_workspace_bytes(sc.scene, sc.mlp, chunk, pn.ENGINE_SIMT)
    keep = []
    for i in range(n):
        sh = shards[i]
        sh.scene, sh.mlp = C.pointer(sc.scene), C.pointer(sc.mlp)
        b = need if ws_bytes is None else ws_bytes
        ws = torch.full((max(b, 1),), 0xAB, dtype=torch.uint8)     # each shard its own workspace, garbage-filled
        sh.workspace, sh.workspace_bytes = ws.data_ptr(), b
        if plan is not None:
            copy = plan[0].clone()                                 # each device its own copy of the plan
            sh.plan, sh.plan_bytes = copy.data_ptr(), plan[1]
            keep.append(copy)
        keep.append(ws)
    out = torch.full((max(count, 1), max(nc, 1)), fill)
    rc = L.pnr_mgpu_field_eval(h, shards, C.byref(src), count, chunk, pn.ENGINE_SIMT, channel, nc, eu.ptr(out), None)
    if rc == 0:
        assert L.pnr_mgpu_size(h) == n
    ok(L.pnr_mgpu_destroy(h))
    return rc, out[:count]


def bits(a, b):
    assert a.shape == b.shape
    assert np.array_equal(a.numpy().view(np.int32), b.numpy().view(np.int32))


DEVICES = [[0], [0, 1], [0, 0], [0, 0, 1, 1], [0, 1, 2, 3]]
SOURCES = {"grid": (pn.POINTS_GRID, {}), "lattice": (pn.POINTS_LATTICE, dict(reso=(9, 7, 8), block=3)),
           "band_apron0": (pn.POINTS_BAND, dict(reso=(5, 5, 17), block=2, apron=0)),
           "band_apron1": (pn.POINTS_BAND, dict(reso=(4, 4, 13), block=3, apron=1)),
           "list": (pn.POINTS_LIST, {})}


@pytest.mark.parametrize("source", sorted(SOURCES))
def test_sharded_equals_one_gpu_loop(source):
    kind, kw = SOURCES[source]
    src, count, points, plan, _keep = make_source(kind, **kw)
    assert 20 < count < 200, count
    channels = ((3, 1), (0, 3), (1, 3), (0, 4))
    for chunk, lists in ((7, DEVICES), (count, [[0], [0, 1, 2]])):  # ragged last chunk; one chunk, empty shards
        ref = one_gpu(points, count, chunk, 0, 4)
        assert torch.isfinite(ref).all()
        for k, devices in enumerate(lists):
            channel, nc = channels[k % len(channels)]
            rc, got = sharded(devices, src, count, chunk, channel, nc, plan)
            assert rc == 0, lib().pnr_last_error().decode()
            bits(got, ref[:, channel:channel + nc].contiguous())


def test_empty_shards_and_no_points():
    src, count, points, _, _keep = make_source(pn.POINTS_GRID, reso=(3, 3, 2))     # 18 points
    ref = one_gpu(points, count, 8, 0, 4)                                           # 3 chunks
    for devices in ([0, 0, 0, 0], [0, 1, 2, 3, 4, 5, 6]):
        rc, got = sharded(devices, src, count, 8, 0, 4)
        assert rc == 0
        bits(got, ref)
    for kind in (pn.POINTS_GRID, pn.POINTS_LATTICE, pn.POINTS_LIST):
        src, _, _, _, _keep = make_source(kind, count=0)
        rc, got = sharded([0, 1], src, 0, 5, 3, 1, fill=-7.0)
        assert rc == 0 and got.shape == (0, 1)
    rc, out = sharded([0, 1], make_source(pn.POINTS_GRID)[0], 0, 5, 3, 1)   # nothing written
    assert rc == 0


def test_shards_own_contiguous_runs_of_whole_chunks():
    """torch.chunk over the chunk indices: with 10 chunks on 4 shards, shard i owns chunks [3i, 3i + 3)."""
    src, count, points, _, _keep = make_source(pn.POINTS_GRID, reso=(4, 5, 2))     # 40 points
    ref = one_gpu(points, count, 4, 3, 1)
    # a shard without a usable workspace fails before anything is written, whichever shard it is
    L, sc = lib(), scene()
    need = L.pnr_mgpu_field_workspace_bytes(sc.scene, sc.mlp, 4, pn.ENGINE_SIMT)
    for bad in range(4):
        h = C.c_void_p()
        ok(L.pnr_mgpu_create((C.c_int32 * 4)(0, 1, 2, 3), 4, C.byref(h)))
        shards = (pn.PnrFieldShard * 4)()
        wss = [torch.zeros(need, dtype=torch.uint8) for _ in range(4)]
        for i, sh in enumerate(shards):
            sh.scene, sh.mlp = C.pointer(sc.scene), C.pointer(sc.mlp)
            sh.workspace, sh.workspace_bytes = wss[i].data_ptr(), need - (1 if i == bad else 0)
        out = torch.full((count, 1), -7.0)
        assert L.pnr_mgpu_field_eval(h, shards, C.byref(src), count, 4, pn.ENGINE_SIMT, 3, 1, eu.ptr(out),
                                     None) == PNR_ERR_WORKSPACE
        assert (out == -7.0).all()
        ok(L.pnr_mgpu_destroy(h))
    rc, got = sharded([0, 1, 2, 3], src, count, 4, 3, 1)
    assert rc == 0
    bits(got, ref)


def test_error_codes():
    L, sc = lib(), scene()
    grid, count, _, _, _ = make_source(pn.POINTS_GRID)
    for kind in (0, 5, -1):
        bad = pn.point_source(kind, LO, HI, (5, 4, 6))
        assert sharded([0, 1], bad, count, 7, 3, 1)[0] == PNR_ERR_INVALID
        assert b"kind" in L.pnr_last_error()
    for channel, nc in ((-1, 1), (0, 0), (3, 2), (4, 1), (0, 5), (1, -1)):
        assert sharded([0, 1], grid, count, 7, channel, nc)[0] == PNR_ERR_INVALID
        assert b"channel" in L.pnr_last_error()
    assert sharded([0, 1], grid, count + 1, 7, 3, 1)[0] == PNR_ERR_INVALID          # past the grid
    assert sharded([0, 1], grid, -1, 7, 3, 1)[0] == PNR_ERR_INVALID
    assert sharded([0, 1], grid, count, 0, 3, 1)[0] == PNR_ERR_INVALID              # chunk < 1
    assert sharded([0, 1], pn.point_source(pn.POINTS_GRID, LO, HI, (0, 4, 6)), 0, 7, 3, 1)[0] == PNR_ERR_INVALID
    lat, n_lat, _, _, _ = make_source(pn.POINTS_LATTICE, reso=(9, 7, 8), block=3)
    assert sharded([0, 1], lat, n_lat + 1, 7, 3, 1)[0] == PNR_ERR_INVALID
    assert sharded([0, 1], pn.point_source(pn.POINTS_LATTICE, LO, HI, (9, 7, 8), 1), 4, 7, 3, 1)[0] == PNR_ERR_INVALID
    band, M, _, plan, _ = make_source(pn.POINTS_BAND, reso=(5, 5, 17), block=2)
    assert sharded([0, 1], band, M, 7, 3, 1, plan)[0] == 0
    for n_points in (M - 1, M + 1):                      # n_points that disagrees with the count
        src = pn.point_source(pn.POINTS_BAND, LO, HI, (5, 5, 17), 2, 0, n_points)
        assert sharded([0, 1], src, M, 7, 3, 1, plan)[0] == PNR_ERR_INVALID
    assert sharded([0, 1], band, M, 7, 3, 1, None)[0] == PNR_ERR_INVALID            # no plan
    assert sharded([0, 1], band, M, 7, 3, 1, (plan[0], plan[1] - 1))[0] == PNR_ERR_WORKSPACE
    src = pn.point_source(pn.POINTS_BAND, LO, HI, (5, 5, 17), 2, 0, M)
    src.apron = 2
    assert sharded([0, 1], src, M, 7, 3, 1, plan)[0] == PNR_ERR_INVALID
    src = pn.point_source(pn.POINTS_BAND, LO, HI, (5, 5, 17), 300, 0, M)           # block 300
    assert sharded([0, 1], src, M, 7, 3, 1, plan)[0] == PNR_ERR_INVALID
    lst = pn.PnrPointSource()
    lst.kind = pn.POINTS_LIST
    assert sharded([0, 1], lst, 5, 7, 3, 1)[0] == PNR_ERR_INVALID                    # no rows
    need = L.pnr_mgpu_field_workspace_bytes(sc.scene, sc.mlp, 7, pn.ENGINE_SIMT)
    assert need > 0
    assert sharded([0, 1], grid, count, 7, 3, 1, ws_bytes=need - 1)[0] == PNR_ERR_WORKSPACE
    assert L.pnr_mgpu_field_workspace_bytes(sc.scene, sc.mlp, 0, pn.ENGINE_SIMT) == 0
    assert L.pnr_mgpu_field_workspace_bytes(None, sc.mlp, 7, pn.ENGINE_SIMT) == 0
    # a scene of two objects, an incomplete shard, NULL arguments
    h = C.c_void_p()
    ok(L.pnr_mgpu_create((C.c_int32 * 2)(0, 1), 2, C.byref(h)))
    shards = (pn.PnrFieldShard * 2)()
    out = torch.zeros(count)
    assert L.pnr_mgpu_field_eval(h, shards, C.byref(grid), count, 7, pn.ENGINE_SIMT, 3, 1, eu.ptr(out),
                                 None) == PNR_ERR_INVALID
    assert b"shard" in L.pnr_last_error()
    two = pn.PnrScene.from_buffer_copy(sc.scene)
    two.SB = 2
    ws = torch.zeros(need, dtype=torch.uint8)
    for sh in shards:
        sh.scene, sh.mlp = C.pointer(two), C.pointer(sc.mlp)
        sh.workspace, sh.workspace_bytes = ws.data_ptr(), need
    assert L.pnr_mgpu_field_eval(h, shards, C.byref(grid), count, 7, pn.ENGINE_SIMT, 3, 1, eu.ptr(out),
                                 None) == PNR_ERR_INVALID
    assert b"one object" in L.pnr_last_error()
    assert L.pnr_mgpu_field_eval(h, None, C.byref(grid), count, 7, pn.ENGINE_SIMT, 3, 1, eu.ptr(out),
                                 None) == PNR_ERR_INVALID
    assert L.pnr_mgpu_field_eval(None, shards, C.byref(grid), count, 7, pn.ENGINE_SIMT, 3, 1, eu.ptr(out),
                                 None) == PNR_ERR_INVALID
    ok(L.pnr_mgpu_destroy(h))


PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "pnr.h"
#define F(T, m) printf(#T "." #m " %zu\n", offsetof(T, m))
int main(void) {
  printf("PnrPointSource %zu\nPnrFieldShard %zu\n", sizeof(PnrPointSource), sizeof(PnrFieldShard));
  F(PnrPointSource, kind); F(PnrPointSource, lo); F(PnrPointSource, hi); F(PnrPointSource, reso);
  F(PnrPointSource, block); F(PnrPointSource, apron); F(PnrPointSource, n_points); F(PnrPointSource, xyz0);
  F(PnrPointSource, viewdirs0);
  F(PnrFieldShard, scene); F(PnrFieldShard, mlp); F(PnrFieldShard, plan); F(PnrFieldShard, plan_bytes);
  F(PnrFieldShard, workspace); F(PnrFieldShard, workspace_bytes); F(PnrFieldShard, stream);
  printf("%d %d %d %d\n", PNR_POINTS_GRID, PNR_POINTS_LATTICE, PNR_POINTS_BAND, PNR_POINTS_LIST);
  return 0;
}
"""


def test_struct_layouts_match_the_header(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text(PROBE)
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(eu.ROOT, "include"), "-o", str(exe), str(src)], check=True)
    lines = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines()
    got = dict(line.rsplit(" ", 1) for line in lines[:-1])
    assert int(got["PnrPointSource"]) == C.sizeof(pn.PnrPointSource)
    assert int(got["PnrFieldShard"]) == C.sizeof(pn.PnrFieldShard)
    for T in (pn.PnrPointSource, pn.PnrFieldShard):
        for name, _ in T._fields_:
            assert int(got[f"{T.__name__}.{name}"]) == getattr(T, name).offset, name
    assert [int(v) for v in lines[-1].split()] == [pn.POINTS_GRID, pn.POINTS_LATTICE, pn.POINTS_BAND, pn.POINTS_LIST]
