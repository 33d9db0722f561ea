"""pnr_mc_vertex_attrs (csrc/pnr_recon.cu) on the host emulator (built by tests/recon_emu.py): normals, query points
and view directions bit for bit against the numpy oracle (oracle/pnr_recon_attrs.py vertex_attrs), and the error
codes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import emu_util as eu
import recon_emu
from golden_util import ROOT, load_by_path
from recon_util import padded_random, recon, sphere, torus

attrs = load_by_path("pnr_recon_attrs_oracle", os.path.join(ROOT, "oracle", "pnr_recon_attrs.py"))

PNR_ERR_INVALID, PNR_ERR_WORKSPACE = -1, -2


def ok(rc):
    assert rc == 0, recon_emu.lib().pnr_last_error().decode()


def bounds(lo, hi):
    return (C.c_double * 3)(*map(float, lo)), (C.c_double * 3)(*map(float, hi))


def mc_attrs(vol, iso, lo, hi):
    """pnr_mc_count + pnr_mc_emit + pnr_mc_vertex_attrs on the emulator -> (verts, normals, xyz, viewdirs)."""
    vol = torch.from_numpy(np.ascontiguousarray(vol, dtype=np.float32))
    L = recon_emu.lib()
    nx, ny, nz = vol.shape
    ws = torch.zeros(max(int(L.pnr_mc_workspace_bytes(nx, ny, nz)), 1), dtype=torch.uint8)
    wp = C.c_void_p(ws.data_ptr())
    counts = torch.full((2,), -7, dtype=torch.int64)
    ok(L.pnr_mc_count(eu.ptr(vol), nx, ny, nz, float(iso), C.c_void_p(counts.data_ptr()), wp, ws.numel(), None))
    nv, nt = counts.tolist()
    verts = torch.empty(nv, 3, dtype=torch.float64)
    tris = torch.empty(nt, 3, dtype=torch.int64)
    ok(L.pnr_mc_emit(eu.ptr(vol), nx, ny, nz, float(iso), C.c_void_p(verts.data_ptr()), C.c_void_p(tris.data_ptr()),
                     nv, nt, wp, ws.numel(), None))
    normals = torch.full((nv, 3), 7.0, dtype=torch.float64)
    xyz, vd = torch.full((nv, 3), 7.0), torch.full((nv, 3), 7.0)
    ok(L.pnr_mc_vertex_attrs(eu.ptr(vol), nx, ny, nz, float(iso), *bounds(lo, hi), C.c_void_p(normals.data_ptr()),
                             eu.ptr(xyz), eu.ptr(vd), nv, wp, ws.numel(), None))
    return verts.numpy(), normals.numpy(), xyz.numpy(), vd.numpy()


def assert_same_attrs(vol, iso, lo, hi):
    v, n, xyz, vd = mc_attrs(vol, iso, lo, hi)
    rv, _ = recon.marching_cubes(vol, iso)
    rn, rxyz, rvd = attrs.vertex_attrs(vol, iso, lo, hi)
    assert np.array_equal(v.view(np.int64), rv.view(np.int64))
    assert n.shape == rn.shape
    assert np.array_equal(n.view(np.int64), rn.view(np.int64))             # bit for bit
    assert np.array_equal(xyz.view(np.int32), rxyz.view(np.int32))
    assert np.array_equal(vd.view(np.int32), rvd.view(np.int32))
    return n


BOX = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))


def test_sphere_and_torus():
    n = assert_same_attrs(sphere((40, 36, 44), 12.3), 0.0, (-0.55, -0.6, -0.5), (0.6, 0.5, 0.55))
    assert len(n) > 2000
    assert_same_attrs(torus((26, 24, 12), 7.0, 2.6), 0.25, *BOX)


@pytest.mark.parametrize("seed", range(4))
def test_random_fields(seed):
    g = np.random.default_rng(200 + seed)
    shape = tuple(int(n) for n in g.integers(2, 14, size=3))
    assert_same_attrs(g.standard_normal(shape).astype(np.float32), float(g.uniform(-0.3, 0.3)), *BOX)
    assert_same_attrs(padded_random((7, 6, 8), seed), 0.0, *BOX)      # +-1 values: many flat edges (fallback)


def test_non_finite_fields():
    g = np.random.default_rng(9)
    vol = g.standard_normal((9, 10, 11)).astype(np.float32)
    flat = vol.reshape(-1)
    idx = g.permutation(flat.size)
    flat[idx[:20]] = np.nan
    flat[idx[20:30]] = np.inf
    flat[idx[30:40]] = -np.inf
    flat[idx[40:80]] = np.float32(0.25)       # exactly iso: outside
    n = assert_same_attrs(vol, 0.25, *BOX)
    assert np.isfinite(n).all()
    odd = sphere((21, 21, 21), 5.3)
    odd[10, 10, 10] = np.nan                  # the grid origin of an odd grid over a centred box
    assert np.isfinite(assert_same_attrs(odd, 0.0, *BOX)).all()


def test_awkward_bounds():
    vol = sphere((13, 9, 11), 3.7) + np.float32(0.3) * np.sin(np.arange(13 * 9 * 11)).reshape(13, 9, 11).astype(
        np.float32)
    for lo, hi in (((-1.3, 0.1, 2.0), (0.7, 0.1000001, -3.5)),      # a thin axis and a reversed one
                   ((0.0, 0.0, 0.0), (0.0, 1.0, 1.0)),              # a flat axis: h = 0
                   ((-1e-3, 5.0, -7.25), (2e-3, 5.5, 1e4))):
        n = assert_same_attrs(vol, 0.1, lo, hi)
        assert np.isfinite(n).all()


def test_sizes_across_scan_tiles():
    for shape in ((13, 11, 12), (17, 16, 18)):
        assert_same_attrs(sphere(shape, min(shape) * 0.4) + 0.3 * np.sin(np.arange(np.prod(shape))).reshape(shape)
                          .astype(np.float32), 0.0, *BOX)
    assert_same_attrs(padded_random((72, 70, 70), 3), 0.0, *BOX)


def test_outputs_may_be_null_and_a_dimension_of_one_writes_nothing():
    vol = torch.from_numpy(sphere((9, 8, 7), 3.1))
    L = recon_emu.lib()
    ws = torch.zeros(int(L.pnr_mc_workspace_bytes(9, 8, 7)), dtype=torch.uint8)
    wp = C.c_void_p(ws.data_ptr())
    counts = torch.zeros(2, dtype=torch.int64)
    ok(L.pnr_mc_count(eu.ptr(vol), 9, 8, 7, 0.0, C.c_void_p(counts.data_ptr()), wp, ws.numel(), None))
    nv = int(counts[0])
    _, rn, rxyz, rvd = mc_attrs(vol.numpy(), 0.0, *BOX)
    xyz = torch.full((nv, 3), 7.0)
    ok(L.pnr_mc_vertex_attrs(eu.ptr(vol), 9, 8, 7, 0.0, *bounds(*BOX), None, eu.ptr(xyz), None, nv, wp, ws.numel(),
                             None))
    assert np.array_equal(xyz.numpy().view(np.int32), rxyz.view(np.int32))
    ok(L.pnr_mc_vertex_attrs(eu.ptr(vol), 9, 8, 7, 0.0, *bounds(*BOX), None, None, None, nv, wp, ws.numel(), None))
    flat = torch.full((4, 3), 7.0)
    ok(L.pnr_mc_vertex_attrs(None, 1, 8, 7, 0.0, *bounds(*BOX), None, eu.ptr(flat), None, 4, None, 0, None))
    assert (flat == 7.0).all()


def test_error_codes():
    L = recon_emu.lib()
    vol = torch.zeros(4, 4, 4)
    need = int(L.pnr_mc_workspace_bytes(4, 4, 4))
    ws = torch.zeros(need, dtype=torch.uint8)
    wp = C.c_void_p(ws.data_ptr())
    lo, hi = bounds(*BOX)
    xyz = torch.empty(3, 3)

    def call(v=eu.ptr(vol), dims=(4, 4, 4), lo=lo, hi=hi, n_verts=0, wp=wp, nbytes=need):
        return L.pnr_mc_vertex_attrs(v, *dims, 0.0, lo, hi, None, eu.ptr(xyz), None, n_verts, wp, nbytes, None)
    assert call() == 0
    assert call(dims=(0, 4, 4)) == PNR_ERR_INVALID
    assert call(dims=(4, -1, 4)) == PNR_ERR_INVALID
    assert call(dims=(4096, 4096, 8192)) == PNR_ERR_INVALID                 # > 2^36 points
    assert call(v=None) == PNR_ERR_INVALID
    assert call(lo=None) == PNR_ERR_INVALID
    assert call(hi=None) == PNR_ERR_INVALID
    assert call(n_verts=-1) == PNR_ERR_INVALID
    assert call(nbytes=need - 1) == PNR_ERR_WORKSPACE
    assert call(wp=None, nbytes=0) == PNR_ERR_WORKSPACE
