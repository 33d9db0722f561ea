"""Mesh-extraction kernels (csrc/pnr_recon.cu) on the host emulator (built by tests/recon_emu.py): pnr_grid_points
against the reference's grid and view directions (tests/golden/recon_ns*.npz), pnr_mc_count / pnr_mc_emit bit for bit
against the numpy oracle, and the error codes."""
import ctypes as C

import numpy as np
import pytest
import torch

import emu_util as eu
import golden_util as gu
import recon_emu
from recon_util import padded_random, recon, sphere, torus

PNR_ERR_INVALID, PNR_ERR_WORKSPACE = -1, -2


def ok(rc):
    assert rc == 0, recon_emu.lib().pnr_last_error().decode()


def grid_points(lo, hi, reso, first, count, dirs=True):
    xyz = torch.empty(count, 3)
    vd = torch.empty(count, 3) if dirs else None
    ok(recon_emu.lib().pnr_grid_points((C.c_double * 3)(*lo), (C.c_double * 3)(*hi), (C.c_int32 * 3)(*reso), first, count,
       eu.ptr(xyz), eu.ptr(vd), None))
    return xyz.numpy(), (vd.numpy() if dirs else None)


def mc(vol, iso):
    """pnr_mc_count + pnr_mc_emit on the emulator -> (verts, tris, counts)."""
    vol = torch.from_numpy(np.ascontiguousarray(vol, dtype=np.float32))
    L = recon_emu.lib()
    nx, ny, nz = vol.shape
    ws = torch.zeros(max(int(L.pnr_mc_workspace_bytes(nx, ny, nz)), 1), dtype=torch.uint8)
    counts = torch.full((2,), -7, dtype=torch.int64)
    ok(L.pnr_mc_count(eu.ptr(vol), nx, ny, nz, float(iso), C.c_void_p(counts.data_ptr()), C.c_void_p(ws.data_ptr()),
                      ws.numel(), None))
    nv, nt = counts.tolist()
    verts = torch.empty(nv, 3, dtype=torch.float64)
    tris = torch.empty(nt, 3, dtype=torch.int64)
    ok(L.pnr_mc_emit(eu.ptr(vol), nx, ny, nz, float(iso), C.c_void_p(verts.data_ptr()), C.c_void_p(tris.data_ptr()),
                     nv, nt, C.c_void_p(ws.data_ptr()), ws.numel(), None))
    return verts.numpy(), tris.numpy()


def assert_same_mesh(vol, iso):
    v, t = mc(vol, iso)
    rv, rt = recon.marching_cubes(vol, iso)
    assert v.shape == rv.shape and t.shape == rt.shape
    assert np.array_equal(v.view(np.int64), rv.view(np.int64))        # bit for bit
    assert np.array_equal(t, rt)
    return v, t


@pytest.mark.parametrize("ns", [1, 2])
@pytest.mark.parametrize("grid", ["box", "odd", "flat"])
def test_grid_points_bit_equal_to_reference(ns, grid):
    z = np.load(f"{gu.GOLD}/recon_ns{ns}.npz")
    lo, hi, reso = (z[f"{grid}/{k}"].tolist() for k in ("lo", "hi", "reso"))
    N = int(np.prod(reso))
    xyz, vd = grid_points(lo, hi, reso, 0, N)
    assert np.array_equal(xyz.view(np.int32), z[grid + "/points"].view(np.int32))
    ref = z[grid + "/dirs"]
    assert np.array_equal(np.isnan(vd), np.isnan(ref))
    assert np.array_equal(vd[~np.isnan(vd)].view(np.int32), ref[~np.isnan(ref)].view(np.int32))
    if grid == "odd":
        assert np.isnan(vd[np.all(xyz == 0, axis=1)]).all()
    # chunks as util.recon evaluates them, without the directions
    for first, count in ((0, 37), (37, 100), (N - 5, 5)):
        part, none = grid_points(lo, hi, reso, first, count, dirs=False)
        assert none is None and np.array_equal(part.view(np.int32), z[grid + "/points"][first:first + count].view(np.int32))


def test_grid_points_match_numpy_linspace_on_awkward_bounds():
    lo, hi, reso = (-1.3, 0.1, 2.0), (0.7, 0.1000001, -3.5), (13, 3, 1)
    xyz, _ = grid_points(lo, hi, reso, 0, 13 * 3)
    assert np.array_equal(xyz.view(np.int32), recon.grid_points(lo, hi, reso).view(np.int32))


def test_sphere_and_torus_non_cubic():
    v, t = assert_same_mesh(sphere((21, 17, 19), 6.4), 0.0)
    assert recon.is_closed_oriented(t) and recon.euler_characteristic(v, t) == 2
    v, t = assert_same_mesh(torus((26, 24, 12), 7.0, 2.6), 0.25)
    assert recon.is_closed_oriented(t) and recon.euler_characteristic(v, t) == 0


@pytest.mark.parametrize("seed", range(4))
def test_random_fields(seed):
    g = np.random.default_rng(100 + seed)
    shape = tuple(int(n) for n in g.integers(2, 14, size=3))
    assert_same_mesh(g.standard_normal(shape).astype(np.float32), float(g.uniform(-0.3, 0.3)))
    assert_same_mesh(padded_random((7, 6, 8), seed), 0.0)


def test_non_finite_corners_and_values_equal_to_iso():
    g = np.random.default_rng(7)
    vol = g.standard_normal((9, 10, 11)).astype(np.float32)
    flat = vol.reshape(-1)
    idx = g.permutation(flat.size)
    flat[idx[:20]] = np.nan
    flat[idx[20:30]] = np.inf
    flat[idx[30:40]] = -np.inf
    flat[idx[40:80]] = np.float32(0.25)       # exactly iso: outside
    v, t = assert_same_mesh(vol, 0.25)
    assert np.isfinite(v).all()


def test_a_dimension_of_one_gives_no_cells():
    for shape in ((1, 6, 7), (5, 1, 4), (3, 4, 1)):
        v, t = mc(np.random.default_rng(0).standard_normal(shape).astype(np.float32), 0.0)
        assert v.shape == (0, 3) and t.shape == (0, 3)


def test_sizes_across_scan_tiles():
    # 4096-element scan tiles: 3N edge slots over several tiles, then N cells over several, then more than 256 tiles
    for shape in ((13, 11, 12), (17, 16, 18)):
        assert_same_mesh(sphere(shape, min(shape) * 0.4) + 0.3 * np.sin(np.arange(np.prod(shape))).reshape(shape)
                         .astype(np.float32), 0.0)
    assert_same_mesh(padded_random((72, 70, 70), 3), 0.0)


def test_error_codes():
    L = recon_emu.lib()
    vol = torch.zeros(4, 4, 4)
    counts = torch.zeros(2, dtype=torch.int64)
    cp = C.c_void_p(counts.data_ptr())
    need = int(L.pnr_mc_workspace_bytes(4, 4, 4))
    ws = torch.zeros(need, dtype=torch.uint8)
    wp = C.c_void_p(ws.data_ptr())
    assert L.pnr_mc_workspace_bytes(0, 4, 4) == 0 and L.pnr_mc_workspace_bytes(1, 4, 4) == 0
    assert L.pnr_mc_count(eu.ptr(vol), 0, 4, 4, 0.0, cp, wp, need, None) == PNR_ERR_INVALID
    assert L.pnr_mc_count(eu.ptr(vol), 4, -1, 4, 0.0, cp, wp, need, None) == PNR_ERR_INVALID
    assert L.pnr_mc_count(eu.ptr(vol), 4096, 4096, 8192, 0.0, cp, wp, need, None) == PNR_ERR_INVALID   # > 2^36 points
    assert L.pnr_mc_count(eu.ptr(vol), 4, 4, 4, 0.0, None, wp, need, None) == PNR_ERR_INVALID
    assert L.pnr_mc_count(None, 4, 4, 4, 0.0, cp, wp, need, None) == PNR_ERR_INVALID
    assert L.pnr_mc_count(eu.ptr(vol), 4, 4, 4, 0.0, cp, wp, need - 1, None) == PNR_ERR_WORKSPACE
    assert L.pnr_mc_count(eu.ptr(vol), 4, 4, 4, 0.0, cp, None, 0, None) == PNR_ERR_WORKSPACE
    assert L.pnr_mc_emit(eu.ptr(vol), 4, 4, 4, 0.0, None, None, -1, 0, wp, need, None) == PNR_ERR_INVALID
    assert L.pnr_mc_emit(eu.ptr(vol), 4, 4, 4, 0.0, None, None, 3, 0, wp, need, None) == PNR_ERR_INVALID
    assert L.pnr_mc_emit(eu.ptr(vol), 4, 4, 4, 0.0, None, None, 0, 0, wp, need - 1, None) == PNR_ERR_WORKSPACE
    counts.fill_(5)
    assert L.pnr_mc_count(None, 1, 4, 4, 0.0, cp, None, 0, None) == 0 and counts.tolist() == [0, 0]
    xyz = torch.empty(4, 3)
    lo, hi = (C.c_double * 3)(0, 0, 0), (C.c_double * 3)(1, 1, 1)
    assert L.pnr_grid_points(lo, hi, (C.c_int32 * 3)(2, 0, 2), 0, 0, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    assert L.pnr_grid_points(lo, hi, (C.c_int32 * 3)(2, 2, 2), 5, 4, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    assert L.pnr_grid_points(lo, hi, (C.c_int32 * 3)(2, 2, 2), 0, 4, None, None, None) == PNR_ERR_INVALID
    assert L.pnr_grid_points(None, hi, (C.c_int32 * 3)(2, 2, 2), 0, 4, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
