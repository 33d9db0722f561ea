"""Narrow-band mesh extraction (the pnr_band_* entry points of csrc/pnr_recon.cu) on the host emulator (built by
tests/recon_emu.py): lattice and refinement points, plan counts, mesh and vertex attributes bit for bit against the
numpy oracle (oracle/pnr_recon_band.py), repeatability, workspace sizes and the error codes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import emu_util as eu
import golden_util as gu
import recon_emu
from golden_util import ROOT, load_by_path
from recon_util import padded_random, recon, single_cell, sphere, torus, two_spheres

band = load_by_path("pnr_recon_band_oracle", os.path.join(ROOT, "oracle", "pnr_recon_band.py"))

PNR_ERR_INVALID, PNR_ERR_WORKSPACE = -1, -2
BOX = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))


def ok(rc):
    assert rc == 0, recon_emu.lib().pnr_last_error().decode()


def r3(reso):
    return (C.c_int32 * 3)(*reso)


def b3(lo, hi):
    return (C.c_double * 3)(*map(float, lo)), (C.c_double * 3)(*map(float, hi))


def bits(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def run_band(vol, iso, b, lo=BOX[0], hi=BOX[1], apron=True):
    """Every pnr_band_* entry point on the emulator against the oracle; -> (verts, tris, normals, xyz, viewdirs,
    plan counts)."""
    L = recon_emu.lib()
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    reso = vol.shape
    flat = vol.reshape(-1)
    # the coarse lattice: pnr_grid_points' bits at the lattice's grid indices
    lat = band.lattice_flat(reso, b)
    xyz, vd = torch.empty(len(lat), 3), torch.empty(len(lat), 3)
    ok(L.pnr_band_lattice_points(*b3(lo, hi), r3(reso), b, 0, len(lat), eu.ptr(xyz), eu.ptr(vd), None))
    rxyz, rvd = band.lattice_points(lo, hi, reso, b)
    bits(xyz.numpy(), rxyz)
    bits(vd.numpy(), rvd)
    # the plan
    nbytes = int(L.pnr_band_plan_bytes(r3(reso), b, int(apron)))
    plan = torch.zeros(nbytes, dtype=torch.uint8)
    pp = C.c_void_p(plan.data_ptr())
    counts = torch.full((2,), -7, dtype=torch.int64)
    coarse = torch.from_numpy(np.ascontiguousarray(flat[lat]))
    ok(L.pnr_band_plan(eu.ptr(coarse), r3(reso), b, float(iso), int(apron), C.c_void_p(counts.data_ptr()), pp,
                       nbytes, None))
    _, active = band.plan(flat[lat], reso, b, iso)
    idx = band.refine_index(active, reso, b, apron)
    n_active, M = counts.tolist()
    assert (n_active, M) == (int(active.sum()), len(idx))
    # the refinement points, whole and in chunks
    xyz, vd = torch.empty(M, 3), torch.empty(M, 3)
    ok(L.pnr_band_points(*b3(lo, hi), r3(reso), b, int(apron), pp, nbytes, M, 0, M, eu.ptr(xyz), eu.ptr(vd), None))
    gxyz = recon.grid_points(lo, hi, reso)[idx]
    bits(xyz.numpy(), gxyz)
    bits(vd.numpy(), recon.fake_viewdirs(gxyz))
    if M > 7:
        part = torch.empty(5, 3)
        ok(L.pnr_band_points(*b3(lo, hi), r3(reso), b, int(apron), pp, nbytes, M, M - 7, 5, eu.ptr(part), None, None))
        bits(part.numpy(), gxyz[M - 7:M - 2])
    # marching cubes over the refinement sigma
    sigma = torch.from_numpy(np.ascontiguousarray(flat[idx]))
    ws = torch.zeros(max(int(L.pnr_band_mc_workspace_bytes(M)), 1), dtype=torch.uint8)
    wp = C.c_void_p(ws.data_ptr())
    head = (eu.ptr(sigma), M, r3(reso), b, int(apron), float(iso), pp, nbytes)
    mc = torch.full((2,), -7, dtype=torch.int64)
    ok(L.pnr_band_mc_count(*head, C.c_void_p(mc.data_ptr()), wp, ws.numel(), None))
    nv, nt = mc.tolist()
    verts = torch.empty(nv, 3, dtype=torch.float64)
    tris = torch.empty(nt, 3, dtype=torch.int64)
    ok(L.pnr_band_mc_emit(*head, C.c_void_p(verts.data_ptr()), C.c_void_p(tris.data_ptr()), nv, nt, wp, ws.numel(),
                          None))
    rv, rt, _ = band.marching_cubes(vol, iso, b)
    bits(verts.numpy(), rv)
    bits(tris.numpy(), rt)
    out = [verts.numpy(), tris.numpy()]
    if apron:
        normals = torch.full((nv, 3), 7.0, dtype=torch.float64)
        axyz, avd = torch.full((nv, 3), 7.0), torch.full((nv, 3), 7.0)
        ok(L.pnr_band_mc_vertex_attrs(eu.ptr(sigma), M, r3(reso), b, 1, float(iso), *b3(lo, hi), pp, nbytes,
                                      C.c_void_p(normals.data_ptr()), eu.ptr(axyz), eu.ptr(avd), nv, wp, ws.numel(),
                                      None))
        rn, rxyz, rvd = band.vertex_attrs(vol, iso, lo, hi, b)
        bits(normals.numpy(), rn)
        bits(axyz.numpy(), rxyz)
        bits(avd.numpy(), rvd)
        out += [normals.numpy(), axyz.numpy(), avd.numpy()]
    return out + [(n_active, M)]


def assert_complete(vol, iso, b, closed=None, euler=None):
    """complete coverage: the band's mesh is the dense one; -> whether coverage was complete"""
    v, t, complete = band.marching_cubes(vol, iso, b)
    if not complete:
        return False
    rv, rt = recon.marching_cubes(vol, iso)
    bits(v, rv)
    bits(t, rt)
    if closed is not None:
        assert recon.is_closed_oriented(t) == closed
    if euler is not None:
        assert recon.euler_characteristic(v, t) == euler
    return True


SHAPES = {
    "sphere": (lambda: sphere((21, 17, 19), 6.4), 0.0, 2),
    "torus": (lambda: torus((26, 24, 12), 7.0, 2.6), 0.25, 0),
    "two_spheres": (lambda: two_spheres((24, 14, 15), 4.1, 5.3), 0.0, 4),
    "padded_random": (lambda: padded_random((9, 8, 10), 1), 0.0, None),
}


@pytest.mark.parametrize("b", [2, 3, 4, 8])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_shapes(shape, b):
    make, iso, euler = SHAPES[shape]
    vol = make()
    for apron in (False, True):
        run_band(vol, iso, b, apron=apron)
    if band.marching_cubes(vol, iso, b)[2]:
        assert assert_complete(vol, iso, b, closed=True, euler=euler)      # every shape here is a closed surface


@pytest.mark.parametrize("b", [2, 3, 4, 8])
def test_resolutions_multiple_of_b_or_not_and_smaller_than_b(b):
    for shape in ((2 * b + 1, 3 * b + 1, b + 1), (2 * b, 3 * b, b), (2 * b + 2, b + 3, 3 * b - 1), (b - 1 if b > 2 else
                  2, 2, 3), (2, b + 1, 5)):
        vol = sphere(shape, min(shape) * 0.45) + np.float32(0.2) * np.sin(np.arange(np.prod(shape))).reshape(
            shape).astype(np.float32)
        run_band(vol, 0.0, b)


@pytest.mark.parametrize("b", [2, 3])
def test_single_cell_configurations(b):
    for cfg in range(0, 256, 7):
        run_band(single_cell(cfg), 0.0, b)


def test_empty_full_and_flat_volumes():
    for vol in (-np.ones((9, 7, 8), np.float32), np.ones((9, 7, 8), np.float32)):
        v, t, n, _, _, (n_active, M) = run_band(vol, 0.0, 3)
        assert len(v) == len(t) == len(n) == 0 and n_active == 0 and M == 0
    v, t, _, _, _, counts = run_band(np.random.default_rng(0).standard_normal((1, 6, 7)).astype(np.float32), 0.0, 2)
    assert len(v) == len(t) == 0 and counts == (0, 0)


def test_non_finite_corners():
    g = np.random.default_rng(7)
    vol = sphere((13, 14, 12), 4.7) + np.float32(0.5) * g.standard_normal((13, 14, 12)).astype(np.float32)
    flat = vol.reshape(-1)
    lat = band.lattice_flat(vol.shape, 3)
    flat[lat[::5]] = np.nan                             # lattice corners too
    flat[lat[1::7]] = np.inf
    flat[lat[2::9]] = -np.inf
    idx = g.permutation(flat.size)
    flat[idx[:20]] = np.nan
    flat[idx[20:30]] = np.inf
    flat[idx[30:40]] = -np.inf
    flat[idx[40:60]] = np.float32(0.25)                 # exactly iso: outside
    for b in (2, 3, 4):
        n = run_band(vol, 0.25, b)[2]
        assert np.isfinite(n).all()
    odd = sphere((21, 21, 21), 5.3)
    odd[10, 10, 10] = np.nan                            # the grid origin of an odd grid over a centred box
    run_band(odd, 0.0, 4)


def test_a_blob_no_lattice_point_sees_is_missed():
    vol = -np.ones((17, 17, 17), np.float32)
    vol[5:7, 5:7, 5:7] = 1.0                            # inside cells of block 1 (b = 4) / block 0 (b = 8) only
    vol[14, 14, 14] = 1.0                               # a second one, in the last block of either
    for b in (4, 8):                                    # lattice indices 0, 4, 8, 12, 16 / 0, 8, 16: none inside
        v, t, complete = band.marching_cubes(vol, 0.0, b)
        assert not complete and len(t) == 0
        run_band(vol, 0.0, b)
    assert len(recon.marching_cubes(vol, 0.0)[1]) > 0
    # a surface the lattice sees seeds block 0: the band keeps the first blob (block 1 is active) but not the second
    vol[0:2, 0:2, 0:2] = 1.0
    v, t, complete = band.marching_cubes(vol, 0.0, 4)
    rv, rt = recon.marching_cubes(vol, 0.0)
    assert not complete and 0 < len(t) < len(rt)
    assert (v < 8).all() and (rv > 13).any()
    run_band(vol, 0.0, 4)


def test_sizes_across_scan_tiles():
    vol = sphere((40, 37, 45), 15.5) + np.float32(0.4) * np.sin(np.arange(40 * 37 * 45)).reshape(40, 37, 45).astype(
        np.float32)
    for b in (4, 8):
        run_band(vol, 0.0, b)
    run_band(padded_random((36, 34, 35), 2), 0.0, 4)


@pytest.mark.parametrize("ns", [1, 2])
def test_golden_grids(ns):
    z = np.load(f"{gu.GOLD}/recon_ns{ns}.npz")
    for grid in ("box", "odd", "flat"):
        lo, hi, reso = (z[f"{grid}/{k}"].tolist() for k in ("lo", "hi", "reso"))
        vol = z[f"{grid}/coarse"][:, 3].reshape(reso).astype(np.float32)
        if min(reso) < 2:
            continue
        iso = float(np.median(vol[np.isfinite(vol)]))
        for b in (2, 3, 4, 8):
            run_band(vol, iso, b, lo, hi)


def test_repeatable():
    vol = torus((30, 28, 16), 8.0, 3.1)
    first = run_band(vol, 0.1, 3)
    again = run_band(vol, 0.1, 3)
    for a, b in zip(first[:-1], again[:-1]):
        bits(a, b)


def test_workspace_grows_with_the_band_not_the_grid():
    L = recon_emu.lib()
    # the plan is sized by the block grid (blocks, and 2 or 3 runs of points per block and axis)
    big = r3((1024, 1024, 1024))
    assert L.pnr_band_plan_bytes(big, 16, 1) < L.pnr_band_plan_bytes(big, 4, 1) < L.pnr_band_plan_bytes(big, 2, 1)
    # 2 flag bytes per block, 4 bytes per run box: 2 runs per block and axis (3 with the apron)
    assert L.pnr_band_plan_bytes(big, 8, 0) < (2 + 4 * 8 + 1) * 128 ** 3
    assert L.pnr_band_plan_bytes(big, 8, 1) < (2 + 4 * 27 + 1) * 128 ** 3
    # the marching-cubes workspace by the refinement points: 37 bytes each, as the dense one per grid point
    assert L.pnr_band_mc_workspace_bytes(10 ** 6) < L.pnr_band_mc_workspace_bytes(10 ** 7)
    assert 37 * 10 ** 6 <= L.pnr_band_mc_workspace_bytes(10 ** 6) <= 37.1 * 10 ** 6       # plus the scan tile sums
    # a thin shell: the refinement set is a small part of the grid and grows with the shell, not with the grid
    small = run_band(sphere((49, 49, 49), 6.2), 0.0, 4, apron=False)[-1]
    big = run_band(sphere((97, 97, 97), 6.2), 0.0, 4, apron=False)[-1]      # the same sphere on the same lattice
    assert big == small
    assert small[1] < 49 ** 3 // 4


def make_plan(vol, b, apron):
    """a plan of vol's lattice on the emulator -> (plan tensor, its bytes, refinement points)"""
    L = recon_emu.lib()
    reso = vol.shape
    nbytes = int(L.pnr_band_plan_bytes(r3(reso), b, apron))
    plan = torch.zeros(nbytes, dtype=torch.uint8)
    counts = torch.zeros(2, dtype=torch.int64)
    coarse = torch.from_numpy(np.ascontiguousarray(vol.reshape(-1)[band.lattice_flat(reso, b)]))
    ok(L.pnr_band_plan(eu.ptr(coarse), r3(reso), b, 0.0, apron, C.c_void_p(counts.data_ptr()),
                       C.c_void_p(plan.data_ptr()), nbytes, None))
    return plan, nbytes, int(counts[1])


def test_error_codes():
    L = recon_emu.lib()
    reso = r3((6, 6, 6))
    lo, hi = b3(*BOX)
    nbytes = int(L.pnr_band_plan_bytes(reso, 2, 0))
    plan = torch.zeros(nbytes, dtype=torch.uint8)
    pp = C.c_void_p(plan.data_ptr())
    coarse = torch.full((64,), -1.0)
    counts = torch.zeros(2, dtype=torch.int64)
    cp = C.c_void_p(counts.data_ptr())
    xyz = torch.empty(300, 3)
    assert L.pnr_band_plan_bytes(reso, 1, 0) == 0 and L.pnr_band_plan_bytes(reso, 257, 0) == 0
    assert L.pnr_band_plan_bytes(reso, 2, 2) == 0
    assert L.pnr_band_plan_bytes(r3((0, 6, 6)), 2, 0) == 0 and L.pnr_band_plan_bytes(r3((4096, 4096, 8192)), 8, 0) == 0
    assert L.pnr_band_plan_bytes(None, 2, 0) == 0

    def plan_call(b=2, dims=(6, 6, 6), apron=0, nb=nbytes, p=pp, c=cp, src=eu.ptr(coarse)):
        return L.pnr_band_plan(src, r3(dims), b, 0.0, apron, c, p, nb, None)
    assert plan_call() == 0
    for b in (1, 0, -3, 257):
        assert plan_call(b=b) == PNR_ERR_INVALID
    assert plan_call(dims=(0, 6, 6)) == PNR_ERR_INVALID
    assert plan_call(dims=(6, -1, 6)) == PNR_ERR_INVALID
    assert plan_call(dims=(4096, 4096, 8192)) == PNR_ERR_INVALID              # > 2^36 points
    assert plan_call(apron=2) == PNR_ERR_INVALID
    assert plan_call(c=None) == PNR_ERR_INVALID
    assert plan_call(src=None) == PNR_ERR_INVALID
    assert plan_call(nb=nbytes - 1) == PNR_ERR_WORKSPACE
    assert plan_call(p=None, nb=0) == PNR_ERR_WORKSPACE
    assert L.pnr_band_plan(eu.ptr(coarse), None, 2, 0.0, 0, cp, pp, nbytes, None) == PNR_ERR_INVALID
    # lattice and refinement points
    assert L.pnr_band_lattice_points(lo, hi, reso, 2, 0, 64, eu.ptr(xyz), None, None) == 0
    assert L.pnr_band_lattice_points(lo, hi, reso, 2, 1, 64, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    assert L.pnr_band_lattice_points(lo, hi, reso, 2, -1, 4, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    assert L.pnr_band_lattice_points(lo, hi, reso, 2, 0, 4, None, None, None) == PNR_ERR_INVALID
    assert L.pnr_band_lattice_points(None, hi, reso, 2, 0, 4, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    assert L.pnr_band_lattice_points(lo, hi, reso, 1, 0, 4, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    assert L.pnr_band_points(lo, hi, reso, 2, 0, pp, nbytes, 10, 5, 6, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    assert L.pnr_band_points(lo, hi, reso, 2, 0, pp, nbytes - 1, 10, 0, 4, eu.ptr(xyz), None,
                             None) == PNR_ERR_WORKSPACE
    assert L.pnr_band_points(lo, hi, reso, 2, 0, pp, nbytes, 10, 0, 4, None, None, None) == PNR_ERR_INVALID
    assert L.pnr_band_points(lo, hi, reso, 2, 3, pp, nbytes, 10, 0, 4, eu.ptr(xyz), None, None) == PNR_ERR_INVALID
    # marching cubes: the plan's header must match the call
    vol = sphere((17, 16, 18), 2.6)
    plan0, nb0, M0 = make_plan(vol, 2, 0)
    plan1, nb1, M1 = make_plan(vol, 2, 1)
    assert 0 < M0 < M1
    sigma = torch.zeros(M1)
    ws_need = int(L.pnr_band_mc_workspace_bytes(M1))
    ws = torch.zeros(ws_need, dtype=torch.uint8)
    wp = C.c_void_p(ws.data_ptr())
    assert L.pnr_band_mc_workspace_bytes(-1) == 0
    dims = r3(vol.shape)

    def count(M=M0, b=2, apron=0, plan=plan0, nb=nb0, w=wp, wn=ws_need, s=eu.ptr(sigma), c=cp, d=dims):
        return L.pnr_band_mc_count(s, M, d, b, apron, 0.0, C.c_void_p(plan.data_ptr()), nb, c, w, wn, None)
    assert count() == 0
    assert count(apron=1, plan=plan1, nb=nb1, M=M1) == 0
    assert count(M=M0 + 1) == PNR_ERR_INVALID                                  # not the plan's point count
    assert count(M=M0 - 1) == PNR_ERR_INVALID
    assert count(M=0) == PNR_ERR_INVALID
    assert count(M=-1) == PNR_ERR_INVALID
    assert count(d=r3((17, 16, 19))) == PNR_ERR_INVALID                           # plan made for another grid
    assert count(plan=torch.zeros(nb0, dtype=torch.uint8)) == PNR_ERR_INVALID  # not a plan
    assert count(b=1) == PNR_ERR_INVALID
    assert count(c=None) == PNR_ERR_INVALID
    assert count(s=None) == PNR_ERR_INVALID
    assert count(nb=nb0 - 1) == PNR_ERR_WORKSPACE
    assert count(wn=int(L.pnr_band_mc_workspace_bytes(M0)) - 1) == PNR_ERR_WORKSPACE
    assert count(w=None, wn=0) == PNR_ERR_WORKSPACE
    head0 = (eu.ptr(sigma), M0, dims, 2, 0, 0.0, C.c_void_p(plan0.data_ptr()), nb0)
    head1 = (eu.ptr(sigma), M1, dims, 2, 1, 0.0)
    pp1 = (C.c_void_p(plan1.data_ptr()), nb1)
    assert L.pnr_band_mc_emit(*head0, None, None, -1, 0, wp, ws_need, None) == PNR_ERR_INVALID
    assert L.pnr_band_mc_emit(*head0, None, None, 3, 0, wp, ws_need, None) == PNR_ERR_INVALID
    assert L.pnr_band_mc_emit(*head0, None, None, 0, 0, wp, 10, None) == PNR_ERR_WORKSPACE
    assert L.pnr_band_mc_emit(*head0[:1], M0 + 2, *head0[2:], None, None, 0, 0, wp, ws_need, None) == PNR_ERR_INVALID
    assert L.pnr_band_mc_vertex_attrs(*head1, lo, hi, *pp1, None, None, None, 0, wp, ws_need, None) == 0
    assert L.pnr_band_mc_vertex_attrs(*head1, None, hi, *pp1, None, None, None, 0, wp, ws_need,
                                      None) == PNR_ERR_INVALID
    assert L.pnr_band_mc_vertex_attrs(*head1, lo, hi, *pp1, None, None, None, -1, wp, ws_need,
                                      None) == PNR_ERR_INVALID
    assert L.pnr_band_mc_vertex_attrs(*head1, lo, hi, *pp1, None, None, None, 0, wp, 10, None) == PNR_ERR_WORKSPACE
    # vertex attributes read the apron: a plan without one is refused, whatever apron the call claims
    assert L.pnr_band_mc_vertex_attrs(*head0[:4], 0, 0.0, lo, hi, *head0[6:], None, None, None, 0, wp, ws_need,
                                      None) == PNR_ERR_INVALID
    assert L.pnr_band_mc_vertex_attrs(*head0[:4], 1, 0.0, lo, hi, *head0[6:], None, None, None, 0, wp, ws_need,
                                      None) == PNR_ERR_INVALID
