"""The narrow-band mesh oracle (oracle/pnr_recon_band.py), numpy only: complete coverage gives the dense mesh and keeps
closed surfaces closed, partial coverage gives exactly the dense mesh of the active cells, and the lattice, plan and
refinement set are what their definitions say."""
import os

import numpy as np
import pytest

import golden_util as gu
from golden_util import ROOT, load_by_path
from recon_util import padded_random, recon, single_cell, sphere, torus, two_spheres

band = load_by_path("pnr_recon_band_oracle", os.path.join(ROOT, "oracle", "pnr_recon_band.py"))

BS = [2, 3, 4, 8]


def masked_dense(vol, iso, b):
    """the definition restated cell by cell: the dense triangles of the active cells, their vertices renumbered in
    dense order"""
    vol = np.asarray(vol, np.float32)
    rv, rt = recon.marching_cubes(vol, iso)
    if min(vol.shape) < 2:
        return rv, rt
    _, active = band.plan_of_volume(vol, iso, b)
    ins = recon.inside(vol, iso)
    keep, k = [], 0
    for x in range(vol.shape[0] - 1):
        for y in range(vol.shape[1] - 1):
            for z in range(vol.shape[2] - 1):
                cfg = sum(int(ins[x + (q & 1), y + ((q >> 1) & 1), z + ((q >> 2) & 1)]) << q for q in range(8))
                n = int(recon.TRI_COUNT[cfg])
                if active[x // b, y // b, z // b]:
                    keep += range(k, k + n)
                k += n
    t = rt[np.array(keep, dtype=np.int64)]
    used = np.unique(t)
    return rv[used], np.searchsorted(used, t).reshape(-1, 3)


def check(vol, iso, b):
    v, t, complete = band.marching_cubes(vol, iso, b)
    mv, mt = masked_dense(vol, iso, b)
    assert np.array_equal(v.view(np.int64), mv.view(np.int64)) and np.array_equal(t, mt)
    rv, rt = recon.marching_cubes(vol, iso)
    if complete:
        assert np.array_equal(v.view(np.int64), rv.view(np.int64)) and np.array_equal(t, rt)
    else:
        assert len(t) < len(rt)
    if len(t):
        assert np.array_equal(np.unique(t), np.arange(len(v)))          # every vertex is used
    return v, t, complete


@pytest.mark.parametrize("b", BS)
def test_closed_shapes_stay_closed_under_complete_coverage(b):
    for vol, iso, euler in ((sphere((21, 17, 19), 6.4), 0.0, 2), (torus((30, 28, 14), 8.0, 3.3), 0.25, 0),
                            (two_spheres((24, 14, 15), 4.1, 5.3), 0.0, 4), (padded_random((9, 8, 10), 1), 0.0, None)):
        v, t, complete = check(vol, iso, b)
        if complete:
            assert recon.is_closed_oriented(t)
            if euler is not None:
                assert recon.euler_characteristic(v, t) == euler
    assert check(sphere((33, 31, 35), 11.0), 0.0, b)[2]                 # a large sphere: every lattice sees it


@pytest.mark.parametrize("b", BS)
def test_resolutions(b):
    for shape in ((2 * b + 1, 3 * b + 1, b + 1), (2 * b, 3 * b, b), (b + 3, 2 * b - 1, 2 * b + 2), (max(b - 1, 2), 3, 2),
                  (1, 5, 6)):
        vol = sphere(shape, min(shape) * 0.45) + np.float32(0.2) * np.sin(np.arange(np.prod(shape))).reshape(
            shape).astype(np.float32)
        check(vol, 0.0, b)


def test_single_cells_empty_full_and_non_finite():
    for cfg in range(256):
        check(single_cell(cfg), 0.0, 2)
    for vol in (-np.ones((9, 7, 8), np.float32), np.ones((9, 7, 8), np.float32)):
        v, t, complete = check(vol, 0.0, 3)
        assert len(v) == len(t) == 0 and complete
        seeded, active = band.plan_of_volume(vol, 0.0, 3)
        assert not seeded.any() and not active.any()
        assert len(band.refine_index(active, vol.shape, 3, True)) == 0
    g = np.random.default_rng(3)
    vol = sphere((13, 14, 12), 4.7) + np.float32(0.5) * g.standard_normal((13, 14, 12)).astype(np.float32)
    flat = vol.reshape(-1)
    lat = band.lattice_flat(vol.shape, 3)
    flat[lat[::4]] = np.nan
    flat[lat[1::6]] = np.inf
    flat[lat[2::5]] = -np.inf
    for b in BS:
        check(vol, 0.25, b)


def test_a_blob_smaller_than_a_block_is_missed():
    vol = -np.ones((17, 17, 17), np.float32)
    vol[5:7, 5:7, 5:7] = 1.0
    v, t, complete = check(vol, 0.0, 8)
    assert not complete and len(t) == 0 and len(recon.marching_cubes(vol, 0.0)[1]) > 0
    vol[0:2, 0:2, 0:2] = 1.0                            # a surface at a lattice point: its blocks are active
    v, t, complete = check(vol, 0.0, 8)
    assert complete


def test_lattice_plan_and_refinement_set_definitions():
    for n, b, want in ((10, 4, [0, 4, 8, 9]), (9, 4, [0, 4, 8]), (3, 4, [0, 2]), (1, 4, [0]), (2, 2, [0, 1])):
        assert band.lattice_index(n, b).tolist() == want
    reso, b = (11, 9, 13), 3
    vol = sphere(reso, 3.2)
    seeded, active = band.plan_of_volume(vol, 0.0, b)
    assert active.shape == (4, 3, 4) and seeded.any() and (active >= seeded).all()
    for apron in (False, True):
        idx = band.refine_index(active, reso, b, apron)
        assert (np.diff(idx) > 0).all()
        pts = np.stack(np.unravel_index(idx, reso), -1)
        want = np.zeros(reso, dtype=bool)
        d = 1 if apron else 0
        for i, j, k in zip(*np.nonzero(active)):       # closed cells of each active block, widened by the apron
            lo = np.array([i, j, k]) * b - d
            hi = np.minimum((np.array([i, j, k]) + 1) * b, np.array(reso) - 1) + d
            lo, hi = np.maximum(lo, 0), np.minimum(hi, np.array(reso) - 1)
            want[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = True
        got = np.zeros(reso, dtype=bool)
        got[tuple(pts.T)] = True
        assert np.array_equal(got, want)                # exactly the closed cells (and apron) of the active blocks


@pytest.mark.parametrize("ns", [1, 2])
def test_golden_grids(ns):
    z = np.load(f"{gu.GOLD}/recon_ns{ns}.npz")
    for grid in ("box", "odd", "flat"):
        reso = z[f"{grid}/reso"].tolist()
        vol = z[f"{grid}/coarse"][:, 3].reshape(reso).astype(np.float32)
        iso = float(np.median(vol[np.isfinite(vol)]))
        for b in BS:
            check(vol, iso, b)
