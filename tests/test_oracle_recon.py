"""The marching-cubes tables and the numpy oracle of mesh extraction (oracle/make_mc_tables.py, oracle/pnr_recon.py):
generated header up to date, closed and consistently oriented meshes, the right topology and volume."""
import os

import numpy as np
import pytest

from golden_util import ROOT
from recon_util import mc_tables, padded_random, recon, single_cell, sphere, torus, two_spheres


def test_committed_tables_are_the_generators_output():
    with open(os.path.join(ROOT, "pixel-nerf_b200", "csrc", "pnr_mc_tables.cuh")) as f:
        assert f.read() == mc_tables.render_header()


def test_table_rows_are_sized_from_the_generator():
    t = mc_tables.tables()
    assert t["max_tris"] == max(t["tri_count"])
    assert all(len(row) == 3 * t["max_tris"] for row in t["tris"])
    assert t["tri_count"][0] == 0 and t["tri_count"][255] == 0


def test_every_single_cell_configuration_is_closed_and_oriented():
    for cfg in range(1, 255):
        v, t = recon.marching_cubes(single_cell(cfg), 0.0)
        assert recon.is_closed_oriented(t), cfg
        assert recon.signed_volume(v, t) > 0, cfg
        assert len(np.unique(t)) == len(v), cfg          # every vertex is used


def test_sphere_euler_characteristic_and_volume():
    r = 11.3
    v, t = recon.marching_cubes(sphere((30, 27, 32), r), 0.0)
    assert recon.is_closed_oriented(t)
    assert recon.euler_characteristic(v, t) == 2
    assert recon.components(t) == 1
    assert abs(recon.signed_volume(v, t) / (4.0 / 3.0 * np.pi * r ** 3) - 1.0) < 0.03


def test_inverted_sphere_faces_the_other_way():
    v, t = recon.marching_cubes(-sphere((20, 20, 20), 6.0), 0.0)
    assert recon.is_closed_oriented(t)
    assert recon.signed_volume(v, t) < 0      # the inside is everything but the ball: normals point into the ball


def test_torus_and_two_spheres():
    v, t = recon.marching_cubes(torus((34, 34, 16), 9.0, 3.5), 0.0)
    assert recon.is_closed_oriented(t)
    assert recon.euler_characteristic(v, t) == 0
    v, t = recon.marching_cubes(two_spheres((36, 20, 20), 5.0, 8.0), 0.0)
    assert recon.is_closed_oriented(t)
    assert recon.components(t) == 2
    assert recon.euler_characteristic(v, t) == 4


def test_no_fan_diagonal_lies_in_a_cube_face():
    """A cell's triangle edges used twice inside the cell are its fans' diagonals; none may lie in a cube face, where the
    neighbouring cell could draw it too."""
    for cfg in range(256):
        uses = {}
        for t in mc_tables.config_triangles(cfg):
            for e in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
                uses[tuple(sorted(e))] = uses.get(tuple(sorted(e)), 0) + 1
        diagonals = [e for e, n in uses.items() if n == 2]
        assert not any(mc_tables.shares_face(*e) for e in diagonals), cfg


@pytest.mark.parametrize("seed", range(12))
def test_random_fields_with_ambiguous_faces_stay_watertight(seed):
    v, t = recon.marching_cubes(padded_random((6, 6, 6), seed), 0.0)
    assert len(t) > 0
    assert recon.is_closed_oriented(t)
    assert recon.signed_volume(v, t) > 0


def test_vertices_interpolate_to_iso_on_their_edge():
    iso = 0.37
    vol = sphere((15, 12, 17), 5.2) + np.float32(0.4) * np.sin(np.arange(15 * 12 * 17)).reshape(15, 12, 17).astype(
        np.float32)
    v, _ = recon.marching_cubes(vol, iso)
    lower = np.floor(v).astype(np.int64)
    frac = v - lower
    axis = np.argmax(frac, axis=1)
    assert (np.count_nonzero(frac, axis=1) <= 1).all()          # on a grid edge
    upper = lower + np.eye(3, dtype=np.int64)[axis]
    sa = vol[tuple(lower.T)].astype(np.float64)
    sb = vol[tuple(upper.T)].astype(np.float64)
    t = frac[np.arange(len(v)), axis]
    assert ((sa > iso) != (sb > iso)).all()
    np.testing.assert_allclose(sa + t * (sb - sa), iso, atol=1e-12)


def test_inside_test_excludes_non_finite_values():
    vol = np.array([np.nan, np.inf, -np.inf, 0.5, 0.5000001, 2.0], dtype=np.float32)
    assert recon.inside(vol, 0.5).tolist() == [False, False, False, False, True, True]
