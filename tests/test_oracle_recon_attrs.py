"""Per-vertex normals and query points of the numpy oracle (oracle/pnr_recon_attrs.py vertex_attrs, the reference
pnr_mc_vertex_attrs is checked against): normals agree with the winding and with a sphere's radial direction, the
fallback along a flat edge, non-finite sigma kept out of the normals, and save_obj with normals."""
import os
import sys

import numpy as np
import pytest

from golden_util import ROOT, load_by_path
from recon_util import recon, sphere, torus

sys.path.insert(0, os.path.join(ROOT, "pixel-nerf_b200", "src"))
attrs = load_by_path("pnr_recon_attrs_oracle", os.path.join(ROOT, "oracle", "pnr_recon_attrs.py"))


def unit_box(shape):
    """Bounds that make world units index units (h = 1 on every axis)."""
    return (0.0, 0.0, 0.0), tuple(float(n - 1) for n in shape)


def attrs_and_mesh(vol, iso=0.0, bounds=None):
    lo, hi = bounds or unit_box(vol.shape)
    n, xyz, vd = attrs.vertex_attrs(vol, iso, lo, hi)
    v, t = recon.marching_cubes(vol, iso)
    assert n.shape == v.shape and xyz.shape == v.shape and vd.shape == v.shape
    assert n.dtype == np.float64 and xyz.dtype == np.float32 and vd.dtype == np.float32
    return n, xyz, vd, v, t


@pytest.mark.parametrize("field", ["sphere", "torus"])
def test_normals_agree_with_the_winding(field):
    vol = sphere((40, 36, 44), 12.3) if field == "sphere" else torus((48, 48, 48), 14.2, 5.1)
    n, xyz, vd, v, t = attrs_and_mesh(vol)
    assert len(t) > 5000
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    face = np.cross(b - a, c - a)                      # counter-clockwise from outside: toward decreasing sigma
    vsum = n[t[:, 0]] + n[t[:, 1]] + n[t[:, 2]]
    assert (np.einsum("ij,ij->i", face, vsum) > 0).all()
    np.testing.assert_allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-12)
    assert np.array_equal(vd, (-n).astype(np.float32))
    # with h = 1 the query point is the vertex itself
    assert np.array_equal(xyz, v.astype(np.float32))


def test_sphere_normals_are_radial():
    shape = (40, 36, 44)
    n, _, _, v, _ = attrs_and_mesh(sphere(shape, 12.3))
    radial = v - (np.array(shape) - 1) / 2.0
    radial /= np.linalg.norm(radial, axis=1, keepdims=True)
    angle = np.degrees(np.arccos(np.clip(np.einsum("ij,ij->i", n, radial), -1.0, 1.0)))
    print(f"{len(v)} vertices, largest angle to radial {angle.max():.3f} deg")
    assert angle.max() < 0.2


def test_world_units_and_query_points_on_a_non_cubic_box():
    shape = (40, 36, 44)
    vol = sphere(shape, 12.3)
    lo, hi = (-0.55, -0.6, -0.5), (0.6, 0.5, 0.55)
    n, xyz, _, v, _ = attrs_and_mesh(vol, bounds=(lo, hi))
    h = (np.array(hi) - np.array(lo)) / (np.array(shape) - 1)
    # the normal of an anisotropic grid is the index-space gradient divided by h, normalised
    n1, _, _, _, _ = attrs_and_mesh(vol)
    g = n1 / h
    np.testing.assert_allclose(n, g / np.linalg.norm(g, axis=1, keepdims=True), atol=1e-12)
    # on integer coordinates the query point has np.linspace's bits (the grid points'); elsewhere lo + v h
    grid = recon.grid_points(lo, hi, shape).reshape(shape + (3,))
    idx = np.floor(v).astype(np.int64)
    on = v == idx
    at_grid = grid[tuple(idx.T)]
    assert np.array_equal(xyz[on], at_grid[on])
    np.testing.assert_allclose(xyz, v * h + np.array(lo), atol=1e-6)


def test_flat_edge_falls_back_to_the_edge_axis():
    # +, -, +, - along x: the central differences vanish at x = 1 and x = 2, so G = 0 on the middle edge
    vol = np.empty((4, 2, 3), dtype=np.float32)
    vol[:] = np.array([1.0, -1.0, 1.0, -1.0], dtype=np.float32)[:, None, None]
    n, _, _, v, _ = attrs_and_mesh(vol)
    mid = v[:, 0] == 1.5
    assert mid.sum() == 6
    assert np.array_equal(n[mid], np.tile([-1.0, 0.0, 0.0], (6, 1)))     # from the inside corner x = 2 to x = 1
    assert np.array_equal(n[v[:, 0] == 0.5], np.tile([1.0, 0.0, 0.0], (6, 1)))
    assert np.array_equal(n[v[:, 0] == 2.5], np.tile([1.0, 0.0, 0.0], (6, 1)))
    # x runs backwards in the world: every normal turns over, the fallback with them
    lo, hi = (3.0, 0.0, 0.0), (0.0, 1.0, 2.0)
    nb, _, _, _, _ = attrs_and_mesh(vol, bounds=(lo, hi))
    assert np.array_equal(nb, -n)
    # a flat box (lo = hi) divides by h = 0: the fallback again
    nf, _, _, _, _ = attrs_and_mesh(vol, bounds=((0.0, 0.0, 0.0), (0.0, 1.0, 2.0)))
    assert np.array_equal(nf[mid], n[mid]) and np.isfinite(nf).all()


def test_gradient_rules():
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    vol = np.zeros((5, 2, 2), dtype=np.float32)
    vol[:, 0, 0] = [1.0, 2.0, nan, 4.0, 7.0]
    g = attrs.grid_gradient(vol)[:, 0, 0, 0]
    # x = 0 forward; x = 1 backward (its upper neighbour is NaN); x = 2 central across the NaN; x = 3 forward;
    # x = 4 backward
    assert g.tolist() == [1.0, 1.0, 1.0, 3.0, 3.0]
    vol[:, 0, 0] = [inf, 2.0, 5.0, -inf, nan]
    g = attrs.grid_gradient(vol)[:, 0, 0, 0]
    assert g.tolist() == [0.0, 3.0, 3.0, 0.0, 0.0]


def test_non_finite_sigma_gives_no_nan_normal():
    g = np.random.default_rng(11)
    vol = g.standard_normal((9, 10, 11)).astype(np.float32)
    flat = vol.reshape(-1)
    idx = g.permutation(flat.size)
    flat[idx[:25]] = np.nan
    flat[idx[25:40]] = np.inf
    flat[idx[40:55]] = -np.inf
    n, xyz, vd, v, _ = attrs_and_mesh(vol, 0.1, bounds=((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)))
    assert len(v) > 500
    assert np.isfinite(n).all() and np.isfinite(xyz).all() and np.isfinite(vd).all()
    np.testing.assert_allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-12)


def test_a_nan_at_the_grid_origin_stays_out_of_its_neighbours_normals():
    """An odd grid over a box centred on 0 has a point at the origin, where sigma is NaN (0 / 0 view direction).  The
    normals of every vertex whose edge and corner neighbours avoid it are those of the field without the NaN."""
    shape = (21, 21, 21)
    clean = sphere(shape, 5.3)
    vol = clean.copy()
    vol[10, 10, 10] = np.nan
    box = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    n0, x0, _, v0, _ = attrs_and_mesh(clean, bounds=box)
    n1, x1, _, v1, _ = attrs_and_mesh(vol, bounds=box)
    assert np.isfinite(n1).all()
    far0 = np.abs(v0 - 10.0).max(axis=1) > 2.0
    far1 = np.abs(v1 - 10.0).max(axis=1) > 2.0
    assert far0.sum() > 100 and far0.sum() == far1.sum()
    assert np.array_equal(n1[far1], n0[far0]) and np.array_equal(x1[far1], x0[far0])
    assert (~far1).sum() == 6                          # the NaN point's own little surface


def test_empty_and_degenerate_volumes():
    n, xyz, vd = attrs.vertex_attrs(np.zeros((1, 4, 4), np.float32), 0.0, (0, 0, 0), (1, 1, 1))
    assert n.shape == xyz.shape == vd.shape == (0, 3)
    n, xyz, vd = attrs.vertex_attrs(-np.ones((4, 4, 4), np.float32), 0.0, (0, 0, 0), (1, 1, 1))
    assert n.shape == (0, 3)


def _old_obj(vertices, triangles, vert_rgb=None):
    """The OBJ text save_obj wrote before it took normals."""
    rows = vertices if vert_rgb is None else np.concatenate([vertices, vert_rgb], axis=1)
    vfmt = "v" + " %.4f" * rows.shape[1] + "\n"
    return "".join(vfmt % tuple(r) for r in rows) + "".join(
        "f %d %d %d\n" % (a + 1, b + 1, c + 1) for a, b, c in triangles)


def test_save_obj_with_normals(tmp_path):
    from util import recon as urecon
    n, _, _, v, t = attrs_and_mesh(sphere((14, 12, 13), 4.1))
    rgb = np.random.default_rng(0).random(v.shape).astype(np.float32)
    path = tmp_path / "mesh.obj"
    urecon.save_obj(v, t, str(path), vert_rgb=rgb, vert_normals=n)
    lines = path.read_text().splitlines()
    vl = [ln for ln in lines if ln.startswith("v ")]
    vn = [ln for ln in lines if ln.startswith("vn ")]
    fl = [ln for ln in lines if ln.startswith("f ")]
    assert len(vl) == len(vn) == len(v) and len(fl) == len(t) and len(lines) == 2 * len(v) + len(t)
    assert lines[:len(v)] == vl and lines[len(v):2 * len(v)] == vn          # v lines, then vn lines, then faces
    assert all(len(ln.split()) == 7 for ln in vl)
    assert all(ln == "vn %.4f %.4f %.4f" % tuple(x) for ln, x in zip(vn, n))
    np.testing.assert_allclose(np.array([[float(x) for x in ln.split()[1:]] for ln in vn]), n, atol=0.5e-4 + 1e-12)
    pairs = np.array([[[int(i) for i in c.split("//")] for c in ln.split()[1:]] for ln in fl])
    assert np.array_equal(pairs[..., 0], pairs[..., 1]) and np.array_equal(pairs[..., 0] - 1, t)
    # without normals the file is what it always was
    for kw in ({}, {"vert_rgb": rgb}):
        urecon.save_obj(v, t, str(path), **kw)
        assert path.read_bytes() == _old_obj(v, t, kw.get("vert_rgb")).encode()
