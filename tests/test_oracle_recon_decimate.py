"""The decimation oracle (oracle/pnr_recon_decimate.py) on analytic meshes: closed meshes stay closed with every
directed edge once, each component keeps its Euler characteristic (the torus its genus), the target is met, a
decimated sphere stays outward-facing and near its radius, a flat patch loses most interior vertices at zero error
with its boundary and area unchanged, max_error bounds every collapse, a mesh at or under the target comes back, and
degenerate inputs pass through."""
import numpy as np
import pytest

from components_util import BIG, SMALL, mesh_of
from decimate_util import (area, bipyramid, bits_equal, boundary_edges, dec, euler_per_component, flat_patch, is_closed,
                           rows_of, sphere_mesh, torus_mesh)


@pytest.mark.parametrize("mesh", ["sphere", "torus", "spheres"])
def test_closed_topology_and_target(mesh):
    v, t = {"sphere": sphere_mesh, "torus": torus_mesh, "spheres": lambda: mesh_of([BIG] + SMALL)}[mesh]()
    t = t.astype(np.int64)
    assert is_closed(t)
    chi = euler_per_component(v, t)
    target = len(t) // 4
    ov, ot = dec.decimate(v, t, target_triangles=target)
    assert len(ot) in (target - 1, target), (len(ot), target)
    assert is_closed(ot)
    rows = rows_of(ov, v)
    assert (np.diff(rows) > 0).all() and bits_equal(ov, v[rows])
    # components keep their Euler characteristic: relabel by the input rows' smallest id
    got = {int(rows[k]): x for k, x in euler_per_component(ov, ot).items()}
    assert sorted(got.values()) == sorted(chi.values())
    if mesh == "torus":
        assert list(chi.values()) == [0] and list(got.values()) == [0]


def test_sphere_to_2000_faces_outward_and_stays_on_the_radius():
    v, t = sphere_mesh(48, 20.0)
    c = (np.array([48, 48, 48]) - 1) / 2.0                       # the grid's centre in vertex coordinates
    ov, ot = dec.decimate(v, t, target_triangles=2000)
    assert len(ot) in (1999, 2000) and is_closed(ot)
    p = ov.astype(np.float64) - c
    n = np.cross(p[ot[:, 1]] - p[ot[:, 0]], p[ot[:, 2]] - p[ot[:, 0]])
    centroid = p[ot].mean(1)
    assert ((n * centroid).sum(1) > 0).all()                     # every triangle faces outward
    g = np.random.default_rng(0)
    w = g.dirichlet([1, 1, 1], size=(len(ot), 4))
    pts = np.einsum("tkj,tjd->tkd", w, p[ot]).reshape(-1, 3)
    r = np.linalg.norm(pts, axis=1)
    print(f"{len(ot)} triangles, sample radius {r.min():.3f} .. {r.max():.3f} of 20")
    # the vertices lie on the sphere to within marching cubes' error, and the flat triangles between them cut
    # inside by their sagitta: every sample is within 0.2 voxel inside and 0.1 voxel outside the radius
    assert r.max() < 20.1 and r.min() > 19.8


def test_flat_patch_at_zero_error():
    v, t = flat_patch(24)
    interior = 22 * 22
    tris, _, counts, errs, reason = dec.rounds(v, t, max_error=0.0)
    assert reason in ("error bound", "no valid collapse left") and (errs == 0).all()
    assert boundary_edges(tris) == boundary_edges(t)
    assert area(v, tris) == pytest.approx(area(v, t), rel=1e-12)
    left = len(np.setdiff1d(np.unique(tris), np.unique(t[np.isin(t, list({a for e in boundary_edges(t) for a in e}))])))
    print(f"{sum(counts)} collapses in {len(counts)} rounds; {left} of {interior} interior vertices left")
    assert sum(counts) == interior and left == 0                 # every interior vertex is gone
    # the same with a target below what is reachable stops for lack of valid collapses, not for the bound
    assert dec.rounds(v, t, target_triangles=0)[4] == "no valid collapse left"


def test_max_error_bounds_every_collapse():
    v, t = sphere_mesh(32, 12.0)
    for bound in (0.0, 0.01, 0.05):
        tris, _, counts, errs, reason = dec.rounds(v, t, max_error=bound)
        assert (errs <= bound).all() and reason == "error bound", (bound, reason)
        print(f"max_error {bound}: {len(t)} -> {len(tris)} triangles in {len(counts)} rounds")
    tris_both = dec.rounds(v, t, target_triangles=len(t) // 2, max_error=0.05)
    assert len(tris_both[0]) >= len(t) // 2 - 1


def test_target_at_or_above_the_mesh_returns_it():
    v, t = sphere_mesh(20, 6.0)
    rgb = np.random.default_rng(1).random((len(v), 3)).astype(np.float32)
    for target in (len(t), len(t) + 5):
        out = dec.decimate(v, t, rgb, target_triangles=target)
        assert bits_equal(out[0], v) and bits_equal(out[1], t) and bits_equal(out[2], rgb)
    # unused vertices are dropped, the rest renumbered in order
    v2 = np.concatenate([v[:1] + 100, v])
    out = dec.decimate(v2, t + 1, target_triangles=len(t))
    assert bits_equal(out[0], v) and bits_equal(out[1], t)


def test_empty_and_degenerate_inputs():
    out = dec.decimate(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), target_triangles=0)
    assert out[0].shape == (0, 3) and out[1].shape == (0, 3)
    v, t = sphere_mesh(20, 6.0)
    n = len(v)
    # a zero-area sliver (a repeated position), a repeated id and a fin on a non-manifold edge
    v = np.concatenate([v, v[t[0, :1]], v[t[0, 1:2]] + 5.0])
    extra = np.array([[t[0, 0], t[0, 1], n], [t[1, 0], t[1, 0], t[1, 2]], [t[2, 0], t[2, 1], n + 1]])
    t2 = np.concatenate([t, extra])
    q = dec.quadrics(v, t2)
    assert np.isfinite(q).all()
    ov, ot, ids = dec.decimate(v, t2, np.arange(len(v)), target_triangles=len(t2) // 3)
    assert len(ot) <= len(t2) // 3 + 1
    kept = {tuple(x) for x in ids[ot].tolist()}
    for tri in extra.tolist():                                   # the degenerate triangles are never touched
        assert tuple(tri) in kept
    assert bits_equal(ov, v[ids])


def test_the_tetrahedron_is_kept():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float64)
    t = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], dtype=np.int64)
    ov, ot = dec.decimate(v, t, target_triangles=0)
    assert bits_equal(ov, v) and bits_equal(ot, t)


def test_vertices_over_64_corners_are_frozen():
    """The apexes of a bipyramid with a ring of 100 have 100 corners: they are frozen for the whole call, so the
    ring collapses around them but they stay, and the mesh keeps its height instead of flattening into a disk."""
    v, t = bipyramid(100)
    assert list(np.nonzero(dec.frozen(t, len(v)))[0]) == [100, 101]
    for kw in (dict(max_error=0.05), dict(target_triangles=8)):
        tris, _, counts, errs, reason = dec.rounds(v, t, **kw)
        assert {100, 101} <= set(np.unique(tris).tolist()) and is_closed(tris)
        assert sum(counts) > 50 and (errs <= kw.get("max_error", np.inf)).all()
        print(kw, f"{len(t)} -> {len(tris)} triangles in {len(counts)} rounds ({reason})")
