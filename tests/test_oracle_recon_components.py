"""The connected-components rule (oracle/pnr_recon_components.py, the restatement pnr_mesh_components /
pnr_mesh_compact_* and util.recon.keep_components are compared against): labels against a plain union-find on random
soups; on one large and four small spheres meshed by the marching-cubes oracle, keeping the largest or those above a
size gives exactly the marching cubes of just those spheres; ties, meshes kept whole, unused vertices and empty meshes."""
import numpy as np
import pytest

from components_util import BIG, SMALL, bits_equal, comp, mesh_of, random_soup, union_find_labels
from recon_util import recon


@pytest.mark.parametrize("seed", range(6))
def test_labels_match_a_plain_union_find(seed):
    g = np.random.default_rng(100 + seed)
    n = int(g.integers(1, 300))
    tris = random_soup(seed, n, int(g.integers(0, 2 * n)))
    label = comp.labels(tris, n)
    assert np.array_equal(label, union_find_labels(tris, n))
    assert (label <= np.arange(n)).all() and (label[label] == label).all()
    counts = comp.tri_counts(tris, label)
    assert counts.sum() == len(tris) and (counts[label != np.arange(n)] == 0).all()
    if len(tris):
        assert np.count_nonzero(counts) == recon.components(tris)      # the existing independent count


def test_largest_is_the_big_sphere_alone():
    v, t = mesh_of([BIG] + SMALL)
    assert comp.labels(t, len(v)).max() > 0 and np.count_nonzero(comp.tri_counts(t, comp.labels(t, len(v)))) == 5
    kv, kt = comp.keep_components(v, t, largest=1)
    want_v, want_t = mesh_of([BIG])
    assert bits_equal(kv, want_v) and bits_equal(kt, want_t)
    assert recon.is_closed_oriented(kt)


def test_min_triangles_keeps_the_spheres_above_it():
    v, t = mesh_of([BIG] + SMALL)
    sizes = {r: len(mesh_of([s])[1]) for s in SMALL for r in [s[1]]}
    assert len(set(sizes.values())) == len(SMALL)                       # distinct sizes
    for k in sorted(sizes.values()) + [1, max(sizes.values()) + 1]:
        kv, kt = comp.keep_components(v, t, largest=None, min_triangles=k)
        want_v, want_t = mesh_of([BIG] + [s for s in SMALL if sizes[s[1]] >= k])
        assert bits_equal(kv, want_v) and bits_equal(kt, want_t), k
        assert recon.is_closed_oriented(kt)
    # largest and min_triangles together: the two largest of those above the smallest size
    kv, kt = comp.keep_components(v, t, largest=2, min_triangles=sorted(sizes.values())[1])
    biggest_small = max(SMALL, key=lambda s: sizes[s[1]])
    want_v, want_t = mesh_of([BIG, biggest_small])
    assert bits_equal(kv, want_v) and bits_equal(kt, want_t)


def test_ties_go_to_the_smaller_vertex_id():
    # two identical spheres 20 voxels apart along x: the same cells, so the same triangle count; the one at lower x has
    # the smaller vertex ids
    a, b = ((-10.0, 0.0, 0.0), 4.0), ((10.0, 0.0, 0.0), 4.0)
    v, t = mesh_of([a, b])
    la = comp.labels(t, len(v))
    counts = comp.tri_counts(t, la)
    assert sorted(counts[counts > 0].tolist()) == [len(t) // 2] * 2
    kv, kt = comp.keep_components(v, t, largest=1)
    want_v, want_t = mesh_of([a])
    assert bits_equal(kv, want_v) and bits_equal(kt, want_t)
    # and on a soup: components {5, 6, 7} and {0, 1, 2} of one triangle each, listed larger ids first
    tris = np.array([[5, 6, 7], [0, 1, 2]])
    verts = np.arange(24, dtype=np.float32).reshape(8, 3)
    kv, kt = comp.keep_components(verts, tris, largest=1)
    assert bits_equal(kv, verts[:3]) and bits_equal(kt, np.array([[0, 1, 2]]))


def test_everything_kept_is_bit_equal_and_unused_vertices_drop():
    v, t = mesh_of([BIG] + SMALL)
    g = np.random.default_rng(3)
    normals, rgb = g.normal(size=v.shape), g.random(v.shape).astype(np.float32)
    out = comp.keep_components(v, t, normals, rgb, largest=None)
    for got, want in zip(out, (v, t, normals, rgb)):
        assert bits_equal(got, want)
    # unused vertices: vertex 0 and the last, inserted around the mesh
    v2 = np.concatenate([v[:1] * 0 + 9.0, v, v[:1] * 0 - 9.0])
    out = comp.keep_components(v2, (t + 1).astype(np.int32), normals[np.r_[0, :len(v), 0]], largest=None)
    assert bits_equal(out[0], v) and bits_equal(out[1], t.astype(np.int32)) and bits_equal(out[2], normals)


def test_empty_meshes_and_lonely_vertices():
    shapes = lambda out: [(a.shape, a.dtype) for a in out]     # noqa: E731
    attr = np.zeros((0, 2, 2), dtype=np.float16)
    out = comp.keep_components(np.zeros((0, 3)), np.zeros((0, 3), dtype=np.int64), attr)
    assert shapes(out) == [((0, 3), np.float64), ((0, 3), np.int64), ((0, 2, 2), np.float16)]
    verts = np.ones((4, 3), dtype=np.float32)
    out = comp.keep_components(verts, np.zeros((0, 3), dtype=np.int32), np.arange(4), largest=None)
    assert shapes(out) == [((0, 3), np.float32), ((0, 3), np.int32), ((0,), np.arange(4).dtype)]
    label = comp.labels(np.zeros((0, 3), dtype=np.int64), 4)
    assert np.array_equal(label, np.arange(4)) and not comp.tri_counts(np.zeros((0, 3)), label).any()
