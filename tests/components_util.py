"""Meshes for the connected-components tests: random triangle soups with many components, a plain-Python union-find
to check the oracle with, and an analytic scene of one large and several small spheres; plus the oracle
(oracle/pnr_recon_components.py) itself."""
import os

import numpy as np

from golden_util import ROOT, load_by_path
from recon_util import recon

comp = load_by_path("pnr_recon_components_oracle", os.path.join(ROOT, "oracle", "pnr_recon_components.py"))


def union_find_labels(tris, n_verts):
    """label[v] = the smallest vertex id of v's component, by a plain union-find over every edge of every triangle."""
    parent = list(range(n_verts))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b, c in np.asarray(tris).tolist():
        for u, v in ((a, b), (b, c), (a, c)):
            ru, rv = find(u), find(v)
            if ru != rv:
                parent[max(ru, rv)] = min(ru, rv)
    return np.array([find(v) for v in range(n_verts)], dtype=np.int64)


def random_soup(seed, n_verts, n_tris, sizes=None):
    """Triangles [n_tris, 3] int64 over n_verts vertices, each triangle's three vertices drawn from one group of a
    random partition of the vertices (group sizes from 1 to `sizes`' largest; some vertices end up unused), with the
    vertex ids shuffled so that the groups interleave in id order."""
    g = np.random.default_rng(seed)
    if sizes is None:
        sizes = g.integers(1, max(2, n_verts // 8), size=n_verts)
    sizes = np.asarray(sizes, dtype=np.int64)
    sizes = sizes[np.cumsum(sizes) <= n_verts]
    start = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    group = g.choice(len(sizes), size=n_tris, p=sizes / sizes.sum())
    local = (g.random((n_tris, 3)) * sizes[group][:, None]).astype(np.int64)
    perm = g.permutation(n_verts)
    return perm[start[group][:, None] + local].astype(np.int64)


SHAPE = (48, 40, 40)
# (centre, radius) in the centred voxel coordinates of recon_util.centred: one large sphere and four small ones of
# different sizes, at least 14 voxels apart, so no cell near one sphere sees another
BIG = ((-8.0, 0.0, 0.0), 10.0)
SMALL = [((15.0, 12.0, 12.0), 2.5), ((15.0, -12.0, 12.0), 3.5), ((15.0, 12.0, -12.0), 1.6), ((16.0, -12.0, -12.0), 4.0)]


def sphere_field(spheres, shape=SHAPE):
    """sigma = max over the spheres of (r - |x - c|), each term rounded to float32: inside (> 0) within any sphere."""
    axes = [np.arange(n, dtype=np.float64) - (n - 1) / 2.0 for n in shape]
    X, Y, Z = np.meshgrid(*axes, indexing="ij")
    vol = np.full(shape, -np.inf, dtype=np.float32)
    for (cx, cy, cz), r in spheres:
        s = (r - np.sqrt((X - cx) ** 2 + (Y - cy) ** 2 + (Z - cz) ** 2)).astype(np.float32)
        vol = np.maximum(vol, s)
    return vol


def mesh_of(spheres):
    return recon.marching_cubes(sphere_field(spheres), 0.0)


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
