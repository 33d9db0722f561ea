"""Meshes and checks for the decimation tests: analytic marching-cubes meshes, a flat open patch, mesh invariants
(closedness, Euler characteristic per component, boundary edges, area), and the oracle (oracle/pnr_recon_decimate.py)
itself."""
import os

import numpy as np

from components_util import bits_equal, comp  # noqa: F401  (re-exported for the tests)
from golden_util import ROOT, load_by_path
from recon_util import recon, sphere, torus

dec = load_by_path("pnr_recon_decimate_oracle", os.path.join(ROOT, "oracle", "pnr_recon_decimate.py"))


def sphere_mesh(n=32, r=12.0):
    v, t = recon.marching_cubes(sphere((n, n, n), r), 0.0)
    return v, t.astype(np.int64)


def torus_mesh(n=40, R=11.0, r=4.5):
    v, t = recon.marching_cubes(torus((n, n, n), R, r), 0.0)
    return v, t.astype(np.int64)


def flat_patch(n=24, seed=0):
    """An (n x n)-vertex grid in the plane z = 0 with jittered interior points, two triangles per cell, oriented +z."""
    g = np.random.default_rng(seed)
    X, Y = np.meshgrid(np.arange(n, dtype=np.float64), np.arange(n, dtype=np.float64), indexing="ij")
    inner = (X > 0) & (X < n - 1) & (Y > 0) & (Y < n - 1)
    X = X + np.where(inner, g.uniform(-0.3, 0.3, X.shape), 0.0)
    Y = Y + np.where(inner, g.uniform(-0.3, 0.3, Y.shape), 0.0)
    v = np.stack([X.ravel(), Y.ravel(), np.zeros(n * n)], axis=1)
    i, j = np.meshgrid(np.arange(n - 1), np.arange(n - 1), indexing="ij")
    a = (i * n + j).ravel()
    b, c, d = a + n, a + n + 1, a + 1
    t = np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)]).astype(np.int64)
    return v, t


def bipyramid(k):
    """A closed bipyramid: a ring of k vertices in the unit circle (slightly twisted, to break ties) and two apexes at
    z = +-1 with k corners each."""
    a = np.arange(k) * 2 * np.pi / k
    ring = np.stack([np.cos(a), np.sin(a), 0.01 * np.sin(3 * a)], 1)
    v = np.concatenate([ring, [[0, 0, 1.0], [0, 0, -1.0]]])
    i = np.arange(k)
    t = np.concatenate([np.stack([i, (i + 1) % k, np.full(k, k)], 1), np.stack([(i + 1) % k, i, np.full(k, k + 1)], 1)])
    return v, t.astype(np.int64)


def directed_edges(t):
    return np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])


def is_closed(t):
    """Every directed edge appears once and its reverse once."""
    e = directed_edges(t)
    s = {tuple(x) for x in e.tolist()}
    return len(s) == len(e) and all((b, a) in s for a, b in s)


def boundary_edges(t):
    e = directed_edges(t)
    s = {tuple(x) for x in e.tolist()}
    return {x for x in s if (x[1], x[0]) not in s}


def euler_per_component(v, t):
    """{smallest vertex id of the component: V - E + F} over the components with triangles."""
    t = np.asarray(t, np.int64)
    n = len(v)
    label = comp.labels(t, n)
    used = np.unique(t)
    e = np.sort(directed_edges(t), axis=1)
    e = np.unique(e[:, 0] * n + e[:, 1]) // n                     # first vertex of each undirected edge
    chi = (np.bincount(label[used], minlength=n) - np.bincount(label[e], minlength=n) +
           np.bincount(label[t[:, 0]], minlength=n))
    return {int(r): int(chi[r]) for r in np.unique(label[t[:, 0]])}


def directed_edges_once(t):
    """No directed edge appears twice (every edge manifold and consistently oriented)."""
    e = directed_edges(np.asarray(t, np.int64))
    k = e[:, 0] * (int(e.max()) + 1 if len(e) else 1) + e[:, 1]
    return len(np.unique(k)) == len(k)


def area(v, t):
    v = np.asarray(v, np.float64)
    return 0.5 * np.linalg.norm(np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]]), axis=1).sum()


def rows_of(out_v, v):
    """The input row of every output vertex (they are input rows, in input order)."""
    idx = {tuple(r): i for i, r in reversed(list(enumerate(np.asarray(v).tolist())))}
    return np.array([idx[tuple(r)] for r in np.asarray(out_v).tolist()], dtype=np.int64)
