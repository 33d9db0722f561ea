"""Fields for the mesh-extraction tests and the oracle / table modules they check against."""
import os

import numpy as np

from golden_util import ROOT, load_by_path

recon = load_by_path("pnr_recon_oracle", os.path.join(ROOT, "oracle", "pnr_recon.py"))
mc_tables = recon.mc_tables


def centred(shape):
    """Coordinates of a grid of `shape`, centred on its middle."""
    axes = [np.arange(n, dtype=np.float64) - (n - 1) / 2.0 for n in shape]
    return np.meshgrid(*axes, indexing="ij")


def sphere(shape, r, centre=(0.0, 0.0, 0.0)):
    """r - |p - centre|: inside (> 0) within radius r."""
    X, Y, Z = centred(shape)
    return (r - np.sqrt((X - centre[0]) ** 2 + (Y - centre[1]) ** 2 + (Z - centre[2]) ** 2)).astype(np.float32)


def torus(shape, R, r):
    X, Y, Z = centred(shape)
    q = np.sqrt(X * X + Y * Y) - R
    return (r - np.sqrt(q * q + Z * Z)).astype(np.float32)


def two_spheres(shape, r, gap):
    return np.maximum(sphere(shape, r, (-gap, 0, 0)), sphere(shape, r, (gap, 0, 0)))


def padded_random(shape, seed):
    """Random +-1 values inside a border of -1 (so the surface is closed); many faces are ambiguous."""
    g = np.random.default_rng(seed)
    v = -np.ones(shape, dtype=np.float32)
    v[1:-1, 1:-1, 1:-1] = g.choice(np.array([-1.0, 1.0], dtype=np.float32), size=tuple(n - 2 for n in shape))
    return v


def single_cell(cfg):
    """Configuration `cfg` (bit k = corner k inside) in the middle of a 4^3 grid of outside values."""
    v = -np.ones((4, 4, 4), dtype=np.float32)
    for k in range(8):
        if (cfg >> k) & 1:
            v[1 + (k & 1), 1 + ((k >> 1) & 1), 1 + ((k >> 2) & 1)] = 1.0
    return v
