"""
ORACLE -- numpy restatement of pnr_mc_vertex_attrs (csrc/pnr_recon.cu): the per-vertex normals, query points and view
directions of the mesh oracle/pnr_recon.py's marching_cubes extracts, in the kernel's operation order, so that the
kernel is compared against it bit for bit.

  grid_gradient   vol -> float64 [nx][ny][nz][3], the sigma gradient at each grid point in index units: per axis the
                  central difference (s[p+e] - s[p-e]) / 2 where both neighbours exist and are finite, else
                  s[p+e] - s[p] or s[p] - s[p-e] where both of its values are finite, else 0
  vertex_attrs    vol, iso, lo, hi -> (normals float64 [N][3], xyz float32 [N][3], viewdirs float32 [N][3]) of the
                  marching_cubes vertices, in their order: G = ((1 - t) g(a) + t g(b)) / h with the vertex's t and
                  h = (hi - lo) / (n - 1); normal -G / sqrt((Gx^2 + Gy^2) + Gz^2), or the edge's axis from its inside
                  corner to its outside one (in world coordinates) where that length is 0 or not finite;
                  xyz = lo + v h (hi at v = n - 1) rounded to float32; viewdirs = -normal in float32
"""
import importlib.util
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("pnr_recon_oracle_base", os.path.join(_HERE, "pnr_recon.py"))
_recon = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_recon)
inside = _recon.inside


def grid_gradient(vol):
    v = np.asarray(vol, dtype=np.float32).astype(np.float64)
    g = np.zeros(v.shape + (3,))
    for k in range(3):
        c = np.moveaxis(v, k, 0)
        up = np.full_like(c, np.nan)                   # a missing neighbour counts as non-finite
        dn = np.full_like(c, np.nan)
        up[:-1], dn[1:] = c[1:], c[:-1]
        fu, fd, fc = np.isfinite(up), np.isfinite(dn), np.isfinite(c)
        with np.errstate(invalid="ignore", over="ignore"):
            gk = np.where(fu & fd, (up - dn) / 2.0, np.where(fu & fc, up - c, np.where(fd & fc, c - dn, 0.0)))
        np.moveaxis(g[..., k], k, 0)[...] = gk
    return g


def vertex_attrs(vol, iso, lo, hi):
    vol = np.asarray(vol, dtype=np.float32)
    dims = vol.shape
    if min(dims) < 2:
        return np.zeros((0, 3)), np.zeros((0, 3), dtype=np.float32), np.zeros((0, 3), dtype=np.float32)
    ins = inside(vol, iso)
    v64 = vol.astype(np.float64)
    # the crossed edges, their vertex order and t, as marching_cubes finds them
    flags = np.zeros(dims + (3,), dtype=bool)
    flags[:-1, :, :, 0] = ins[:-1] != ins[1:]
    flags[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    flags[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    slots = np.nonzero(flags.reshape(-1))[0]
    pt, axis = slots // 3, slots % 3
    lower = np.stack(np.unravel_index(pt, dims), -1)
    upper = lower + np.eye(3, dtype=np.int64)[axis]
    sa = v64[tuple(lower.T)]
    sb = v64[tuple(upper.T)]
    with np.errstate(invalid="ignore", divide="ignore"):
        t = (float(iso) - sa) / (sb - sa)
    t = np.where(np.isfinite(sa) & np.isfinite(sb), t, 0.5)
    g = grid_gradient(vol)
    ga, gb = g[tuple(lower.T)], g[tuple(upper.T)]
    lo, hi, n = np.asarray(lo, np.float64), np.asarray(hi, np.float64), np.asarray(dims)
    h = (hi - lo) / (n - 1)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        G = ((1.0 - t)[:, None] * ga + t[:, None] * gb) / h
        length = np.sqrt((G[:, 0] * G[:, 0] + G[:, 1] * G[:, 1]) + G[:, 2] * G[:, 2])
        ok = (length > 0) & np.isfinite(length)
        normals = -G / np.where(ok, length, 1.0)[:, None]
    rows = np.nonzero(~ok)[0]
    normals[rows] = 0.0
    normals[rows, axis[rows]] = np.where(ins[tuple(lower[rows].T)] != (h[axis[rows]] < 0), 1.0, -1.0)
    v = lower.astype(np.float64)
    v[np.arange(len(axis)), axis] += t
    xyz = np.where(v == n - 1, hi, v * h + lo).astype(np.float32)
    return normals, xyz, (-normals).astype(np.float32)
