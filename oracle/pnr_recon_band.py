"""
ORACLE -- numpy restatement of narrow-band mesh extraction (the pnr_band_* entry points of csrc/pnr_recon.cu,
util/recon.py marching_cubes(..., block=b)), the reference the kernels are compared against bit for bit.

  blocks          block i of an axis covers the cells [i b, min((i + 1) b, n - 1)); nb = ceil((n - 1) / b) per axis
  lattice_index   the grid indices min(j b, n - 1), j = 0 .. nb, of one axis; the coarse lattice is their product in
                  ij order, so block i's corners are lattice points i and i + 1 and every lattice point is a grid point
  plan            coarse sigma [nb0 + 1][nb1 + 1][nb2 + 1] -> (seeded, active) block flags: seeded when the 8 corners
                  are not all in the same state (inside: finite and sigma > iso), active when it or one of its 26
                  neighbours is seeded
  refine_index    the refinement set, as flat grid indices in ij order: the grid points of the active blocks' closed
                  cells ([i b, min((i + 1) b, n - 1)] per axis), with the apron widened by one point on each side (the
                  neighbours the vertex normals read)
  marching_cubes  the mesh: pnr_recon.marching_cubes of the dense volume with every cell outside the active blocks
                  treated as empty (configuration 0) and the vertices no remaining triangle uses dropped, in the dense
                  order (vertex ids by (grid point, axis), triangles by cell, then table order)
  kept_vertices   the dense vertex ids of those vertices
  vertex_attrs    pnr_recon_attrs.vertex_attrs of the kept vertices
"""
import importlib.util
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name, file):
    spec = importlib.util.spec_from_file_location(name, os.path.join(_HERE, file))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


recon = _load("pnr_recon_oracle_for_band", "pnr_recon.py")
attrs = _load("pnr_recon_attrs_oracle_for_band", "pnr_recon_attrs.py")


def n_blocks(n, b):
    return (n - 1 + b - 1) // b


def lattice_index(n, b):
    return np.minimum(np.arange(n_blocks(n, b) + 1, dtype=np.int64) * b, n - 1)


def lattice_flat(reso, b):
    """flat grid indices of the coarse lattice, in its ij order"""
    ix, iy, iz = np.meshgrid(*[lattice_index(n, b) for n in reso], indexing="ij")
    return np.ravel_multi_index((ix.reshape(-1), iy.reshape(-1), iz.reshape(-1)), tuple(reso))


def lattice_points(lo, hi, reso, b):
    """(xyz, viewdirs) float32 of the lattice: pnr_recon.grid_points' values at the lattice's grid indices"""
    xyz = recon.grid_points(lo, hi, reso)[lattice_flat(reso, b)]
    return xyz, recon.fake_viewdirs(xyz)


def plan(coarse, reso, b, iso):
    nb = [n_blocks(n, b) for n in reso]
    if min(nb) == 0:
        z = np.zeros(nb, dtype=bool)
        return z, z
    ins = recon.inside(np.asarray(coarse, np.float32).reshape([m + 1 for m in nb]), iso)
    corners = [ins[dx:dx + nb[0], dy:dy + nb[1], dz:dz + nb[2]] for dz in (0, 1) for dy in (0, 1) for dx in (0, 1)]
    seeded = np.any([c != corners[0] for c in corners[1:]], axis=0)
    pad = np.pad(seeded, 1)
    active = np.zeros_like(seeded)
    for dx in range(3):
        for dy in range(3):
            for dz in range(3):
                active |= pad[dx:dx + nb[0], dy:dy + nb[1], dz:dz + nb[2]]
    return seeded, active


def plan_of_volume(vol, iso, b):
    """plan() of the coarse lattice sampled from a dense volume"""
    vol = np.asarray(vol, np.float32)
    return plan(vol.reshape(-1)[lattice_flat(vol.shape, b)], vol.shape, b, iso)


def cover(n, b, nb, apron):
    """bool [n][nb]: grid index x of an axis lies in block C's closed cells (widened by the apron)"""
    d = 1 if apron else 0
    x = np.arange(n)[:, None]
    C = np.arange(nb)[None, :]
    return (C * b - d <= x) & (x <= np.minimum((C + 1) * b, n - 1) + d)


def refine_index(active, reso, b, apron=False):
    """flat grid indices of the refinement set, ascending (ij order)"""
    if active.size == 0:
        return np.zeros(0, dtype=np.int64)
    cx, cy, cz = (cover(n, b, m, apron).astype(np.int64) for n, m in zip(reso, active.shape))
    t = np.tensordot(cx, active.astype(np.int64), (1, 0))          # [nx][nby][nbz]
    t = np.tensordot(t, cy, (1, 1)).transpose(0, 2, 1) > 0            # [nx][ny][nbz]
    t = np.tensordot(t.astype(np.int64), cz, (2, 1)) > 0              # [nx][ny][nz]
    return np.flatnonzero(t)


def _cells(vol, iso):
    """cube configuration per cell of the dense volume, as pnr_recon.marching_cubes finds it"""
    ins = recon.inside(vol, iso)
    dims = vol.shape
    cube = np.zeros(tuple(d - 1 for d in dims), dtype=np.int64)
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        cube |= ins[dx:dims[0] - 1 + dx, dy:dims[1] - 1 + dy, dz:dims[2] - 1 + dz].astype(np.int64) << k
    return cube


def active_cells(active, dims, b):
    """bool [nx - 1][ny - 1][nz - 1]: the cell lies in an active block"""
    return active[np.ix_(*[np.arange(d - 1) // b for d in dims])]


def _kept(vol, iso, b):
    """(dense verts, dense tris, tris kept, kept vertex ids, complete coverage)"""
    vol = np.asarray(vol, np.float32)
    dims = vol.shape
    verts, tris = recon.marching_cubes(vol, iso)
    if min(dims) < 2:
        return verts, tris, tris, np.zeros(0, np.int64), True
    _, active = plan_of_volume(vol, iso, b)
    cube = _cells(vol, iso).reshape(-1)
    cnt = recon.TRI_COUNT[cube]
    on = active_cells(active, dims, b).reshape(-1)
    keep_tri = np.repeat(on, cnt)                      # dense triangles run over cells in linear order
    kt = tris[keep_tri]
    used = np.unique(kt)
    complete = bool(on[cnt > 0].all())
    return verts, tris, kt, used, complete


def marching_cubes(vol, iso, b):
    """-> (vertices float64 [N][3] in index space, triangles int64 [M][3], complete coverage)"""
    verts, _, kt, used, complete = _kept(vol, iso, b)
    return verts[used], np.searchsorted(used, kt).astype(np.int64).reshape(-1, 3), complete


def kept_vertices(vol, iso, b):
    """ids, in the dense mesh, of marching_cubes(vol, iso, b)'s vertices"""
    return _kept(vol, iso, b)[3]


def vertex_attrs(vol, iso, lo, hi, b):
    """(normals, xyz, viewdirs) of marching_cubes(vol, iso, b)'s vertices"""
    _, _, _, used, _ = _kept(vol, iso, b)
    n, xyz, vd = attrs.vertex_attrs(vol, iso, lo, hi)
    return n[used], xyz[used], vd[used]
