"""
ORACLE -- numpy restatement of mesh extraction (csrc/pnr_recon.cu, util/recon.py), the reference the kernels are
compared against bit for bit.

  grid_points     util.gen_grid(*zip(c1, c2, reso), ij_indexing=True) (src/util/util.py:93-110): float32 points,
                  x slowest; each axis is np.linspace(lo, hi, n, dtype=float32), i.e. computed in float64 and rounded
  fake_viewdirs   -grid / torch.norm(grid, dim=-1) of src/util/recon.py:54 in float32 (NaN at the origin)
  marching_cubes  vol [nx][ny][nz] -> (vertices float64 [N][3] in index space, triangles int64 [M][3]):
                  a corner is inside when it is finite and sigma > iso; one vertex per crossed grid edge, numbered in
                  (grid point, axis) order; at t = (iso - s_a) / (s_b - s_a) from the edge's lower corner a in
                  float64 (0.5 when the outside corner is NaN or infinite); triangles per cell from oracle/make_mc_tables.py's tables,
                  cells in linear order, each cell's in table order.
"""
import importlib.util
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("pnr_make_mc_tables", os.path.join(_HERE, "make_mc_tables.py"))
mc_tables = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mc_tables)

_T = mc_tables.tables()
EDGE_CORNER = np.array(_T["edge_corner"], dtype=np.int64)
EDGE_AXIS = np.array(_T["edge_axis"], dtype=np.int64)
TRI_COUNT = np.array(_T["tri_count"], dtype=np.int64)
TRIS = np.array(_T["tris"], dtype=np.int64).reshape(256, -1, 3)


def grid_points(lo, hi, reso):
    axes = [np.linspace(a, b, n, dtype=np.float32) for a, b, n in zip(lo, hi, reso)]
    return np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)


def fake_viewdirs(grid):
    """float32; torch's CPU norm of gen_grid's transposed (non-contiguous) grid sums (x*x + y*y) + z*z."""
    x, y, z = grid[:, 0], grid[:, 1], grid[:, 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        return -grid / np.sqrt((x * x + y * y) + z * z)[:, None]


def inside(vol, iso):
    v = np.asarray(vol, dtype=np.float32).astype(np.float64)
    return np.isfinite(v) & (v > float(iso))


def marching_cubes(vol, iso):
    vol = np.asarray(vol, dtype=np.float32)
    dims = vol.shape
    if min(dims) < 2:
        return np.zeros((0, 3)), np.zeros((0, 3), dtype=np.int64)
    ins = inside(vol, iso)
    v64 = vol.astype(np.float64)
    # edge slots (point, axis), point-major
    flags = np.zeros(dims + (3,), dtype=bool)
    flags[:-1, :, :, 0] = ins[:-1] != ins[1:]
    flags[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    flags[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    flat = flags.reshape(-1)
    vid = np.cumsum(flat) - flat                       # exclusive scan: vertex id of each crossed edge
    slots = np.nonzero(flat)[0]
    pt, axis = slots // 3, slots % 3
    lower = np.stack(np.unravel_index(pt, dims), -1)
    upper = lower + np.eye(3, dtype=np.int64)[axis]
    sa = v64[tuple(lower.T)]
    sb = v64[tuple(upper.T)]
    with np.errstate(invalid="ignore", divide="ignore"):
        t = (float(iso) - sa) / (sb - sa)
    t = np.where(np.isfinite(sa) & np.isfinite(sb), t, 0.5)
    verts = lower.astype(np.float64)
    verts[np.arange(len(axis)), axis] += t
    # cells, linear order of their lower corner
    cube = np.zeros(tuple(d - 1 for d in dims), dtype=np.int64)
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        cube |= ins[dx:dims[0] - 1 + dx, dy:dims[1] - 1 + dy, dz:dims[2] - 1 + dz].astype(np.int64) << k
    cells = np.nonzero(TRI_COUNT[cube.reshape(-1)])[0]
    cidx = np.stack(np.unravel_index(cells, cube.shape), -1)            # (nc, 3) lower corners
    cfg = cube.reshape(-1)[cells]
    tri_e = TRIS[cfg]                                                  # (nc, max_tris, 3) edge numbers
    keep = np.arange(TRIS.shape[1])[None, :] < TRI_COUNT[cfg][:, None]
    corner = EDGE_CORNER[tri_e]
    off = np.stack([corner & 1, (corner >> 1) & 1, (corner >> 2) & 1], -1)  # (nc, max_tris, 3, 3)
    p = cidx[:, None, None, :] + off                                   # padding rows (-1) index real edges; dropped
    slot = np.ravel_multi_index(tuple(np.moveaxis(p, -1, 0)), dims) * 3 + EDGE_AXIS[tri_e]
    tris = vid[slot][keep]
    return verts, tris.reshape(-1, 3).astype(np.int64)


# ---- mesh checks used by the tests ---------------------------------------------------------------------------------
def directed_edges(tris):
    return np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])


def is_closed_oriented(tris):
    """Every directed edge once and every undirected edge exactly twice (a closed, consistently oriented surface)."""
    d = directed_edges(tris)
    if len(np.unique(d, axis=0)) != len(d):
        return False
    u = np.sort(d, axis=1)
    _, counts = np.unique(u, axis=0, return_counts=True)
    return bool((counts == 2).all())


def signed_volume(verts, tris):
    a, b, c = verts[tris[:, 0]], verts[tris[:, 1]], verts[tris[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def euler_characteristic(verts, tris):
    used = np.unique(tris)
    e = np.unique(np.sort(directed_edges(tris), axis=1), axis=0)
    return len(used) - len(e) + len(tris)


def components(tris):
    parent = np.arange(int(tris.max()) + 1 if len(tris) else 0)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in directed_edges(tris):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
    return len({find(v) for v in np.unique(tris)})
