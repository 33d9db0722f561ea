"""
ORACLE -- numpy / scipy restatement of the connected components of a triangle mesh (csrc/pnr_recon.cu
pnr_mesh_components / pnr_mesh_compact_*, util/recon.py keep_components), the reference the kernels and the Python
policy are compared against bit for bit.

  labels           two vertices are connected when some triangle uses both; label[v] = the smallest vertex id of v's
                   component (scipy.sparse.csgraph.connected_components on the graph of the edges (a, b), (a, c))
  tri_counts       tri_count[r] = the triangles whose vertices have label r, 0 where r is not a label
  keep_components  components ranked by triangle count, descending, ties to the smaller label; the first `largest`
                   (all with largest=None) of those with at least min_triangles triangles are kept; the kept vertices
                   and triangles in their original order, triangles through the new vertex ids, every attribute
                   compacted by the same rows
"""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components


def labels(tris, n_verts):
    tris = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
    if len(tris) and (tris.min() < 0 or tris.max() >= n_verts):
        raise ValueError("vertex id outside [0, n_verts)")
    rows = np.concatenate([tris[:, 0], tris[:, 0]])
    cols = np.concatenate([tris[:, 1], tris[:, 2]])
    graph = sp.coo_matrix((np.ones(len(rows), dtype=np.int8), (rows, cols)), shape=(n_verts, n_verts)).tocsr()
    n_comp, comp = connected_components(graph, directed=False)
    smallest = np.full(n_comp, n_verts, dtype=np.int64)
    np.minimum.at(smallest, comp, np.arange(n_verts, dtype=np.int64))
    return smallest[comp]


def tri_counts(tris, label):
    tris = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
    return np.bincount(label[tris[:, 0]], minlength=len(label)).astype(np.int64)


def kept_roots(tri_count, largest=1, min_triangles=1):
    """The labels of the kept components, in rank order."""
    roots = np.nonzero(tri_count)[0]
    # rank: more triangles first, then the smaller root (lexsort's last key is the primary one)
    ranked = roots[np.lexsort((roots, -tri_count[roots]))]
    ranked = ranked[tri_count[ranked] >= min_triangles]
    return ranked if largest is None else ranked[:largest]


def keep_components(vertices, triangles, *vertex_attrs, largest=1, min_triangles=1):
    vertices, triangles = np.asarray(vertices), np.asarray(triangles)
    n = len(vertices)
    label = labels(triangles, n)
    keep_root = np.zeros(n, dtype=bool)
    keep_root[kept_roots(tri_counts(triangles, label), largest, min_triangles)] = True
    keep_v = keep_root[label]
    new_id = np.cumsum(keep_v) - keep_v
    t = triangles.reshape(-1, 3)
    keep_t = keep_v[t[:, 0]] if len(t) else np.zeros(0, dtype=bool)
    tris = new_id[t[keep_t]].astype(triangles.dtype).reshape(-1, 3)
    return (vertices[keep_v], tris) + tuple(np.asarray(a)[keep_v] for a in vertex_attrs)
