"""
ORACLE -- numpy restatement of mesh decimation (csrc/pnr_mesh.cu pnr_decimate_*, util/recon.py decimate), the
reference the kernels and the Python round loop are compared against bit for bit.  The rule is include/pnr.h's:
rounds of independent half-edge collapses c -> d (d stays where it is) with Garland-Heckbert quadrics.

  quadrics   per triangle (p0, p1, p2): e1 = p1 - p0, e2 = p2 - p0, n = e1 x e2 (n_x = e1y e2z - e1z e2y, ...),
             len2 = (n_x n_x + n_y n_y) + n_z n_z; when len2 > 0: s = sqrt(len2), a = 0.5 s, u = n / s,
             d = -((u_x p0x + u_y p0y) + u_z p0z), Q_t = a * (u_x u_x, u_x u_y, u_x u_z, u_y u_y, u_y u_z, u_z u_z,
             u_x d, u_y d, u_z d, d d) (each product rounded, then scaled by a); else 0.  A vertex's quadric is
             ((0 + Q_t1) + Q_t2) + ... over its corners in ascending triangle id.  A vertex with more than INC_CAP
             corners at the start is frozen for the whole call: never removed, never a d, so its quadric (0) is never
             read, even once collapses around it have taken corners away.
  error      Q = Q_c + Q_d at p = p_d: r_i = ((A_i0 x + A_i1 y) + A_i2 z) + b_i, cost = (((r0 x + r1 y) + r2 z) +
             ((b0 x + b1 y) + b2 z)) + c, tr = (A00 + A11) + A22, err = sqrt((cost if cost > 0 else 0) / tr) when
             tr > 0, else 0.
  classify   corners of v: its incident triangles rotated to (v, x, y) at v's first occurrence; neighbours: the other
             ids; valence: their number (VAL_INF above INC_CAP corners).  fan / removable as in include/pnr.h, and
             never for a frozen vertex.
  select     the collapses of one round, ascending c, as in include/pnr.h; apply: Q_d += Q_c, c -> d, the two
             triangles of each edge cd dropped, the others kept in order.
  decimate   rounds until the target (triangles <= target) or a round that selects nothing; a round selecting more
             than ceil((M - target) / 2) keeps that many of the smallest keys; then the used vertices in order.
"""
import numpy as np

VALENCE_CAP = 32
INC_CAP = 64
VAL_INF = 1 << 30
NONE = np.iinfo(np.int64).max
CHUNK = 1 << 15


def tri_normal(p0, p1, p2):
    e1, e2 = p1 - p0, p2 - p0
    return np.stack([e1[..., 1] * e2[..., 2] - e1[..., 2] * e2[..., 1],
                     e1[..., 2] * e2[..., 0] - e1[..., 0] * e2[..., 2],
                     e1[..., 0] * e2[..., 1] - e1[..., 1] * e2[..., 0]], axis=-1)


def tri_quadrics(xyz, tris):
    p0 = xyz[tris[:, 0]]
    n = tri_normal(p0, xyz[tris[:, 1]], xyz[tris[:, 2]])
    len2 = (n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]
    ok = len2 > 0
    with np.errstate(all="ignore"):
        s = np.sqrt(len2)
        a = 0.5 * s
        u = n / s[:, None]
        ux, uy, uz = u[:, 0], u[:, 1], u[:, 2]
        d = -((ux * p0[:, 0] + uy * p0[:, 1]) + uz * p0[:, 2])
        e = np.stack([ux * ux, ux * uy, ux * uz, uy * uy, uy * uz, uz * uz, ux * d, uy * d, uz * d, d * d], axis=1)
        q = a[:, None] * e
    q[~ok] = 0.0
    return q


def incidence(tris, n_verts):
    """deg [N] (corners per vertex), inc [N, D] triangle ids ascending (-1 padded; empty for deg > INC_CAP)."""
    v = tris.reshape(-1)
    t = np.arange(len(v), dtype=np.int64) // 3
    deg = np.bincount(v, minlength=n_verts).astype(np.int64)
    keep = deg[v] <= INC_CAP
    v, t = v[keep], t[keep]
    order = np.lexsort((t, v))
    v, t = v[order], t[order]
    start = np.cumsum(np.bincount(v, minlength=n_verts)) - np.bincount(v, minlength=n_verts)
    rank = np.arange(len(v)) - start[v]
    D = int(rank.max()) + 1 if len(rank) else 1
    inc = np.full((n_verts, D), -1, dtype=np.int64)
    inc[v, rank] = t
    return deg, inc


def frozen(tris, n_verts):
    """pnr_decimate_init's frozen flags: more than INC_CAP corners."""
    tris = np.asarray(tris, np.int64).reshape(-1)
    return np.bincount(tris, minlength=n_verts) > INC_CAP


def quadrics(xyz, tris):
    xyz, tris = np.asarray(xyz, np.float64), np.asarray(tris, np.int64).reshape(-1, 3)
    n = len(xyz)
    q = np.zeros((n, 10))
    if len(tris) == 0:
        return q
    qt = tri_quadrics(xyz, tris)
    _, inc = incidence(tris, n)
    for k in range(inc.shape[1]):
        rows = np.nonzero(inc[:, k] >= 0)[0]
        q[rows] = q[rows] + qt[inc[rows, k]]
    return q


def collapse_error(qc, qd, p):
    q = qc + qd
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    r0 = ((q[..., 0] * x + q[..., 1] * y) + q[..., 2] * z) + q[..., 6]
    r1 = ((q[..., 1] * x + q[..., 3] * y) + q[..., 4] * z) + q[..., 7]
    r2 = ((q[..., 2] * x + q[..., 4] * y) + q[..., 5] * z) + q[..., 8]
    cost = (((r0 * x + r1 * y) + r2 * z) + ((q[..., 6] * x + q[..., 7] * y) + q[..., 8] * z)) + q[..., 9]
    tr = (q[..., 0] + q[..., 3]) + q[..., 5]
    with np.errstate(all="ignore"):
        e = np.sqrt(np.where(cost > 0, cost, 0.0) / tr)
    return np.where(tr > 0, e, 0.0)


class Mesh:
    """The per-round view of a mesh: corners, neighbours, valence and the fan / removable flags."""

    def __init__(self, tris, n_verts, frozen):
        self.tris, self.n = tris, n_verts
        deg, inc = incidence(tris, n_verts)
        self.inc, self.cnt = inc, (inc >= 0).sum(1)
        valid = inc >= 0
        v = np.arange(n_verts)[:, None]
        abc = tris[np.where(valid, inc, 0)]                                    # [N, D, 3]
        a, b, c = abc[..., 0], abc[..., 1], abc[..., 2]
        self.X = np.where(a == v, b, np.where(b == v, c, a))
        self.Y = np.where(a == v, c, np.where(b == v, a, b))
        self.X[~valid], self.Y[~valid] = -1, -1
        rep = ((a == b) | (b == c) | (a == c)) & valid
        nb = np.concatenate([self.X, self.Y], axis=1)
        nb = np.where((nb < 0) | (nb == v), NONE, nb)
        nb.sort(axis=1)
        dup = np.zeros_like(nb, dtype=bool)
        dup[:, 1:] = nb[:, 1:] == nb[:, :-1]
        nb[dup] = NONE
        nb.sort(axis=1)
        self.U = nb                                                            # neighbours ascending, NONE padded
        val = (nb != NONE).sum(1)
        ok = np.ones(n_verts, dtype=bool)
        start = np.full(n_verts, -1, dtype=np.int64)
        for lo in range(0, n_verts, CHUNK):
            sl = slice(lo, lo + CHUNK)
            U, X, Y = nb[sl], self.X[sl], self.Y[sl]
            outs = (U[:, :, None] == X[:, None, :]).sum(2)
            ins = (U[:, :, None] == Y[:, None, :]).sum(2)
            real = U != NONE
            ok[sl] = ((outs <= 1) & (ins <= 1) | ~real).all(1)
            z = real & (ins == 0)
            start[sl] = np.where(z.any(1), U[np.arange(len(U)), z.argmax(1)], U[:, 0])
        closed = self.cnt == val
        start = np.where(closed, nb[:, 0], start)
        # walk the link x -> y from start; one fan when the walk visits every neighbour
        visited = np.ones(n_verts, dtype=np.int64)
        cur, live = start.copy(), ok & ~rep.any(1) & (self.cnt >= 1)
        for _ in range(inc.shape[1]):
            if not live.any():
                break
            hit = (self.X == cur[:, None]) & live[:, None]
            nxt = np.where(hit.any(1), self.Y[np.arange(n_verts), hit.argmax(1)], -1)
            live &= (nxt >= 0) & (nxt != start)
            visited += live
            cur = np.where(live, nxt, cur)
        fan = ok & ~rep.any(1) & (self.cnt >= 1) & (visited == val)
        removable = fan & closed & (val >= 3) & (val <= VALENCE_CAP)
        over = deg > INC_CAP
        self.val = np.where(over, VAL_INF, val).astype(np.int64)
        self.fan, self.removable = fan & ~over & ~frozen, removable & ~over & ~frozen


def key_less(e1, l1, h1, e2, l2, h2):
    return (e1 < e2) | ((e1 == e2) & ((l1 < l2) | ((l1 == l2) & (h1 < h2))))


def directed_collapses(xyz, tris, q, m, bound):
    """Every valid c -> d with its error, and whether some collapse was valid but for the bound."""
    cs, js = np.nonzero(m.removable[:, None] & (m.X >= 0))
    d = m.X[cs, js]
    keep = m.fan[d] & (m.val[cs] + m.val[d] - 4 <= VALENCE_CAP)
    cs, js, d = cs[keep], js[keep], d[keep]
    o1 = m.Y[cs, js]
    at = m.Y[cs] == d[:, None]
    o2 = m.X[cs, at.argmax(1)]
    keep = (m.val[o1] >= 4) & (m.val[o2] >= 4)
    cs, d = cs[keep], d[keep]
    ok = np.zeros(len(cs), dtype=bool)
    for lo in range(0, len(cs), CHUNK):
        c_, d_ = cs[lo:lo + CHUNK], d[lo:lo + CHUNK]
        Xc = m.X[c_]
        shared = (Xc[:, :, None] == m.U[d_][:, None, :]).any(2) & (Xc >= 0) & (Xc != d_[:, None])
        link = shared.sum(1) == 2
        T = tris[np.where(m.inc[c_] >= 0, m.inc[c_], 0)]                      # [P, D, 3]
        live = (m.inc[c_] >= 0) & ~(T == d_[:, None, None]).any(2)
        p = xyz[T]
        qv = xyz[np.where(T == c_[:, None, None], d_[:, None, None], T)]
        n0 = tri_normal(p[..., 0, :], p[..., 1, :], p[..., 2, :])
        n1 = tri_normal(qv[..., 0, :], qv[..., 1, :], qv[..., 2, :])
        dot = (n0[..., 0] * n1[..., 0] + n0[..., 1] * n1[..., 1]) + n0[..., 2] * n1[..., 2]
        flip = live & (n0 != 0).any(-1) & (dot <= 0)
        ok[lo:lo + CHUNK] = link & ~flip.any(1)
    cs, d = cs[ok], d[ok]
    err = collapse_error(q[cs], q[d], xyz[d])
    within = err <= bound
    return cs[within], d[within], err[within], bool((~within).any())


def select(xyz, tris, q, frozen, max_error=None):
    """pnr_decimate_select: (c, d, err) of the selected collapses in ascending c, and whether the bound held one back."""
    xyz, tris = np.asarray(xyz, np.float64), np.asarray(tris, np.int64).reshape(-1, 3)
    n = len(xyz)
    empty = np.zeros(0, np.int64)
    if n == 0 or len(tris) == 0:
        return empty, empty, np.zeros(0), False
    bound = np.inf if max_error is None else float(max_error)
    m = Mesh(tris, n, frozen)
    c, d, err, over = directed_collapses(xyz, tris, q, m, bound)
    lo, hi = np.minimum(c, d), np.maximum(c, d)
    # each edge: the cheaper valid direction, on a tie the larger id removed
    o = np.lexsort((-c, err, hi, lo))
    c, d, err, lo, hi = c[o], d[o], err[o], lo[o], hi[o]
    first = np.ones(len(c), dtype=bool)
    first[1:] = (lo[1:] != lo[:-1]) | (hi[1:] != hi[:-1])
    c, d, err, lo, hi = c[first], d[first], err[first], lo[first], hi[first]
    # best(v) over the edges at v
    best_err, best_lo, best_hi = np.full(n, np.inf), np.full(n, NONE), np.full(n, NONE)
    best_c = np.full(n, -1, dtype=np.int64)
    ends = np.concatenate([lo, hi])
    e2, l2, h2, c2 = (np.concatenate([a, a]) for a in (err, lo, hi, c))
    o = np.lexsort((h2, l2, e2, ends))
    ends, e2, l2, h2, c2 = ends[o], e2[o], l2[o], h2[o], c2[o]
    f = np.ones(len(ends), dtype=bool)
    f[1:] = ends[1:] != ends[:-1]
    best_err[ends[f]], best_lo[ends[f]], best_hi[ends[f]], best_c[ends[f]] = e2[f], l2[f], h2[f], c2[f]
    # selected: best of both ends and below best(w) of every other neighbour of either end
    cand = np.nonzero(best_c == np.arange(n))[0]
    e, l, h = best_err[cand], best_lo[cand], best_hi[cand]
    dd = np.where(l == cand, h, l)
    s = (best_err[dd] == e) & (best_lo[dd] == l) & (best_hi[dd] == h)
    for a, skip in ((cand, dd), (dd, cand)):
        W = m.U[a]
        real = (W != NONE) & (W != skip[:, None])
        Wi = np.where(real, W, 0)
        beat = key_less(e[:, None], l[:, None], h[:, None], best_err[Wi], best_lo[Wi], best_hi[Wi])
        s &= (beat | ~real).all(1)
    return cand[s], dd[s], e[s], over


def apply(tris, q, c, d):
    """pnr_decimate_apply: (the new triangles, the merged quadrics)."""
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    q = q.copy()
    q[d] = q[d] + q[c]
    to = np.arange(len(q), dtype=np.int64)
    to[c] = d
    r = to[tris]
    moved = (r != tris).any(1)
    rep = (r[:, 0] == r[:, 1]) | (r[:, 1] == r[:, 2]) | (r[:, 0] == r[:, 2])
    return r[~(moved & rep)], q


def trim(c, d, err, keep):
    """The `keep` collapses of smallest key (err, min id, max id), back in ascending c."""
    o = np.lexsort((np.maximum(c, d), np.minimum(c, d), err))[:keep]
    o.sort()
    return c[o], d[o], err[o]


def rounds(xyz, tris, target_triangles=None, max_error=None):
    """The round loop -> (triangles, quadrics, per-round collapse counts, the error of every collapse made, reason)."""
    xyz, tris = np.asarray(xyz, np.float64), np.asarray(tris, np.int64).reshape(-1, 3)
    q, fz = quadrics(xyz, tris), frozen(tris, len(xyz))
    counts, errs = [], []
    while True:
        M = len(tris)
        if target_triangles is not None and M <= target_triangles:
            reason = "target reached"
            break
        c, d, err, over = select(xyz, tris, q, fz, max_error)
        if len(c) == 0:
            reason = "error bound" if over else "no valid collapse left"
            break
        if target_triangles is not None and len(c) > -(-(M - target_triangles) // 2):
            c, d, err = trim(c, d, err, -(-(M - target_triangles) // 2))
        tris, q = apply(tris, q, c, d)
        counts.append(len(c))
        errs.append(err)
    return tris, q, counts, np.concatenate(errs) if errs else np.zeros(0), reason


def decimate(vertices, triangles, *vertex_attrs, target_triangles=None, max_error=None):
    vertices, triangles = np.asarray(vertices), np.asarray(triangles)
    tris, _, _, _, _ = rounds(vertices.astype(np.float64), triangles, target_triangles, max_error)
    used = np.zeros(len(vertices), dtype=bool)
    used[tris.reshape(-1)] = True
    new_id = np.cumsum(used) - used
    out_tris = new_id[tris].astype(triangles.dtype).reshape(-1, 3)
    return (vertices[used], out_tris) + tuple(np.asarray(a)[used] for a in vertex_attrs)
