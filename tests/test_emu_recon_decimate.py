"""pnr_decimate_init / _select / _apply (csrc/pnr_mesh.cu) on the host emulator (built by tests/mesh_emu.py), each
bit for bit against the oracle (oracle/pnr_recon_decimate.py) round after round: random closed and open meshes, ties
(a flat patch where every error is 0), a tetrahedron, a vertex at the valence cap, degenerate triangles, and the
error codes."""
import ctypes as C

import numpy as np
import pytest
import torch

import mesh_emu
from decimate_util import bipyramid, bits_equal, dec, flat_patch, sphere_mesh
from recon_util import padded_random, recon

PNR_ERR_INVALID, PNR_ERR_WORKSPACE = -1, -2


def _p(t):
    return C.c_void_p(t.data_ptr())


def _pad(a, dtype):
    """a CPU tensor of a with one extra row, so that no pointer is NULL"""
    a = np.asarray(a, dtype=dtype)
    return torch.from_numpy(np.concatenate([a, np.zeros((1,) + a.shape[1:], dtype)]))


def run_rounds(v, t, max_error=None, target=None, max_rounds=60):
    """Every entry point on the emulator against the oracle, round after round; returns the rounds run."""
    L = mesh_emu.lib()
    v, t = np.asarray(v, np.float64), np.asarray(t, np.int64).reshape(-1, 3)
    n, m = len(v), len(t)
    ws = torch.empty(int(L.pnr_decimate_workspace_bytes(n, m)), dtype=torch.uint8)
    xyz, T = _pad(v, np.float64), _pad(t, np.int64)
    Q = torch.full((n + 1, 10), -7.0, dtype=torch.float64)
    F = torch.full((n + 1,), 7, dtype=torch.uint8)
    rc = L.pnr_decimate_init(_p(xyz), n, _p(T), m, _p(Q), _p(F), _p(ws), ws.numel(), None)
    assert rc == 0, L.pnr_last_error()
    q, fz = dec.quadrics(v, t), dec.frozen(t, n)
    assert bits_equal(Q.numpy()[:n], q) and (Q.numpy()[n] == -7).all()
    assert bits_equal(F.numpy()[:n], fz.astype(np.uint8)) and F[n] == 7
    tris = t
    bound = float("inf") if max_error is None else max_error
    for r in range(max_rounds):
        k0 = n // 2 + 1
        cs, ds = torch.full((k0,), -7, dtype=torch.int64), torch.full((k0,), -7, dtype=torch.int64)
        es = torch.full((k0,), -7.0, dtype=torch.float64)
        counts = (C.c_int64 * 2)()
        T = _pad(tris, np.int64)
        rc = L.pnr_decimate_select(_p(xyz), n, _p(T), len(tris), _p(Q), _p(F), bound, _p(cs), _p(ds), _p(es),
                                   C.cast(counts, C.POINTER(C.c_int64)), _p(ws), ws.numel(), None)
        assert rc == 0, L.pnr_last_error()
        k = counts[0]
        c, d, err, over = dec.select(v, tris, q, fz, max_error)
        assert bits_equal(cs.numpy()[:k], c) and bits_equal(ds.numpy()[:k], d) and bits_equal(es.numpy()[:k], err)
        assert bool(counts[1]) == over and cs[k] == -7
        if k == 0 or (target is not None and len(tris) <= target):
            return r
        if target is not None:                                      # apply a trimmed subset, as decimate does
            c, d, err = dec.trim(c, d, err, max(1, -(-(len(tris) - target) // 2)))
        out = torch.full((len(tris) + 1, 3), -7, dtype=torch.int64)
        count = C.c_int64(-7)
        ct, dt = _pad(c, np.int64), _pad(d, np.int64)
        rc = L.pnr_decimate_apply(_p(T), len(tris), n, _p(ct), _p(dt), len(c), _p(Q), _p(out), C.byref(count), _p(ws),
                                  ws.numel(), None)
        assert rc == 0, L.pnr_last_error()
        tris, q = dec.apply(tris, q, c, d)
        assert count.value == len(tris) == len(T) - 1 - 2 * len(c)
        assert bits_equal(out.numpy()[:count.value], tris) and (out.numpy()[count.value] == -7).all()
        assert bits_equal(Q.numpy()[:n], q)
    return max_rounds


@pytest.mark.parametrize("seed", [1, 2])
def test_random_closed_and_open_meshes(seed):
    v, t = recon.marching_cubes(padded_random((10, 9, 8), seed), 0.0)
    v = v + np.random.default_rng(seed).uniform(-0.2, 0.2, v.shape)       # break the grid's symmetries
    assert run_rounds(v, t, max_rounds=8) >= 3
    g = np.random.default_rng(seed)
    t_open = t[g.random(len(t)) > 0.1]                                      # holes: boundaries and lone vertices
    assert run_rounds(v, t_open, max_rounds=8) >= 3
    assert run_rounds(v, t, max_error=0.05, max_rounds=8) >= 1
    run_rounds(v, t, target=len(t) - 7, max_rounds=3)                      # a trimmed round


def test_ties_on_a_flat_patch():
    v, t = flat_patch(9)
    assert run_rounds(v, t, max_error=0.0, max_rounds=10) >= 3


def test_sphere_down_to_few_triangles():
    v, t = sphere_mesh(12, 4.0)
    assert run_rounds(v, t, max_rounds=200) < 200                           # stops: no valid collapse left


def test_tetrahedron():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float64)
    t = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    assert run_rounds(v, t) == 0


@pytest.mark.parametrize("k", [31, 32, 33])
def test_valence_at_the_cap(k):
    v, t = bipyramid(k)
    m = dec.Mesh(t, len(v), dec.frozen(t, len(v)))
    assert m.val[k] == k and bool(m.removable[k]) == (k <= 32)
    run_rounds(v, t, max_rounds=4)


@pytest.mark.parametrize("k", [64, 65, 100])
def test_vertices_over_64_corners_are_frozen(k):
    """Apexes of 64 corners are examined; of 65 or 100 frozen, with a quadric of 0, while the ring collapses around
    them and takes their corners away below 64."""
    v, t = bipyramid(k)
    assert list(dec.frozen(t, len(v))[k:]) == [k > 64] * 2
    assert run_rounds(v, t, max_error=0.05, max_rounds=12) >= 2
    assert run_rounds(v, t, max_rounds=12) >= 2


def test_degenerate_triangles():
    v, t = sphere_mesh(10, 3.0)
    n = len(v)
    v = np.concatenate([v, v[t[0, :1]], v[t[0, 1:2]] + 2.0])
    t = np.concatenate([t, [[t[0, 0], t[0, 1], n], [t[1, 0], t[1, 0], t[1, 2]], [t[2, 0], t[2, 1], n + 1]]])
    run_rounds(v, t, max_rounds=6)


def test_no_triangles_and_no_vertices():
    assert run_rounds(np.zeros((5, 3)), np.zeros((0, 3), np.int64)) == 0
    assert run_rounds(np.zeros((0, 3)), np.zeros((0, 3), np.int64)) == 0


def test_error_codes():
    L = mesh_emu.lib()
    v, t = sphere_mesh(8, 2.5)
    n, m = len(v), len(t)
    xyz, T = _pad(v, np.float64), _pad(t, np.int64)
    need = int(L.pnr_decimate_workspace_bytes(n, m))
    assert L.pnr_decimate_workspace_bytes(-1, m) == 0
    ws = torch.empty(need, dtype=torch.uint8)
    Q = torch.zeros(n + 1, 10, dtype=torch.float64)
    F = torch.zeros(n + 1, dtype=torch.uint8)
    init = lambda tt=T, q=_p(Q), f=_p(F), w=_p(ws), wb=need, nv=n: L.pnr_decimate_init(  # noqa: E731
        _p(xyz), nv, _p(tt) if tt is not None else None, m, q, f, w, wb, None)
    assert init(wb=need - 1) == PNR_ERR_WORKSPACE and init(w=None, wb=0) == PNR_ERR_WORKSPACE
    assert init(nv=-1) == PNR_ERR_INVALID and init(tt=None) == PNR_ERR_INVALID
    assert init(q=None) == PNR_ERR_INVALID and init(f=None) == PNR_ERR_INVALID
    for bad in (n, -1):
        Tb = T.clone()
        Tb[m // 2, 1] = bad
        assert init(tt=Tb) == PNR_ERR_INVALID
        assert b"outside [0, n_verts)" in L.pnr_last_error()
    assert init() == 0
    cs, ds = torch.zeros(n, dtype=torch.int64), torch.zeros(n, dtype=torch.int64)
    es = torch.zeros(n, dtype=torch.float64)
    counts = (C.c_int64 * 2)()
    cp = C.cast(counts, C.POINTER(C.c_int64))
    sel = lambda bound, w=need, out=cs, cnt=cp, f=_p(F): L.pnr_decimate_select(  # noqa: E731
        _p(xyz), n, _p(T), m, _p(Q), f, bound, _p(out), _p(ds), _p(es), cnt, _p(ws), w, None)
    assert sel(-1.0) == PNR_ERR_INVALID and sel(float("nan")) == PNR_ERR_INVALID
    assert sel(1.0, w=need - 1) == PNR_ERR_WORKSPACE
    assert sel(1.0, cnt=None) == PNR_ERR_INVALID
    assert L.pnr_decimate_select(_p(xyz), n, _p(T), m, _p(Q), _p(F), 1.0, None, _p(ds), _p(es), cp, _p(ws), need,
                                 None) == PNR_ERR_INVALID
    assert sel(1.0, f=None) == PNR_ERR_INVALID
    assert sel(float("inf")) == 0 and counts[0] > 0
    out = torch.zeros(m + 1, 3, dtype=torch.int64)
    count = C.c_int64(0)
    app = lambda k, w=need, o=out, cnt=C.byref(count): L.pnr_decimate_apply(  # noqa: E731
        _p(T), m, n, _p(cs), _p(ds), k, _p(Q), _p(o) if o is not None else None, cnt, _p(ws), w, None)
    assert app(-1) == PNR_ERR_INVALID and app(n // 2 + 1) == PNR_ERR_INVALID
    assert app(1, o=None) == PNR_ERR_INVALID and app(1, cnt=None) == PNR_ERR_INVALID
    assert app(1, w=need - 1) == PNR_ERR_WORKSPACE
    assert app(counts[0]) == 0 and count.value == m - 2 * counts[0]
