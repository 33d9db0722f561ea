"""pnr_mesh_components and pnr_mesh_compact_count / _emit (csrc/pnr_mesh.cu) on the host emulator (built by
tests/mesh_emu.py): labels, triangle counts, the component count and the compacted mesh bit for bit against the
oracle (oracle/pnr_recon_components.py) on random soups with many components, a long path whose ids decrease along it
(deep trees for find), one giant component, no triangles and no vertices, and the error codes."""
import ctypes as C

import numpy as np
import pytest
import torch

import mesh_emu
from components_util import comp, random_soup

PNR_ERR_INVALID, PNR_ERR_WORKSPACE = -1, -2


def _p(t):
    return C.c_void_p(t.data_ptr())


def _i64(a):
    """int64 CPU tensor of a, padded with one row so that no pointer is NULL"""
    a = np.asarray(a, dtype=np.int64)
    return torch.from_numpy(np.concatenate([a, np.zeros((1,) + a.shape[1:], np.int64)]))


def emu_components(tris, n):
    L = mesh_emu.lib()
    m = len(tris)
    t = _i64(tris)
    ws = torch.empty(int(L.pnr_mesh_workspace_bytes(n, m)), dtype=torch.uint8)
    label = torch.full((n + 1,), -7, dtype=torch.int64)
    tri_count = torch.full((n + 1,), -7, dtype=torch.int64)
    count = C.c_int64(-7)
    rc = L.pnr_mesh_components(_p(t), m, n, _p(label), _p(tri_count), C.byref(count), _p(ws), ws.numel(), None)
    assert rc == 0, L.pnr_last_error().decode()
    assert label[n] == -7 and tri_count[n] == -7                  # nothing past the end
    return label.numpy()[:n], tri_count.numpy()[:n], count.value


def emu_compact(tris, n, label, keep_root):
    L = mesh_emu.lib()
    m = len(tris)
    t = _i64(tris)
    lab = _i64(label)
    keep = torch.from_numpy(np.concatenate([np.asarray(keep_root, dtype=np.uint8), [0]]).astype(np.uint8))
    ws = torch.empty(int(L.pnr_mesh_workspace_bytes(n, m)), dtype=torch.uint8)
    counts = torch.full((2,), -7, dtype=torch.int64)
    rc = L.pnr_mesh_compact_count(_p(t), m, n, _p(lab), _p(keep), _p(counts), _p(ws), ws.numel(), None)
    assert rc == 0, L.pnr_last_error().decode()
    nv, nt = counts.tolist()
    vert_ids = torch.full((nv + 1,), -7, dtype=torch.int64)
    tris_out = torch.full((nt + 1, 3), -7, dtype=torch.int64)
    rc = L.pnr_mesh_compact_emit(_p(t), m, n, _p(vert_ids), _p(tris_out), nv, nt, _p(ws), ws.numel(), None)
    assert rc == 0, L.pnr_last_error().decode()
    assert vert_ids[nv] == -7 and (tris_out[nt] == -7).all()
    return vert_ids.numpy()[:nv], tris_out.numpy()[:nt]


def check(tris, n, largest=1, min_triangles=1):
    """Both kernels against the oracle; the compaction with the roots the oracle's policy keeps."""
    label, tri_count, count = emu_components(tris, n)
    want_label = comp.labels(tris, n)
    want_count = comp.tri_counts(tris, want_label)
    assert np.array_equal(label, want_label)
    assert np.array_equal(tri_count, want_count)
    assert count == np.count_nonzero(want_count)
    keep_root = np.zeros(n, dtype=np.uint8)
    keep_root[comp.kept_roots(want_count, largest, min_triangles)] = 1
    vert_ids, tris_out = emu_compact(tris, n, label, keep_root)
    verts = np.arange(n, dtype=np.int64)[:, None]                   # a vertex's old id, as its "position"
    want_v, want_t = comp.keep_components(verts, np.asarray(tris, dtype=np.int64).reshape(-1, 3), largest=largest,
                                          min_triangles=min_triangles)
    assert np.array_equal(vert_ids, want_v[:, 0]) and np.array_equal(tris_out, want_t)
    return label, count


@pytest.mark.parametrize("seed", range(5))
def test_random_soups(seed):
    g = np.random.default_rng(seed)
    n = int(g.integers(200, 3000))
    tris = random_soup(seed, n, int(g.integers(n // 4, 2 * n)))
    label, count = check(tris, n)
    assert count > 10
    check(tris, n, largest=None, min_triangles=3)
    check(tris, n, largest=4, min_triangles=2)


def test_long_path_with_decreasing_ids():
    n = 5000
    ids = np.arange(n - 1, -1, -1)
    tris = np.stack([ids[:-2], ids[1:-1], ids[2:]], 1)              # a strip walked from the largest id down
    label, count = check(tris, n)
    assert count == 1 and (label == 0).all()
    # the same strip, walked from both ends inward, and as its reverse
    check(np.concatenate([tris[::2], tris[1::2][::-1]]), n)
    check(tris[:, ::-1].copy(), n)


def test_one_giant_component():
    n = 4000
    g = np.random.default_rng(11)
    tris = g.integers(0, n, size=(3 * n, 3))
    tris[:n, 0] = np.arange(n)                                     # every vertex used
    tris[:n, 1] = (np.arange(n) + 1) % n                           # and chained into one ring
    label, count = check(tris, n)
    assert count == 1 and (label == 0).all()


def test_no_triangles_and_no_vertices():
    label, tri_count, count = emu_components(np.zeros((0, 3)), 5)
    assert np.array_equal(label, np.arange(5)) and not tri_count.any() and count == 0
    v, t = emu_compact(np.zeros((0, 3)), 5, label, np.ones(5))
    assert np.array_equal(v, np.arange(5)) and t.shape == (0, 3)
    label, tri_count, count = emu_components(np.zeros((0, 3)), 0)
    assert label.shape == (0,) and count == 0
    v, t = emu_compact(np.zeros((0, 3)), 0, label, np.zeros(0))
    assert v.shape == (0,) and t.shape == (0, 3)
    # vertices no triangle uses are components of their own with no triangle
    tris = np.array([[3, 4, 6]])
    label, count = check(tris, 8)
    _, tri_count, _ = emu_components(tris, 8)
    assert np.array_equal(label, [0, 1, 2, 3, 3, 5, 3, 7]) and np.array_equal(tri_count, [0, 0, 0, 1, 0, 0, 0, 0])


def test_error_codes():
    L = mesh_emu.lib()
    n, m = 4, 2
    tris = _i64([[0, 1, 2], [1, 2, 3]])
    label, tri_count = torch.zeros(n, dtype=torch.int64), torch.zeros(n, dtype=torch.int64)
    keep, counts = torch.ones(n, dtype=torch.uint8), torch.zeros(2, dtype=torch.int64)
    out_v, out_t = torch.zeros(n, dtype=torch.int64), torch.zeros(m, 3, dtype=torch.int64)
    need = int(L.pnr_mesh_workspace_bytes(n, m))
    ws = torch.empty(need, dtype=torch.uint8)
    count = C.c_int64(0)
    assert L.pnr_mesh_workspace_bytes(-1, 0) == 0 and L.pnr_mesh_workspace_bytes(0, -1) == 0

    def comps(t=_p(tris), m=m, n=n, lab=_p(label), tc=_p(tri_count), c=C.byref(count), w=_p(ws), wb=need):
        return L.pnr_mesh_components(t, m, n, lab, tc, c, w, wb, None)

    def ccount(t=_p(tris), m=m, n=n, lab=_p(label), k=_p(keep), c=_p(counts), w=_p(ws), wb=need):
        return L.pnr_mesh_compact_count(t, m, n, lab, k, c, w, wb, None)

    def emit(t=_p(tris), m=m, n=n, v=_p(out_v), o=_p(out_t), nv=n, nt=m, w=_p(ws), wb=need):
        return L.pnr_mesh_compact_emit(t, m, n, v, o, nv, nt, w, wb, None)
    assert comps() == 0 and count.value == 1
    assert ccount() == 0 and counts.tolist() == [4, 2]
    assert emit() == 0 and out_v.tolist() == [0, 1, 2, 3] and out_t.tolist() == [[0, 1, 2], [1, 2, 3]]
    for f in (comps, ccount, emit):
        for kw in (dict(t=None), dict(m=-1), dict(n=-1)):
            assert f(**kw) == PNR_ERR_INVALID, (f.__name__, kw)
        assert f(wb=need - 1) == PNR_ERR_WORKSPACE, f.__name__
        assert f(w=None) == PNR_ERR_WORKSPACE, f.__name__
        assert f(t=None, m=0, wb=int(L.pnr_mesh_workspace_bytes(n, 0))) == 0, f.__name__
    for kw in (dict(lab=None), dict(tc=None), dict(c=None)):
        assert comps(**kw) == PNR_ERR_INVALID, kw
    for kw in (dict(lab=None), dict(k=None), dict(c=None)):
        assert ccount(**kw) == PNR_ERR_INVALID, kw
    for kw in (dict(v=None), dict(o=None), dict(nv=-1), dict(nt=-1)):
        assert emit(**kw) == PNR_ERR_INVALID, kw
    # ids out of range, found on the device: equal to n_verts, negative, huge, and any vertex with n_verts = 0
    for bad in ([0, 1, 4], [4, 1, 2], [0, -1, 2], [-(2 ** 63), 0, 1], [0, 1, 2 ** 62]):
        t = _i64([[0, 1, 2], bad])
        assert comps(t=_p(t)) == PNR_ERR_INVALID, bad
        assert b"outside [0, n_verts)" in L.pnr_last_error(), bad
        assert ccount(t=_p(t)) == 0 and counts.tolist()[1] <= 1    # a triangle out of range is never kept
    assert comps(n=0, wb=int(L.pnr_mesh_workspace_bytes(0, m))) == PNR_ERR_INVALID
    assert comps(m=1, n=3, wb=int(L.pnr_mesh_workspace_bytes(3, 1))) == 0
