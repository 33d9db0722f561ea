"""Decimation on the H100: `util.recon.decimate` bit for bit against the oracle (oracle/pnr_recon_decimate.py) on the
C2 scene's marching_cubes mesh (normals and colours) and its fuse_views(colors="views") mesh after keep_components,
on the GPU marching cubes of the analytic sphere and torus, the same bits from two calls on a dense 256^3 mesh of
millions of triangles with its boundary kept, and the refusals."""
import numpy as np
import pytest
import torch

from decimate_util import bipyramid, bits_equal, dec, directed_edges_once, euler_per_component, is_closed
from recon_util import sphere, torus
from test_gpu_recon import C1_, C2_, c2_net
from test_gpu_recon import _Spy as _VolSpy

pytestmark = pytest.mark.gpu


def assert_matches_oracle(mesh, **kw):
    from util import recon as urecon
    got = urecon.decimate(*mesh, **kw)
    want = dec.decimate(*mesh, **kw)
    assert len(got) == len(want) == len(mesh)
    for a, b in zip(got, want):
        assert bits_equal(a, b)
    return got


def test_analytic_sphere_and_torus_through_the_gpu_marching_cubes():
    import pnr_native as pn
    for vol in (sphere((64, 64, 64), 25.0), torus((72, 72, 72), 22.0, 9.0)):
        v, t = (a.cpu().numpy() for a in pn.marching_cubes(torch.from_numpy(vol).cuda(), 0.0))
        got = assert_matches_oracle((v, t), target_triangles=len(t) // 5)
        assert len(got[1]) in (len(t) // 5 - 1, len(t) // 5) and is_closed(got[1])
        assert_matches_oracle((v, t), max_error=0.02)


def c2_iso(net, monkeypatch):
    from util import recon as urecon
    spy = _VolSpy(monkeypatch)
    urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9)
    iso = float(np.quantile(spy.vols[-1], 0.7))
    monkeypatch.undo()
    return iso


def test_decimate_marching_cubes_on_c2_scene(monkeypatch):
    from util import recon as urecon
    net, _, _ = c2_net("tc")
    iso = c2_iso(net, monkeypatch)
    mesh = urecon.marching_cubes(net, C1_, C2_, [40, 36, 44], isosurface=iso, return_colors=True)
    assert len(mesh[1]) > 1000
    got = assert_matches_oracle(mesh, target_triangles=len(mesh[1]) // 4)
    assert got[2].dtype == mesh[2].dtype and got[3].dtype == mesh[3].dtype
    assert_matches_oracle(mesh, max_error=1e-3)
    assert_matches_oracle(urecon.keep_components(*mesh, largest=1), target_triangles=len(mesh[1]) // 3,
                          max_error=1e-2)


def test_decimate_fuse_views_on_c2_scene(monkeypatch):
    from test_gpu_recon_fuse import c2_scene
    from test_gpu_recon_paint import _Spy as _PaintSpy
    from test_gpu_recon_paint import call
    from util import recon as urecon
    net, renderer, poses = c2_scene()
    spy = _PaintSpy(monkeypatch)
    call(net, renderer, poses)
    m = float(np.clip(np.median(spy.fused[-1][1]), 0.05, 1.0))
    mesh = urecon.keep_components(*call(net, renderer, poses, min_opacity=m, return_colors=True, colors="views"),
                                  largest=1)
    assert len(mesh[1]) > 100
    assert_matches_oracle(mesh, target_triangles=len(mesh[1]) // 4)
    # in the other order: decimate, then keep the largest piece
    kept = urecon.keep_components(*urecon.decimate(*mesh, target_triangles=len(mesh[1]) // 2), largest=1)
    assert len(kept[1]) > 0


def test_dense_256_two_calls_same_bits(monkeypatch):
    from util import recon as urecon
    net, _, _ = c2_net("tc")
    # the mesh of scripts/bench_recon_decimate.py at 256^3: [-0.6, 0.6]^3 at the median sigma of a 32^3 probe
    spy = _VolSpy(monkeypatch)
    urecon.marching_cubes(net, [-0.6] * 3, [0.6] * 3, [32] * 3, isosurface=1e9)
    iso = float(np.median(spy.vols[-1]))
    monkeypatch.undo()
    v, t = urecon.marching_cubes(net, [-0.6] * 3, [0.6] * 3, [256] * 3, isosurface=iso)
    print(f"dense 256^3: {len(t)} triangles")
    assert len(t) >= 4_000_000
    target = len(t) // 10
    a = urecon.decimate(v, t, target_triangles=target)
    b = urecon.decimate(v, t, target_triangles=target)
    assert bits_equal(a[0], b[0]) and bits_equal(a[1], b[1])
    assert len(a[1]) in (target - 1, target)
    # the boundary edges come through: the same positions on both sides
    def boundary_positions(vv, tt):
        e = np.concatenate([tt[:, [0, 1]], tt[:, [1, 2]], tt[:, [2, 0]]]).astype(np.int64)
        key = e[:, 0] * len(vv) + e[:, 1]
        rev = e[:, 1] * len(vv) + e[:, 0]
        b = e[~np.isin(key, rev)]
        return np.unique(np.concatenate([vv[b[:, 0]], vv[b[:, 1]]], axis=1), axis=0)
    assert bits_equal(boundary_positions(*a[:2]), boundary_positions(v, t))
    # every directed edge once, before and after, and each component keeps its Euler characteristic
    assert directed_edges_once(t) and directed_edges_once(a[1])
    chi, chi_out = euler_per_component(v, t), euler_per_component(*a[:2])
    print(f"{len(chi)} components, Euler characteristics {sorted(set(chi.values()))}")
    assert sorted(chi.values()) == sorted(chi_out.values())


def test_frozen_apexes_and_tiny_meshes():
    from util import recon as urecon
    v, t = bipyramid(100)                                 # apexes of 100 corners: frozen, never removed
    got = assert_matches_oracle((v, t), max_error=0.05)
    assert bits_equal(got[0][-2:], v[-2:])
    assert_matches_oracle((v, t), target_triangles=8)
    for mesh in ((np.zeros((1, 3)), np.array([[0, 0, 0]])), (np.zeros((0, 3)), np.zeros((0, 3), np.int64)),
                 (np.eye(3), np.array([[0, 1, 2]]))):
        out = urecon.decimate(*mesh, max_error=0.0)
        assert bits_equal(out[0], mesh[0]) and bits_equal(out[1], mesh[1])


def test_refusals():
    from util import recon as urecon
    v = np.zeros((4, 3))
    t = np.array([[0, 1, 2], [1, 2, 3]])
    for kw in (dict(), dict(target_triangles=-1), dict(target_triangles=1.5), dict(target_triangles=True),
               dict(max_error=-1.0), dict(max_error=float("nan")), dict(max_error=float("inf")),
               dict(max_error="1")):
        with pytest.raises(ValueError, match="target_triangles|max_error"):
            urecon.decimate(v, t, **kw)
    for args in ((np.zeros((4, 2)), t), (np.zeros(12), t), (v, t[:, :2]), (v, t.astype(np.float64)),
                 (v, t, np.zeros((3, 3))), (v, t, np.zeros(())), (v, np.array([[0, 1, 4]])),
                 (v, np.array([[0, -1, 2]])), (v, np.array([[0, 1, 2], [2 ** 40, 0, 1]]))):
        with pytest.raises(ValueError):
            urecon.decimate(*args, target_triangles=1)
    with pytest.raises(RuntimeError, match="CUDA"):
        urecon.decimate(v, t, target_triangles=1, device="cpu")
