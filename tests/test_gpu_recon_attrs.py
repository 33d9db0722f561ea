"""Coloured meshes on the H100: pnr_mc_vertex_attrs bit for bit against the numpy oracle, and
`util.recon.marching_cubes(..., return_colors=True)` on the C2 scene.  The tensor engine's sigma differs in its low bits
from run to run, so every output of a pipeline call is checked against the oracle applied to the sigma volume captured
in that same call, never against another call."""
import os

import numpy as np
import pytest
import torch

import golden_util as gu
import tc_fast_oracle as fo
from recon_util import recon
from test_gpu_recon import C1_, C2_, RESO, assert_same_mesh, c2_net, field_err
from test_gpu_tc_fast import RECON_SIGMA

attrs = gu.load_by_path("pnr_recon_attrs_oracle", os.path.join(gu.ROOT, "oracle", "pnr_recon_attrs.py"))

pytestmark = pytest.mark.gpu


class _Spy:
    """Records the sigma volume and the keywords util.recon hands to pnr_native.marching_cubes."""

    def __init__(self, monkeypatch):
        import pnr_native as pn
        self.vols, self.kws = [], []
        real = pn.marching_cubes

        def spy(vol, iso, **kw):
            self.vols.append(vol.detach().cpu().numpy().copy())
            self.kws.append(kw)
            return real(vol, iso, **kw)
        monkeypatch.setattr(pn, "marching_cubes", spy)


def assert_bits(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_kernel_bit_equal_on_256_cubed_analytic_field():
    import pnr_native as pn
    X, Y, Z = np.meshgrid(*[np.linspace(-1, 1, 256)] * 3, indexing="ij")
    vol = (0.55 - np.sqrt(X * X + Y * Y + Z * Z) + 0.08 * np.sin(9 * X) * np.cos(7 * Y) * np.sin(5 * Z)).astype(
        np.float32)
    lo, hi = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
    out = [t.cpu().numpy() for t in pn.marching_cubes(torch.from_numpy(vol).cuda(), 0.0, bounds=(lo, hi))]
    v, t, n, xyz, vd = out
    assert len(t) > 100000
    assert_same_mesh(v, t, *recon.marching_cubes(vol, 0.0))
    rn, rxyz, rvd = attrs.vertex_attrs(vol, 0.0, lo, hi)
    assert_bits(n, rn)
    assert_bits(xyz, rxyz)
    assert_bits(vd, rvd)
    again = [t.cpu().numpy() for t in pn.marching_cubes(torch.from_numpy(vol).cuda(), 0.0, bounds=(lo, hi))]
    for a, b in zip(again, out):
        assert_bits(a, b)
    v2, t2 = (x.cpu().numpy() for x in pn.marching_cubes(torch.from_numpy(vol).cuda(), 0.0))   # no bounds: 2 outputs
    assert_same_mesh(v2, t2, v, t)


def coloured_mesh_checks(net, state, latent, coarse, monkeypatch, tmp_path=None):
    """util.recon.marching_cubes(..., return_colors=True) against the oracle of the volume captured in the same call;
    -> (rgb, reference rgb at the oracle's query points, oracle xyz / viewdirs of the checked vertices)."""
    from util import recon as urecon
    spy = _Spy(monkeypatch)
    urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9, coarse=coarse)
    assert spy.kws[-1] == {}                              # without colours the call is the two-argument one
    iso = float(np.median(spy.vols[-1]))                  # a level the field crosses
    net.train()
    with pytest.warns(UserWarning, match="fake view dirs"):
        res = urecon.marching_cubes(net, C1_, C2_, RESO, isosurface=iso, eval_batch_size=20000, coarse=coarse,
                                    return_colors=True)
    assert net.training                                   # restored
    net.eval()
    verts, tris, normals, rgb = res
    vol = spy.vols[-1]
    assert vol.shape == tuple(RESO)
    # the mesh is the oracle's marching cubes of the same volume, scaled as the reference scales it
    rv, rt = recon.marching_cubes(vol, iso)
    rv = rv * ((np.array(C2_) - np.array(C1_)) / np.array(RESO)) + np.array(C1_)
    assert len(rt) > 1000
    assert_same_mesh(verts, tris, rv, rt)
    # the normals are the oracle's, bit for bit
    rn, rxyz, rvd = attrs.vertex_attrs(vol, iso, C1_, C2_)
    assert_bits(normals, rn)
    assert rgb.dtype == np.float32 and rgb.shape == verts.shape and np.isfinite(rgb).all()
    # the colour is the field at the oracle's query points and view directions (a spread of the vertices)
    idx = np.linspace(0, len(verts) - 1, 1500).astype(np.int64)
    p, d = torch.from_numpy(rxyz[idx])[None], torch.from_numpy(rvd[idx])[None]
    w = gu.synth.bench_mlp_weights(11 if coarse else 12, 512)
    ref = gu.oracle.field_eval(p, d, state, latent, w, 2)[0, :, :3].numpy()
    if tmp_path is not None:
        path = tmp_path / "mesh.obj"
        urecon.save_obj(verts, tris, str(path), vert_rgb=rgb, vert_normals=normals)
        lines = path.read_text().splitlines()
        vl = [ln.split() for ln in lines if ln.startswith("v ")]
        assert len(vl) == len(verts) and all(len(x) == 7 for x in vl)
        assert sum(ln.startswith("vn ") for ln in lines) == len(verts)
        assert sum(ln.startswith("f ") for ln in lines) == len(tris)
    return rgb[idx], ref, (p, d, w)


@pytest.mark.parametrize("coarse", [True, False])
@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_coloured_mesh_on_c2_scene(engine, coarse, monkeypatch, tmp_path):
    net, state, latent = c2_net(engine)
    got, ref, _ = coloured_mesh_checks(net, state, latent, coarse, monkeypatch, tmp_path)
    assert field_err(got, ref) <= 1e-4


def test_coloured_mesh_single_pass_engine(monkeypatch):
    net, state, latent = c2_net("tc_fast")
    got, ref, (p, d, w) = coloured_mesh_checks(net, state, latent, True, monkeypatch)
    fast = fo.field_eval(p, d, state, latent, w, 2)[0, :, :3].numpy()
    err, tight = field_err(got, ref), field_err(got, fast)
    print(f"tc_fast vertex colour: vs fp32 oracle {err:.2e}, vs restatement {tight:.2e}")
    assert err <= RECON_SIGMA and tight <= fo.TIGHT_FIELD


def test_empty_mesh_makes_no_field_call(monkeypatch):
    from util import recon as urecon
    net, _, _ = c2_net("tc")
    calls = []
    forward = net.forward

    def counted(*a, **kw):
        calls.append(1)
        return forward(*a, **kw)
    monkeypatch.setattr(net, "forward", counted)
    verts, tris, normals, rgb = urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9,
                                                      return_colors=True)
    assert len(calls) == 1                                # the sigma grid only
    assert verts.shape == (0, 3) and tris.shape == (0, 3) and normals.shape == (0, 3) and rgb.shape == (0, 3)
    assert normals.dtype == np.float64 and rgb.dtype == np.float32
    assert len(urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9)) == 2
