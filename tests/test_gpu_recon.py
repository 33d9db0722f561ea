"""Mesh extraction on the H100: the marching-cubes kernels bit for bit against the numpy oracle, and
`util.recon.marching_cubes` on a C2-shaped scene (sigma against the oracle field, mesh against the oracle's marching
cubes of the same volume) and on the reference's golden grids."""
import numpy as np
import pytest
import torch

import golden_util as gu
import gpu_util
from recon_util import recon, sphere

pytestmark = pytest.mark.gpu

C2 = gu.synth.CONFIGS["c2"]
ISO = 0.0


def mc_gpu(vol):
    import pnr_native as pn
    v, t = pn.marching_cubes(torch.from_numpy(vol).cuda(), ISO)
    return v.cpu().numpy(), t.cpu().numpy()


def field_err(got, ref):
    """max |got - ref| relative to the field's scale (1 + max |ref|): the tensor engine's split-fp16 products round
    differently from run to run, by a few 1e-5 of the largest sigma."""
    err = float(np.abs(got - ref).max() / (1.0 + np.abs(ref).max()))
    print(f"field error {err:.2e}")
    return err


def assert_same_mesh(v, t, rv, rt):
    assert v.shape == rv.shape and t.shape == rt.shape
    assert np.array_equal(v.view(np.int64), rv.view(np.int64))
    assert np.array_equal(t, rt)


def test_kernels_bit_equal_on_256_cubed_analytic_field():
    X, Y, Z = np.meshgrid(*[np.linspace(-1, 1, 256)] * 3, indexing="ij")
    vol = (0.55 - np.sqrt(X * X + Y * Y + Z * Z) + 0.08 * np.sin(9 * X) * np.cos(7 * Y) * np.sin(5 * Z)).astype(
        np.float32)
    v, t = mc_gpu(vol)
    assert len(t) > 100000
    assert_same_mesh(v, t, *recon.marching_cubes(vol, ISO))
    v2, t2 = mc_gpu(vol)                                # deterministic: same bits again
    assert_same_mesh(v2, t2, v, t)
    assert recon.is_closed_oriented(t)


class _Spy:
    """Records the sigma volume util.recon hands to pnr_native.marching_cubes."""

    def __init__(self, monkeypatch):
        import pnr_native as pn
        self.vols = []
        real = pn.marching_cubes

        def spy(vol, iso):
            self.vols.append(vol.detach().cpu().numpy().copy())
            return real(vol, iso)
        monkeypatch.setattr(pn, "marching_cubes", spy)


def c2_net(engine, NS=2):
    from model import make_model
    cfg = dict(C2, NS=NS)
    net = make_model(gpu_util.model_conf(cfg["d_hidden"]))
    net.mlp_coarse.load_state_dict(gu.synth.bench_mlp_weights(11, cfg["d_hidden"]))
    net.mlp_fine.load_state_dict(gu.synth.bench_mlp_weights(12, cfg["d_hidden"]))
    net = net.cuda().eval()
    net.engine = engine
    src, _, focal, c = gu.synth.make_cameras(cfg)
    latent = gu.synth.make_latent(5, NS, cfg["H"] // 2, cfg["W"] // 2)
    net.set_scene(latent.cuda(), src[None].cuda(), focal.cuda(), c[None].cuda(), cfg["W"], cfg["H"])
    state = gu.oracle.encode_state(src, focal, c[None], cfg["W"], cfg["H"])
    return net, state, latent


C1_, C2_, RESO = [-0.55, -0.6, -0.5], [0.6, 0.5, 0.55], [40, 36, 44]


@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_marching_cubes_on_c2_scene(engine, monkeypatch, tmp_path):
    from util import recon as urecon
    net, state, latent = c2_net(engine)
    spy = _Spy(monkeypatch)
    urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9)
    iso = float(np.median(spy.vols[-1]))                 # a level the field crosses
    net.train()
    with pytest.warns(UserWarning, match="fake view dirs"):
        verts, tris = urecon.marching_cubes(net, C1_, C2_, RESO, isosurface=iso, eval_batch_size=20000)
    assert net.training                                  # restored
    vol = spy.vols[-1]
    assert vol.shape == tuple(RESO)
    # sigma against the oracle field on a spread of grid points
    pts = recon.grid_points(C1_, C2_, RESO)
    idx = np.linspace(0, len(pts) - 1, 1500).astype(np.int64)
    p = torch.from_numpy(pts[idx])[None]
    d = torch.from_numpy(recon.fake_viewdirs(pts[idx]))[None]
    ref = gu.oracle.field_eval(p, d, state, latent, gu.synth.bench_mlp_weights(11, 512), 2)[0, :, 3].numpy()
    assert field_err(vol.reshape(-1)[idx], ref) <= 1e-4
    # the mesh is the oracle's marching cubes of the same volume, scaled as the reference scales it
    rv, rt = recon.marching_cubes(vol, iso)
    rv = rv * ((np.array(C2_) - np.array(C1_)) / np.array(RESO)) + np.array(C1_)
    assert len(rt) > 1000
    assert_same_mesh(verts, tris, rv, rt)
    # the kernels on the real model's volume
    import pnr_native as pn
    kv, kt = pn.marching_cubes(torch.from_numpy(vol).cuda(), iso)
    assert_same_mesh(kv.cpu().numpy(), kt.cpu().numpy(), *recon.marching_cubes(vol, iso))
    # save_obj round trip
    path = tmp_path / "mesh.obj"
    urecon.save_obj(verts, tris, str(path))
    lines = path.read_text().splitlines()
    vl = np.array([[float(x) for x in ln.split()[1:]] for ln in lines if ln.startswith("v ")])
    fl = np.array([[int(x) for x in ln.split()[1:]] for ln in lines if ln.startswith("f ")])
    assert np.array_equal(fl - 1, tris)
    assert np.abs(vl - verts).max() <= 0.5e-4 + 1e-12
    assert all(ln == "v %.4f %.4f %.4f" % tuple(v) for ln, v in zip(lines, verts))
    rgb = np.random.default_rng(0).random(verts.shape)
    urecon.save_obj(verts, tris, str(path), vert_rgb=rgb)
    first = path.read_text().splitlines()[0]
    assert first == "v %.4f %.4f %.4f %.4f %.4f %.4f" % (*verts[0], *rgb[0])


def test_fine_network_and_sigma_idx(monkeypatch):
    from util import recon as urecon
    net, state, latent = c2_net("auto")
    spy = _Spy(monkeypatch)
    reso = [20, 18, 22]
    urecon.marching_cubes(net, C1_, C2_, reso, isosurface=1.0, coarse=False)
    fine = spy.vols[-1]
    urecon.marching_cubes(net, C1_, C2_, reso, isosurface=0.5, sigma_idx=1, coarse=False)
    green = spy.vols[-1]
    pts = recon.grid_points(C1_, C2_, reso)
    p = torch.from_numpy(pts)[None]
    d = torch.from_numpy(recon.fake_viewdirs(pts))[None]
    ref = gu.oracle.field_eval(p, d, state, latent, gu.synth.bench_mlp_weights(12, 512), 2)[0].numpy()
    for got, ch in ((fine, 3), (green, 1)):
        assert field_err(got.reshape(-1), ref[:, ch]) <= 1e-4, ch


def test_refuses_several_objects_and_cpu():
    from util import recon as urecon
    net, _, _ = c2_net("auto")
    net.num_objs = 2
    with pytest.raises(RuntimeError, match="one object"):
        urecon.marching_cubes(net, reso=[8, 8, 8])
    net.num_objs = 1
    with pytest.raises(RuntimeError, match="CUDA"):
        urecon.marching_cubes(net, reso=[8, 8, 8], device="cpu")


@pytest.mark.parametrize("ns", [1, 2])
def test_golden_grids_replayed_through_the_gpu_path(ns, monkeypatch):
    from util import recon as urecon
    z = np.load(f"{gu.GOLD}/recon_ns{ns}.npz")
    case = gu.load_case(str(z["case"]))
    case = dict(case, src_poses=case["src_poses"][:, :ns], latent=case["latent"][:ns], cfg=dict(case["cfg"], NS=ns))
    net = gpu_util.build_net(case)
    spy = _Spy(monkeypatch)
    for grid in ("box", "odd", "flat"):
        lo, hi, reso = (z[f"{grid}/{k}"].tolist() for k in ("lo", "hi", "reso"))
        for coarse, key in ((True, "coarse"), (False, "fine")):
            urecon.marching_cubes(net, lo, hi, reso, isosurface=5.0, coarse=coarse, eval_batch_size=100)
            got = spy.vols[-1].reshape(-1)
            ref = z[f"{grid}/{key}"][:, 3]
            fin = np.isfinite(ref)
            assert fin.sum() >= len(ref) - 1
            assert field_err(got[fin], ref[fin]) <= 1e-4, (grid, key)
