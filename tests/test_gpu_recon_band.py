"""Narrow-band mesh extraction on the H100: the pnr_band_* kernels bit for bit against the numpy oracle
(oracle/pnr_recon_band.py) and the dense kernels, and `util.recon.marching_cubes(..., block=b)` on the C2 scene against
the dense call: the same sigma at every point it evaluates, and exactly the masked-dense mesh of the dense volume."""
import os

import numpy as np
import pytest
import torch

import golden_util as gu
import gpu_util
from recon_util import recon
from test_gpu_recon import C1_, C2_, c2_net, field_err

band = gu.load_by_path("pnr_recon_band_oracle", os.path.join(gu.ROOT, "oracle", "pnr_recon_band.py"))

pytestmark = pytest.mark.gpu


def bits(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def analytic(n):
    X, Y, Z = np.meshgrid(*[np.linspace(-1, 1, n)] * 3, indexing="ij")
    return (0.55 - np.sqrt(X * X + Y * Y + Z * Z) + 0.08 * np.sin(9 * X) * np.cos(7 * Y) * np.sin(5 * Z)).astype(
        np.float32)


@pytest.mark.parametrize("b", [4, 8])
def test_kernels_on_256_cubed_analytic_field(b):
    import pnr_native as pn
    vol = analytic(256)
    reso, lo, hi = list(vol.shape), (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
    flat = vol.reshape(-1)
    lat = band.lattice_flat(reso, b)
    xyz = torch.empty(len(lat), 3, device="cuda")
    vd = torch.empty(len(lat), 3, device="cuda")
    pn.band_lattice_points(lo, hi, reso, b, 0, len(lat), xyz, vd)
    rxyz, rvd = band.lattice_points(lo, hi, reso, b)
    bits(xyz.cpu().numpy(), rxyz)
    bits(vd.cpu().numpy(), rvd)
    plan = pn.band_plan(torch.from_numpy(flat[lat]).cuda(), reso, b, 0.0, apron=True)
    _, active = band.plan(flat[lat], reso, b, 0.0)
    idx = band.refine_index(active, reso, b, True)
    assert (plan.n_active, plan.n_points) == (int(active.sum()), len(idx))
    assert plan.n_points < len(flat) // 4                                 # a thin shell of the grid
    pts = torch.empty(plan.n_points, 3, device="cuda")
    pn.band_points(plan, lo, hi, 0, plan.n_points, pts)
    bits(pts.cpu().numpy(), recon.grid_points(lo, hi, reso)[idx])
    sigma = torch.from_numpy(flat[idx]).cuda()
    out = [t.cpu().numpy() for t in pn.band_marching_cubes(sigma, plan, 0.0, bounds=(lo, hi))]
    v, t, n, axyz, avd = out
    rv, rt, complete = band.marching_cubes(vol, 0.0, b)
    assert complete and len(t) > 100000
    bits(v, rv)
    bits(t, rt)
    rn, rx, rd = band.vertex_attrs(vol, 0.0, lo, hi, b)
    bits(n, rn)
    bits(axyz, rx)
    bits(avd, rd)
    # complete coverage: the dense kernels' mesh and attributes, bit for bit
    dense = [x.cpu().numpy() for x in pn.marching_cubes(torch.from_numpy(vol).cuda(), 0.0, bounds=(lo, hi))]
    for a, d in zip(out, dense):
        bits(a, d)
    again = [x.cpu().numpy() for x in pn.band_marching_cubes(sigma, plan, 0.0, bounds=(lo, hi))]
    for a, d in zip(again, out):
        bits(a, d)


class _Spy:
    """Records what util.recon hands to the library: the dense volume, the coarse lattice sigma and plan, and the
    refinement sigma."""

    def __init__(self, monkeypatch):
        import pnr_native as pn
        self.dense, self.coarse, self.plans, self.band = [], [], [], []
        real_mc, real_plan, real_band = pn.marching_cubes, pn.band_plan, pn.band_marching_cubes

        def mc(vol, iso, **kw):
            self.dense.append(vol.detach().cpu().numpy().copy())
            return real_mc(vol, iso, **kw)

        def plan(coarse, reso, block, iso, apron=False):
            self.coarse.append(coarse.detach().cpu().numpy().copy())
            p = real_plan(coarse, reso, block, iso, apron)
            self.plans.append(p)
            return p

        def band_mc(sigma, plan, iso, **kw):
            self.band.append(sigma.detach().cpu().numpy().copy())
            return real_band(sigma, plan, iso, **kw)
        monkeypatch.setattr(pn, "marching_cubes", mc)
        monkeypatch.setattr(pn, "band_plan", plan)
        monkeypatch.setattr(pn, "band_marching_cubes", band_mc)


def scaled(v, reso):
    return v * ((np.array(C2_) - np.array(C1_)) / np.array(reso)) + np.array(C1_)


@pytest.mark.parametrize("n", [128, 256])
@pytest.mark.parametrize("engine", ["tc", "tc_fast", "simt"])
def test_c2_scene_band_against_dense(engine, n, monkeypatch):
    from util import recon as urecon
    net, _, _ = c2_net(engine)
    spy = _Spy(monkeypatch)
    reso = [n, n, n]
    urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9)
    iso = float(np.percentile(spy.dense[-1], 70))          # a level the field crosses
    dv, dt = urecon.marching_cubes(net, C1_, C2_, reso, isosurface=iso, eval_batch_size=50000)
    vol = spy.dense[-1]
    flat = vol.reshape(-1)
    if n == 128:                                            # the dense colours, for the band's kept vertices
        dense_colour = urecon.marching_cubes(net, C1_, C2_, reso, isosurface=iso, eval_batch_size=50000,
                                             return_colors=True)
        bits(spy.dense[-1], vol)
    for b, colours in ((8, False), (4, True)) if n == 128 else ((8, False),):
        res = urecon.marching_cubes(net, C1_, C2_, reso, isosurface=iso, eval_batch_size=50000, block=b,
                                    return_colors=colours)
        coarse, plan, sigma = spy.coarse[-1], spy.plans[-1], spy.band[-1]
        lat = band.lattice_flat(reso, b)
        _, active = band.plan(coarse, reso, b, iso)
        idx = band.refine_index(active, reso, b, colours)
        assert (plan.n_active, plan.n_points) == (int(active.sum()), len(idx)) and len(sigma) == len(idx)
        # the mesh is exactly the masked-dense mesh of the sigma this call evaluated
        own = flat.copy()
        own[lat] = coarse
        own[idx] = sigma
        own = own.reshape(reso)
        rv, rt, complete = band.marching_cubes(own, iso, b)
        assert len(rt) > 1000
        bits(res[0], scaled(rv, reso))
        bits(res[1], rt)
        if colours:
            bits(res[2], band.vertex_attrs(own, iso, C1_, C2_, b)[0])
            assert res[3].shape == res[0].shape and np.isfinite(res[3]).all()
        # each point's sigma depends only on that point: the band evaluates the dense volume's values
        same_lat = np.array_equal(coarse.view(np.int32), flat[lat].view(np.int32))
        same = np.array_equal(sigma.view(np.int32), flat[idx].view(np.int32))
        print(f"{engine} {n}^3 b={b}: coverage {'complete' if complete else 'partial'}, {len(idx)} of {len(flat)} "
              f"points, field error vs dense {field_err(sigma, flat[idx]):.2e}")
        assert same_lat and same
        # and so it is the masked-dense mesh of the dense volume; under complete coverage the dense mesh itself
        rv, rt, complete = band.marching_cubes(vol, iso, b)
        bits(res[1], rt)
        if complete:
            bits(res[0], dv)
            bits(res[1], dt)
        if colours:                                         # normals and colours of the kept vertices: the dense ones
            used = band.kept_vertices(vol, iso, b)
            bits(res[0], dense_colour[0][used])
            bits(res[2], dense_colour[2][used])
            bits(res[3], dense_colour[3][used])


class _Blob(torch.nn.Module):
    """A smooth analytic field in place of a network, on the GPU: sigma = 40 (0.45 - |p - c|) plus a ripple, rgb from
    the point and the view direction (so that swapping them shows).  Elementwise, so each point's value depends only on
    that point."""
    use_viewdirs, num_objs = True, 1

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, device="cuda"))

    def forward(self, pts, coarse=True, viewdirs=None):
        p = pts - torch.tensor([0.05, -0.03, 0.02], device=pts.device)
        r = torch.sqrt((p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1]) + p[..., 2] * p[..., 2])
        sigma = 40.0 * (0.45 - r + 0.04 * torch.sin(7 * p[..., 0]) * torch.cos(5 * p[..., 1]))
        rgb = torch.sigmoid(3.0 * pts + 2.0 * viewdirs)
        return torch.cat([rgb, sigma[..., None]], -1)


@pytest.mark.parametrize("b", [4, 8])
def test_complete_coverage_through_util_recon_is_the_dense_result(b, monkeypatch):
    from util import recon as urecon
    net = _Blob()
    spy = _Spy(monkeypatch)
    box = ([-0.6] * 3, [0.6] * 3)
    reso = [96, 101, 90]
    with pytest.warns(UserWarning, match="fake view dirs"):
        dense = urecon.marching_cubes(net, *box, reso, isosurface=0.0, eval_batch_size=30000, return_colors=True)
        got = urecon.marching_cubes(net, *box, reso, isosurface=0.0, eval_batch_size=30000, return_colors=True,
                                    block=b)
        v, t = urecon.marching_cubes(net, *box, reso, isosurface=0.0, eval_batch_size=30000, block=b)
    assert band.marching_cubes(spy.dense[-1], 0.0, b)[2]                  # complete coverage
    assert spy.plans[-1].n_points < np.prod(reso) * (0.5 if b == 4 else 0.8)     # the sphere fills much of the box
    assert len(dense[1]) > 20000
    for a, d in zip(got, dense):
        bits(a, d)
    bits(v, dense[0])
    bits(t, dense[1])


@pytest.mark.parametrize("ns", [1, 2])
def test_golden_grids_replayed_through_the_band(ns, monkeypatch):
    from util import recon as urecon
    z = np.load(f"{gu.GOLD}/recon_ns{ns}.npz")
    case = gu.load_case(str(z["case"]))
    case = dict(case, src_poses=case["src_poses"][:, :ns], latent=case["latent"][:ns], cfg=dict(case["cfg"], NS=ns))
    net = gpu_util.build_net(case)
    spy = _Spy(monkeypatch)
    for grid in ("box", "odd", "flat"):
        lo, hi, reso = (z[f"{grid}/{k}"].tolist() for k in ("lo", "hi", "reso"))
        for coarse, key in ((True, "coarse"), (False, "fine")):
            ref = z[f"{grid}/{key}"][:, 3]
            for b in (2, 3):
                urecon.marching_cubes(net, lo, hi, reso, isosurface=5.0, coarse=coarse, eval_batch_size=100, block=b)
                lat = band.lattice_flat(reso, b)
                got = spy.coarse[-1]
                fin = np.isfinite(ref[lat])
                assert fin.sum() >= len(lat) - 1
                assert field_err(got[fin], ref[lat][fin]) <= 1e-4, (grid, key, b)
                if spy.plans[-1].n_points:
                    _, active = band.plan(got, reso, b, 5.0)
                    idx = band.refine_index(active, reso, b)
                    fin = np.isfinite(ref[idx])
                    assert field_err(spy.band[-1][fin], ref[idx][fin]) <= 1e-4, (grid, key, b)


def test_defaults_and_validation(monkeypatch):
    from util import recon as urecon
    net, _, _ = c2_net("tc")
    spy = _Spy(monkeypatch)
    urecon.marching_cubes(net, C1_, C2_, [10, 11, 12], isosurface=1.0)
    assert len(spy.dense) == 1 and not spy.coarse                      # block=None: the dense call
    for bad in (True, 1, 0, -4, 257, 4.0, "8"):
        with pytest.raises(ValueError, match="block"):
            urecon.marching_cubes(net, C1_, C2_, [10, 11, 12], block=bad)
    net.num_objs = 2
    with pytest.raises(RuntimeError, match="one object"):
        urecon.marching_cubes(net, reso=[8, 8, 8], block=4)
    net.num_objs = 1
    v, t, n, rgb = urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9, block=4, return_colors=True)
    assert v.shape == t.shape == n.shape == rgb.shape == (0, 3)
    assert v.dtype == n.dtype == np.float64 and t.dtype == np.int64 and rgb.dtype == np.float32
    assert len(urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9, block=4)) == 2
