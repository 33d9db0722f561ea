"""Vertex colours from the rendered views on the H100: pnr_paint_vertices bit for bit against the numpy oracle
(oracle/pnr_recon_paint.py) on an analytic sphere fused at 128^3 from 64 views, and `util.recon.fuse_views(...,
colors="views")` on the C2 scene.  The tensor engine's renders differ in their low bits from run to run, so the colours
of a call are checked against the oracle applied to the maps captured in that same call, and the vertices no view
paints against the field colours that call computed for them."""
import numpy as np
import pytest
import torch

from fuse_util import views
from paint_util import gradient_colour, paint, sphere_scene_maps
from test_gpu_recon import c2_net
from test_gpu_recon_fuse import BS, C2, FOCAL, HI, LO, RESO, H, W, bits, c2_scene

pytestmark = pytest.mark.gpu


def test_kernel_bit_equal_at_128_cubed_with_64_views():
    import pnr_native as pn
    poses = views(62, 3.0)                                  # 64 views
    r, f, n = 0.5, 160.0, 96
    rgb, depth, opacity = sphere_scene_maps(poses, n, n, f, [((0.0, 0.0, 0.0), r, gradient_colour(r))])
    lo, hi, reso = np.full(3, -1.0), np.full(3, 1.0), (128,) * 3
    h = (hi - lo) / (np.array(reso) - 1)
    trunc = 3.0 * np.sqrt(3.0) * float(h.max())
    rgb_d, depth_d, opacity_d = (torch.from_numpy(a).cuda() for a in (rgb, depth, opacity))
    poses_d = poses.cuda()
    cam = (f, f, n / 2, n / 2)
    tsdf = pn.tsdf_fuse(depth_d, opacity_d, poses_d, *cam, lo, hi, reso, trunc, 0.5)
    v, t, normals, _, _ = pn.marching_cubes(-tsdf, 0.0, bounds=(lo, hi))
    x = v.cpu().numpy() * h + lo
    args = (torch.from_numpy(x).cuda(), normals, rgb_d, depth_d, opacity_d, poses_d, *cam, trunc, 0.5, 1.0)
    col, weight = (a.cpu().numpy() for a in pn.paint_vertices(*args))
    want, want_w = paint.paint_vertices(x, normals.cpu().numpy(), rgb, depth, opacity, poses.numpy(), *cam, trunc, 0.5,
                                        1.0)
    print(f"{len(x)} vertices")
    assert len(x) > 10000
    bits(col, want)
    bits(weight, want_w)
    assert (weight > 0).all()
    col2, weight2 = (a.cpu().numpy() for a in pn.paint_vertices(*args))
    bits(col2, col)                                         # deterministic
    bits(weight2, weight)
    err = np.abs(col - gradient_colour(r)(x)).max(1)
    print(f"max colour error {err.max():.4f}, mean {err.mean():.4f}")


class _Spy:
    """Records the inputs of every pnr_native.tsdf_fuse call, the inputs and outputs of every pnr_native.paint_vertices
    call, and the rows and outputs of every util.recon._colours call."""

    def __init__(self, monkeypatch):
        import pnr_native as pn
        from util import recon as urecon
        self.fused, self.painted, self.coloured = [], [], []
        real_fuse, real_paint, real_colours = pn.tsdf_fuse, pn.paint_vertices, urecon._colours
        host = lambda a: a.cpu().numpy().copy() if torch.is_tensor(a) else a     # noqa: E731

        def tsdf_fuse(depth, opacity, *a):
            self.fused.append((host(depth), host(opacity)))
            return real_fuse(depth, opacity, *a)

        def paint_vertices(*a):
            out = real_paint(*a)
            self.painted.append(([host(x) for x in a], [host(x) for x in out]))
            return out

        def colours(net, xyz, vd, *a):
            out = real_colours(net, xyz, vd, *a)
            self.coloured.append((host(xyz), host(out)))
            return out
        monkeypatch.setattr(pn, "tsdf_fuse", tsdf_fuse)
        monkeypatch.setattr(pn, "paint_vertices", paint_vertices)
        monkeypatch.setattr(urecon, "_colours", colours)


def call(net, renderer, poses, seed=7, **kw):
    from util import recon as urecon
    torch.manual_seed(seed)
    return urecon.fuse_views(net, renderer, poses, W, H, FOCAL, C2["z_near"], C2["z_far"], c1=LO, c2=HI, reso=RESO,
                             ray_batch_size=BS, **kw)


def rerender_rgb(net, renderer, poses, gpus, seed):
    """The kept pass's rgb, rendered again as fuse_views renders it."""
    import pnr_native as pn
    render_par = renderer.bind_parallel(net, gpus)
    V = poses.shape[0]
    rgb = torch.empty(V * H * W, 3, device="cuda")
    torch.manual_seed(seed)
    with torch.no_grad():
        for first in range(0, V * H * W, BS):
            n = min(BS, V * H * W - first)
            rays = pn.gen_rays(poses, W, H, FOCAL, FOCAL, W / 2, H / 2, C2["z_near"], C2["z_far"], first, n)
            rgb[first:first + n] = render_par(rays[None], want_weights=True)["fine"]["rgb"][0]
    return rgb.view(V, H, W, 3).cpu().numpy()


def painted_checks(monkeypatch, gpus=None):
    net, renderer, poses = c2_scene()
    spy = _Spy(monkeypatch)
    call(net, renderer, poses, gpus=gpus)
    m = float(np.clip(np.median(spy.fused[-1][1]), 0.05, 1.0))           # an opacity level the scene crosses
    verts, tris, normals, rgb = call(net, renderer, poses, gpus=gpus, min_opacity=m, return_colors=True,
                                     colors="views")
    assert len(spy.painted) == 1
    (xyz, nrm, rgb_map, depth, opacity, p, *args), (col, weight) = spy.painted[0]
    # the kernel saw the returned vertices and normals, the maps the fusion saw and the call's own parameters
    bits(xyz, verts)
    bits(nrm, normals)
    bits(depth, spy.fused[-1][0])
    bits(opacity, spy.fused[-1][1])
    assert rgb_map.shape == (poses.shape[0], H, W, 3) and np.array_equal(p, poses.cpu().numpy())
    h = (np.array(HI) - np.array(LO)) / (np.array(RESO) - 1)
    assert tuple(args) == (FOCAL, FOCAL, W / 2, H / 2, 3.0 * np.sqrt(3.0) * float(np.abs(h).max()), m,
                           1.0 if renderer.white_bkgd else 0.0)
    want, want_w = paint.paint_vertices(xyz, nrm, rgb_map, depth, opacity, p, *args)
    bits(col, want)
    bits(weight, want_w)
    painted = weight > 0
    print(f"{painted.sum()} of {len(verts)} vertices painted, {(~painted).sum()} from the field")
    assert painted.any()
    bits(rgb[painted], want[painted])
    # the rest: _colours on just their rows, as it returned them
    if (~painted).any():
        assert len(spy.coloured) == 1 and len(spy.coloured[0][0]) == (~painted).sum()
        bits(rgb[~painted], spy.coloured[0][1])
    else:
        assert spy.coloured == []
    assert rgb.dtype == np.float32 and rgb.shape == verts.shape
    assert np.isfinite(rgb).all() and rgb.min() >= 0.0 and rgb.max() <= 1.0
    # the rgb map is the renderer's, in render_frames' pixel order (a re-render: equal up to the engine's low bits)
    close = np.abs(rerender_rgb(net, renderer, poses, gpus, 7) - rgb_map).max(-1) <= 1e-3
    print(f"re-rendered pixels within 1e-3: {close.mean():.4f}")
    assert close.mean() >= 0.99


def test_fuse_views_paints_on_c2_scene(monkeypatch):
    painted_checks(monkeypatch)


def test_fuse_views_paints_two_shards_on_one_gpu(monkeypatch):
    painted_checks(monkeypatch, gpus=[0, 0])


def test_default_colours_unchanged(monkeypatch):
    """colors="field" is the default: the same call gives the same bits with or without it (on the SIMT engine, whose
    renders repeat bit for bit)."""
    from render import NeRFRenderer
    net, _, _ = c2_net("simt")
    renderer = NeRFRenderer(n_coarse=C2["n_coarse"], n_fine=C2["n_fine"], n_fine_depth=C2["n_fine_depth"],
                            white_bkgd=C2["white_bkgd"]).cuda()
    poses = views(10, (C2["z_near"] + C2["z_far"]) / 2, phi=-10.0).cuda()
    spy = _Spy(monkeypatch)
    call(net, renderer, poses)
    m = float(np.clip(np.median(spy.fused[-1][1]), 0.05, 1.0))           # an opacity level the scene crosses
    plain = call(net, renderer, poses, min_opacity=m)
    default = call(net, renderer, poses, min_opacity=m, return_colors=True)
    field = call(net, renderer, poses, min_opacity=m, return_colors=True, colors="field")
    assert len(default[1]) > 100
    for a, b in zip(default, field):
        bits(a, b)
    bits(plain[0], default[0])
    bits(plain[1], default[1])


def test_colours_refusals():
    net, renderer, poses = c2_scene()
    with pytest.raises(ValueError, match="colors"):
        call(net, renderer, poses, return_colors=True, colors="rendered")
    with pytest.raises(ValueError, match="return_colors"):
        call(net, renderer, poses, colors="views")
