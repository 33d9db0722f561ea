"""TSDF fusion on the H100: pnr_tsdf_fuse bit for bit against the numpy oracle (oracle/pnr_recon_fuse.py) at 128^3 with
64 analytic views, and `util.recon.fuse_views` on the C2 scene.  The tensor engine's sigma differs in its low bits from
run to run, so the fused volume and the mesh of a call are checked against the oracle applied to the depth and opacity
maps captured in that same call; that those maps are the renderer's is checked against a re-render under the same
seed."""
import os

import numpy as np
import pytest
import torch

import golden_util as gu
from fuse_util import fuse, index_to_world, sphere_maps, views
from recon_util import recon
from test_gpu_recon import c2_net

attrs = gu.load_by_path("pnr_recon_attrs_oracle", os.path.join(gu.ROOT, "oracle", "pnr_recon_attrs.py"))

pytestmark = pytest.mark.gpu

C2 = gu.synth.CONFIGS["c2"]


def bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_kernel_bit_equal_at_128_cubed_with_64_views():
    import pnr_native as pn
    poses = views(62, 3.0)                                  # 64 views
    depth, opacity = sphere_maps(poses, 96, 96, 160.0, 0.5)
    lo, hi, reso, trunc = (-1.0,) * 3, (1.0,) * 3, (128,) * 3, 0.05
    args = (160.0, 160.0, 48.0, 48.0, lo, hi, reso, trunc, 0.5)
    dev = [torch.from_numpy(x).cuda() for x in (depth, opacity)] + [poses.cuda()]
    got = pn.tsdf_fuse(*dev, *args).cpu().numpy()
    want = fuse.tsdf_fuse(depth, opacity, poses.numpy(), *args)
    bits(got, want)
    bits(pn.tsdf_fuse(*dev, *args).cpu().numpy(), got)     # deterministic
    v, t = recon.marching_cubes(-got, 0.0)
    assert recon.is_closed_oriented(t) and recon.components(t) == 1


class _Spy:
    """Records the inputs and output of every pnr_native.tsdf_fuse call and the volumes handed to marching cubes."""

    def __init__(self, monkeypatch):
        import pnr_native as pn
        self.fused, self.vols = [], []
        real_fuse, real_mc = pn.tsdf_fuse, pn.marching_cubes

        def tsdf_fuse(depth, opacity, poses, *a):
            out = real_fuse(depth, opacity, poses, *a)
            self.fused.append(([x.cpu().numpy().copy() for x in (depth, opacity, poses)], a, out.cpu().numpy().copy()))
            return out

        def mc(vol, iso, **kw):
            self.vols.append(vol.cpu().numpy().copy())
            return real_mc(vol, iso, **kw)
        monkeypatch.setattr(pn, "tsdf_fuse", tsdf_fuse)
        monkeypatch.setattr(pn, "marching_cubes", mc)


W = H = 32
FOCAL = C2["focal"] * W / C2["W"]
LO, HI, RESO = [-0.6] * 3, [0.6] * 3, [40, 36, 44]
BS = 3000                                                   # ragged last batch


def c2_scene():
    from render import NeRFRenderer
    net, _, _ = c2_net("tc")
    renderer = NeRFRenderer(n_coarse=C2["n_coarse"], n_fine=C2["n_fine"], n_fine_depth=C2["n_fine_depth"],
                            white_bkgd=C2["white_bkgd"]).cuda()
    poses = views(10, (C2["z_near"] + C2["z_far"]) / 2, phi=-10.0).cuda()
    return net, renderer, poses


def rerender(net, renderer, poses, gpus, seed):
    """The depth and opacity maps, rendered again as fuse_views renders them."""
    import pnr_native as pn
    render_par = renderer.bind_parallel(net, gpus)
    V = poses.shape[0]
    depth, opacity = torch.empty(V * H * W, device="cuda"), torch.empty(V * H * W, device="cuda")
    torch.manual_seed(seed)
    with torch.no_grad():
        for first in range(0, V * H * W, BS):
            n = min(BS, V * H * W - first)
            rays = pn.gen_rays(poses, W, H, FOCAL, FOCAL, W / 2, H / 2, C2["z_near"], C2["z_far"], first, n)
            best = render_par(rays[None], want_weights=True)["fine"]
            depth[first:first + n], opacity[first:first + n] = best["depth"][0], best["weights"][0].sum(-1)
    return depth.view(V, H, W).cpu().numpy(), opacity.view(V, H, W).cpu().numpy()


def fused_checks(net, renderer, poses, monkeypatch, gpus=None, return_colors=False):
    """fuse_views against the oracle of the maps captured in the same call -> (result, tsdf)."""
    from util import recon as urecon
    spy = _Spy(monkeypatch)
    seed = 7
    kw = dict(c1=LO, c2=HI, reso=RESO, ray_batch_size=BS, gpus=gpus)
    torch.manual_seed(seed)
    urecon.fuse_views(net, renderer, poses, W, H, FOCAL, C2["z_near"], C2["z_far"], **kw)
    m = float(np.clip(np.median(spy.fused[-1][0][1]), 0.05, 1.0))        # an opacity level the scene crosses
    net.train()
    renderer.train()
    torch.manual_seed(seed)
    res = urecon.fuse_views(net, renderer, poses, W, H, FOCAL, C2["z_near"], C2["z_far"], min_opacity=m,
                            return_colors=return_colors, **kw)
    assert net.training and renderer.training                            # restored
    net.eval()
    renderer.eval()
    (depth, opacity, p), a, tsdf = spy.fused[-1]
    assert depth.shape == opacity.shape == (poses.shape[0], H, W) and np.array_equal(p, poses.cpu().numpy())
    assert a[:4] == (FOCAL, FOCAL, W / 2, H / 2) and a[-1] == m
    bits(tsdf, fuse.tsdf_fuse(depth, opacity, p, *a))
    assert (tsdf > 0).any() and (tsdf < 0).any()
    bits(spy.vols[-1], -tsdf)
    rv, rt = recon.marching_cubes(-tsdf, 0.0)
    assert len(rt) > 100, len(rt)
    bits(res[0], index_to_world(rv, LO, HI, RESO))
    bits(res[1], rt)
    # the maps are the renderer's, in render_frames' pixel order (a re-render: equal up to the engine's low bits)
    rd, ro = rerender(net, renderer, poses, gpus, seed)
    close = (np.abs(rd - depth) <= 1e-3) & (np.abs(ro - opacity) <= 1e-3)
    print(f"re-rendered pixels within 1e-3: {close.mean():.4f}")
    assert close.mean() >= 0.99
    return res, tsdf


def test_fuse_views_on_c2_scene(monkeypatch):
    net, renderer, poses = c2_scene()
    fused_checks(net, renderer, poses, monkeypatch)


def test_fuse_views_two_shards_on_one_gpu(monkeypatch):
    net, renderer, poses = c2_scene()
    fused_checks(net, renderer, poses, monkeypatch, gpus=[0, 0])


def test_fuse_views_colours(monkeypatch):
    net, renderer, poses = c2_scene()
    (verts, tris, normals, rgb), tsdf = fused_checks(net, renderer, poses, monkeypatch, return_colors=True)
    assert normals.dtype == np.float64 and normals.shape == verts.shape
    assert np.abs(np.linalg.norm(normals, axis=1) - 1.0).max() < 1e-12
    bits(normals, attrs.vertex_attrs(-tsdf, 0.0, LO, HI)[0])
    assert rgb.dtype == np.float32 and rgb.shape == verts.shape
    assert np.isfinite(rgb).all() and rgb.min() >= 0.0 and rgb.max() <= 1.0


def test_fuse_views_refusals():
    import gpu_util
    from model import make_model
    from util import recon as urecon
    net, renderer, poses = c2_scene()
    call = lambda n=net, p=poses, **kw: urecon.fuse_views(n, renderer, p, W, H, FOCAL, 0.8, 1.8,  # noqa: E731
                                                          reso=[8, 8, 8], **kw)
    net.train()
    renderer.train()
    net.num_objs = 2
    try:
        with pytest.raises(RuntimeError, match="one object"):
            call()
    finally:
        net.num_objs = 1
    for bad in ([1, 0], [3], []):
        with pytest.raises(ValueError, match="gpus"):
            call(gpus=bad)
    with pytest.raises(ValueError, match="poses"):
        call(p=poses[:0])
    with pytest.raises(ValueError, match="min_opacity"):
        call(min_opacity=0.0)
    with pytest.raises(ValueError, match="trunc"):
        call(trunc=-1.0)
    assert net.training and renderer.training
    cpu_net = make_model(gpu_util.model_conf(C2["d_hidden"]))
    cpu_net.num_objs = 1
    with pytest.raises(RuntimeError, match="CUDA only"):
        call(n=cpu_net)
