"""Drop-in smoke: the call sequence of the reference's eval/gen_video.py (lines 103-222: make_model from a conf file,
NeRFRenderer.from_conf, bind_parallel(simple_output=True), util.pose_spherical / util.gen_rays, mutate
n_coarse / n_fine after construction, net.encode, loop over torch.split(rays, ray_batch_size)) against this package."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "pixel-nerf_b200")
pytestmark = pytest.mark.gpu


def test_gen_video_call_sequence():
    sys.path.insert(0, os.path.join(PKG, "src"))
    import numpy as np
    import util
    from model import make_model
    from render import NeRFRenderer

    torch.manual_seed(0)                                 # the scene must not depend on which tests ran before
    conf = util.hocon.parse_file(os.path.join(PKG, "conf", "exp", "srn.conf"))
    conf.put("model.encoder.pretrained", False)          # no network in the test image
    device = util.get_cuda(0)
    net = make_model(conf["model"]).to(device=device)
    # the reference zero-initialises fc_1, which would hide half of the network: perturb like a trained model
    with torch.no_grad():
        for mlp in (net.mlp_coarse, net.mlp_fine):
            for blk in mlp.blocks:
                blk.fc_1.weight.normal_(0, 0.03)
            mlp.lin_out.bias[3] = 2.0
    ray_batch_size = 3000
    renderer = NeRFRenderer.from_conf(conf["renderer"], lindisp=False, eval_batch_size=ray_batch_size).to(device=device)
    render_par = renderer.bind_parallel(net, [0], simple_output=True).eval()

    W = H = 48
    z_near, z_far = 0.8, 1.8
    focal = torch.tensor(49.0, device=device)
    NV = 3
    images = torch.rand(2, 3, H, W) * 2 - 1                    # two source views
    poses = torch.stack([util.pose_spherical(a, -30.0, 1.3) for a in (0.0, 40.0)])
    render_poses = torch.stack([util.pose_spherical(angle, -10.0, 1.3)
                                for angle in np.linspace(-180, 180, NV + 1)[:-1]], 0)
    render_rays = util.gen_rays(render_poses, W, H, focal, z_near, z_far).to(device=device)
    if renderer.n_coarse < 64:                                 # gen_video.py:192-195 mutates attributes
        renderer.n_coarse = 64
        renderer.n_fine = 128
    with torch.no_grad():
        net.encode(images.unsqueeze(0).to(device=device), poses.unsqueeze(0).to(device=device), focal)
        all_rgb = []
        for rays in torch.split(render_rays.view(-1, 8), ray_batch_size, dim=0):
            rgb, _depth = render_par(rays[None])
            all_rgb.append(rgb[0])
        frames = torch.clamp(torch.cat(all_rgb).view(-1, H, W, 3), 0.0, 1.0)
    assert frames.shape == (NV, H, W, 3) and torch.isfinite(frames).all()
    assert frames.std() > 1e-3                                  # not a constant image
    # fused inference == the composed-torch (autograd) path on a slice, same seed -> same samples on this device
    sub = render_rays.view(-1, 8)[1000:1256][None]
    torch.manual_seed(5)
    with torch.no_grad():
        a = renderer(net, sub).fine.rgb
    torch.manual_seed(5)
    b = renderer._forward_torch(type("F", (), {"use_viewdirs": True, "__call__": lambda s, x, coarse=True, viewdirs=None:
                                              net._forward_autograd(x, coarse, viewdirs)})(), sub, False).fine.rgb
    flipped = (a - b).abs().max(-1).values > 1e-3
    assert flipped.float().mean() < 0.05
    assert (a - b)[~flipped].abs().max() < 2e-4
