"""Helpers for the -m gpu parity tests: build the product model for a golden case and run
it through the public classes / the C ABI on cuda:0."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pixel-nerf_b200", "src")
if SRC not in sys.path:
    sys.path.insert(0, SRC)


def model_conf(d_hidden, use_first_pool=True):
    from util import hocon
    mlp = dict(type="resnet", n_blocks=5, d_hidden=d_hidden, combine_layer=3, combine_type="average")
    return hocon.from_dict(dict(
        use_encoder=True, use_global_encoder=False, use_xyz=True, use_code=True,
        code=dict(num_freqs=6, freq_factor=1.5, include_input=True),
        use_viewdirs=True, use_code_viewdirs=False, mlp_coarse=dict(mlp), mlp_fine=dict(mlp),
        encoder=dict(backbone="resnet34", pretrained=False, num_layers=4, use_first_pool=use_first_pool)))


def build_net(case, device="cuda:0", engine="auto"):
    from model import make_model
    cfg = case["cfg"]
    net = make_model(model_conf(cfg["d_hidden"]))
    net.mlp_coarse.load_state_dict(case["wc"])
    if case["wf"] is not None:
        net.mlp_fine.load_state_dict(case["wf"])
    else:
        net.mlp_fine = None
    net = net.to(device).eval()
    net.engine = engine
    c = case["c"].to(device) if case["c"] is not None else None
    net.set_scene(case["latent"].to(device), case["src_poses"].to(device), case["focal"].to(device), c,
                  cfg["W"], cfg["H"])
    return net


def build_renderer(case, depth_std=0.01):
    from render import NeRFRenderer
    cfg = case["cfg"]
    r = NeRFRenderer(n_coarse=cfg["n_coarse"], n_fine=cfg["n_fine"], n_fine_depth=cfg["n_fine_depth"],
                     depth_std=depth_std, white_bkgd=bool(cfg["white_bkgd"]), eval_batch_size=cfg["eval_batch_size"])
    return r.eval()


def render_case_cuda(case, engine="auto", device="cuda:0", depth_std=0.01):
    """Fused render of a golden case with the fixture's noise -> dict like oracle.render."""
    net = build_net(case, device, engine)
    renderer = build_renderer(case, depth_std)
    rays = case["rays"].to(device)
    noise = {k: v.to(device) for k, v in case["noise"].items()}
    with torch.no_grad():
        out = renderer._forward_fused(net, rays, want_weights=True, noise_in=noise, want_z=True)
    res = {}
    for name in ("coarse", "fine"):
        if name in out:
            o = out[name]
            K = o.weights.shape[-1]
            res[name] = dict(rgb=o.rgb.reshape(-1, 3), depth=o.depth.reshape(-1), weights=o.weights.reshape(-1, K),
                             z=o.z.reshape(-1, K))
    return res
