"""
ORACLE TOOLING -- generates tests/golden/grad_cam_{tiny,sb2_d,sb2_d_clamp}.npz by running the UNMODIFIED reference in
grad mode (imported through oracle/ref_harness.py) on CPU, on the inputs and noise of make_golden.py's cases, with the
rays, the camera-to-world source poses, focal, c and the latent all requiring grad.

    python oracle/make_golden_cam.py

Run where a reference checkout is readable (not on the GPU box).  The loss is make_golden_aux.py's (rgb MSEs, the
reference's alpha loss, depth MSEs, a coarse-weights term).  Each fixture records the upstream gradient of each of the six
outputs (retain_grad), so tests replay it with no loss code, and the reference's gradients of the rays, the c2w poses,
focal, c, every MLP parameter and the latent.  `sb2_d_clamp` is sb2_d with depth_std = 0.6, so that many depth-centred
fine samples are clamped to near or far (nerf.py:160) -- with the shipped 0.01 none are.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mg = _load("pnr_make_golden", os.path.join(HERE, "make_golden.py"))   # CASES, case_inputs, GOLD, ref_harness
ref_harness = mg.ref_harness

OUTPUTS = ("coarse.rgb", "coarse.depth", "coarse.weights", "fine.rgb", "fine.depth", "fine.weights")
FIXTURES = {"tiny": ("tiny", 0.01), "sb2_d": ("sb2_d", 0.01), "sb2_d_clamp": ("sb2_d", 0.6)}


def cam_grad_fixture(fixture, lambda_alpha=1.0, lambda_depth=1.0, lambda_weights=0.1):
    name, depth_std = FIXTURES[fixture]
    cs = mg.CASES[name]
    inp = mg.case_inputs(name, cs)
    net, renderer = ref_harness.build_reference(
        cs["d_hidden"], inp["wc"], inp["wf"], cs["n_coarse"], cs["n_fine"], cs["n_fine_depth"], depth_std=depth_std,
        white_bkgd=cs["white_bkgd"], eval_batch_size=cs["eval_batch_size"])
    from model import loss as ref_loss     # the reference's package (ref_harness.import_reference put it on sys.path)
    alpha_loss = ref_loss.get_alpha_loss(ref_harness.DictConf(
        dict(lambda_alpha=lambda_alpha, clamp_alpha=100, init_epoch=0)))
    latent = inp["latent"].clone().requires_grad_(True)
    poses = inp["src_poses"].clone().requires_grad_(True)
    focal = torch.as_tensor(inp["focal"], dtype=torch.float32).clone().requires_grad_(True)
    c = inp["c"] if inp["c"] is not None else torch.tensor([[cs["W"] * 0.5, cs["H"] * 0.5]])  # = the default centre
    c = torch.as_tensor(c, dtype=torch.float32).clone().requires_grad_(True)
    rays = inp["rays"].clone().requires_grad_(True)
    ref_harness.set_scene(net, latent, poses, focal, c, cs["W"], cs["H"])
    g = torch.Generator().manual_seed(inp["seed"] + 6)
    gt = torch.rand(cs["SB"], cs["B"], 3, generator=g)
    g2 = torch.Generator().manual_seed(inp["seed"] + 7)
    depth_gt = cs["z_near"] + (cs["z_far"] - cs["z_near"]) * torch.rand(cs["SB"], cs["B"], generator=g2)
    torch.manual_seed(inp["seed"] + 4)                                # the draws of the case's stored noise
    out = renderer(net, rays, want_weights=True)
    outs = {k: out[k.split(".")[0]][k.split(".")[1]] for k in OUTPUTS}
    for t in outs.values():
        t.retain_grad()
    crit = torch.nn.MSELoss()
    loss = (crit(out.coarse.rgb, gt) + crit(out.fine.rgb, gt) + alpha_loss(out.fine.weights.sum(-1))
            + lambda_depth * (crit(out.coarse.depth, depth_gt) + crit(out.fine.depth, depth_gt))
            + lambda_weights * out.coarse.weights.square().mean())
    loss.backward()
    rec = dict(loss=np.array(loss.item()), depth_std=np.array(depth_std), c=c.detach().numpy(),
               g_rays=rays.grad.numpy(), g_poses=poses.grad.numpy(), g_focal=focal.grad.numpy(), g_c=c.grad.numpy(),
               g_latent=latent.grad.numpy())
    for k, t in outs.items():
        rec["up/" + k] = t.grad.numpy()
    for k, p in net.mlp_coarse.named_parameters():
        rec["gc/" + k] = p.grad.numpy()
    for k, p in net.mlp_fine.named_parameters():
        rec["gf/" + k] = p.grad.numpy()
    path = os.path.join(mg.GOLD, "grad_cam_" + fixture + ".npz")
    np.savez_compressed(path, **rec)
    print(f"grad_cam_{fixture}: wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB), loss {loss.item():.6f}")


if __name__ == "__main__":
    os.makedirs(mg.GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for f in FIXTURES:
        cam_grad_fixture(f)
