"""
ORACLE TOOLING -- generates tests/golden/grad_aux_{tiny,sb2_d}.npz by running the UNMODIFIED reference in grad mode
(imported through oracle/ref_harness.py) on CPU, with the inputs, noise and rgb target of make_golden.py's
grad_fixture.

    python oracle/make_golden_aux.py            # writes both fixtures
    python oracle/make_golden_aux.py --check    # additionally compares oracle/pnr_aux_backward.py with the reference

Run where a reference checkout is readable (not on the GPU box).  The loss covers every output of the renderer:
train.py's rgb MSEs + the reference's own alpha loss (model/loss.py AlphaLossNV2, built by get_alpha_loss from a
`loss.alpha` block with init_epoch = 0) on fine.weights.sum(-1) + MSE of both depths to a seeded target depth + a small
term on coarse.weights.  The fixture records the upstream gradient of each of the six outputs (retain_grad), so the
tests need no loss code, and the reference's gradients of every MLP parameter and of the latent.
"""
import argparse
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


def aux_grad_fixture(name, check, lambda_alpha=1.0, lambda_depth=1.0, lambda_weights=0.1):
    cs = mg.CASES[name]
    inp = mg.case_inputs(name, cs)
    net, renderer = ref_harness.build_reference(
        cs["d_hidden"], inp["wc"], inp["wf"], cs["n_coarse"], cs["n_fine"], cs["n_fine_depth"],
        white_bkgd=cs["white_bkgd"], eval_batch_size=cs["eval_batch_size"])
    from model import loss as ref_loss     # the reference's package (ref_harness.import_reference put it on sys.path)
    alpha_loss = ref_loss.get_alpha_loss(ref_harness.DictConf(
        dict(lambda_alpha=lambda_alpha, clamp_alpha=100, init_epoch=0)))
    latent = inp["latent"].clone().requires_grad_(True)
    ref_harness.set_scene(net, latent, inp["src_poses"], inp["focal"], inp["c"], cs["W"], cs["H"])
    g = torch.Generator().manual_seed(inp["seed"] + 6)
    gt = torch.rand(cs["SB"], cs["B"], 3, generator=g)          # grad_fixture's target
    g2 = torch.Generator().manual_seed(inp["seed"] + 7)
    depth_gt = cs["z_near"] + (cs["z_far"] - cs["z_near"]) * torch.rand(cs["SB"], cs["B"], generator=g2)
    torch.manual_seed(inp["seed"] + 4)
    out = renderer(net, inp["rays"], want_weights=True)
    outs = {k: out[k.split(".")[0]][k.split(".")[1]] for k in OUTPUTS}
    for t in outs.values():
        t.retain_grad()
    crit = torch.nn.MSELoss()
    rgb_loss = crit(out.coarse.rgb, gt) * 1.0 + crit(out.fine.rgb, gt) * 1.0
    a_loss = alpha_loss(out.fine.weights.sum(-1))
    depth_loss = lambda_depth * (crit(out.coarse.depth, depth_gt) + crit(out.fine.depth, depth_gt))
    weights_loss = lambda_weights * out.coarse.weights.square().mean()
    loss = rgb_loss + a_loss + depth_loss + weights_loss
    loss.backward()
    rec = dict(loss=np.array(loss.item()), rgb_gt=gt.numpy(), depth_gt=depth_gt.numpy(),
               alpha_loss=np.array(a_loss.item()), g_latent=latent.grad.numpy())
    for k, t in outs.items():
        rec["up/" + k] = t.grad.numpy()
    for k, p in net.mlp_coarse.named_parameters():
        rec["gc/" + k] = p.grad.numpy()
    if net.mlp_fine is not None:
        for k, p in net.mlp_fine.named_parameters():
            rec["gf/" + k] = p.grad.numpy()
    path = os.path.join(mg.GOLD, "grad_aux_" + name + ".npz")
    np.savez_compressed(path, **rec)
    print(f"grad_aux_{name}: wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB), loss {loss.item():.6f} "
          f"(alpha {a_loss.item():.6f})")
    if check:
        ab = _load("pnr_aux_backward", os.path.join(HERE, "pnr_aux_backward.py"))
        state = mg.oracle.encode_state(inp["src_poses"].reshape(-1, 4, 4), inp["focal"], inp["c"], cs["W"], cs["H"])
        up = {"d_" + k.split(".")[1] + "_" + k.split(".")[0]: t.grad.reshape(cs["SB"] * cs["B"], -1).squeeze(-1)
              for k, t in outs.items()}
        g_c, g_f, d_lat = ab.render_backward(inp["rays"], inp["noise"], state, inp["latent"], inp["wc"], inp["wf"],
                                             cs["NS"], cs["n_coarse"], cs["n_fine"], cs["n_fine_depth"], up,
                                             white_bkgd=cs["white_bkgd"])
        worst = 0.0
        for pre, gd in (("gc/", g_c), ("gf/", g_f or {})):
            for k, v in gd.items():
                ref = torch.from_numpy(rec[pre + k])
                worst = max(worst, ((v - ref).abs().max() / (ref.abs().max() + 1e-12)).item())
        print(f"   check: render_backward worst rel {worst:.2e}, latent "
              f"{((d_lat - latent.grad).abs().max() / latent.grad.abs().max()).item():.2e}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    os.makedirs(mg.GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for name in ("tiny", "sb2_d"):
        aux_grad_fixture(name, a.check)
