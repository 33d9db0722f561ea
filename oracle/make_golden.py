"""
ORACLE TOOLING -- generates tests/golden/*.npz by running the UNMODIFIED reference
(/root/reference/src, imported through oracle/ref_harness.py) on CPU.

    python oracle/make_golden.py            # writes every fixture
    python oracle/make_golden.py --check    # additionally asserts pnr_oracle == reference

Run in the build container only (the GPU box has no /root/reference).  Fixtures hold the
inputs needed to replay a case (or the seeds to regenerate them with
pixel-nerf_b200/synth.py plus a checksum guarding against RNG drift) and the reference's
outputs.  The reference has no tests/golden vectors of its own (SURVEY.md section 4);
these files are what pins the oracle.
"""
import argparse
import importlib.util
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import ref_harness  # noqa: E402


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


synth = _load("pnr_synth", os.path.join(ROOT, "pixel-nerf_b200", "synth.py"))
oracle = _load("pnr_oracle", os.path.join(HERE, "pnr_oracle.py"))

GOLD = os.path.join(ROOT, "tests", "golden")

# name -> case description.  store_weights: small MLPs are stored verbatim, big ones are
# regenerated from the seed at test time (checksum stored).
CASES = {
    "tiny": dict(SB=1, NS=2, W=16, H=16, Hl=8, Wl=8, focal=17.0, c=None, z_near=0.8, z_far=1.8,
                 d_hidden=32, n_coarse=8, n_fine=8, n_fine_depth=4, B=24, white_bkgd=True,
                 eval_batch_size=50000, store_weights=True, fine_mlp=True),
    "tiny_sb2": dict(SB=2, NS=2, W=16, H=12, Hl=6, Wl=8, focal=[15.0, 19.0], c=None, z_near=0.8,
                     z_far=1.8, d_hidden=32, n_coarse=8, n_fine=6, n_fine_depth=2, B=10,
                     white_bkgd=False, eval_batch_size=37, store_weights=True, fine_mlp=False),
    # same shape as tiny_sb2 (whose random MLP happens to give sigma = 0 everywhere: the all-transparent edge case)
    # but with a visible object, so that per-object indexing of rays / latents / focal shows up in rgb and weights
    "sb2_d": dict(SB=2, NS=2, W=16, H=12, Hl=6, Wl=8, focal=[15.0, 19.0], c=None, z_near=0.8,
                      z_far=1.8, d_hidden=32, n_coarse=8, n_fine=6, n_fine_depth=2, B=12,
                      white_bkgd=False, eval_batch_size=37, store_weights=True, fine_mlp=True),
    "ns1_coarse_only": dict(SB=1, NS=1, W=16, H=16, Hl=8, Wl=8, focal=16.4, c=None, z_near=0.8,
                            z_far=1.8, d_hidden=128, n_coarse=16, n_fine=0, n_fine_depth=0, B=32,
                            white_bkgd=True, eval_batch_size=50000, store_weights=False,
                            fine_mlp=False),
    "c2_small": dict(SB=1, NS=2, W=32, H=32, Hl=16, Wl=16, focal=32.8, c=None, z_near=0.8,
                     z_far=1.8, d_hidden=512, n_coarse=64, n_fine=32, n_fine_depth=16, B=48,
                     white_bkgd=True, eval_batch_size=50000, store_weights=False, fine_mlp=True),
    "c3_small": dict(SB=1, NS=1, W=32, H=32, Hl=16, Wl=16, focal=35.0, c=None, z_near=1.2,
                     z_far=4.0, d_hidden=512, n_coarse=64, n_fine=16, n_fine_depth=8, B=32,
                     white_bkgd=True, eval_batch_size=50000, store_weights=False, fine_mlp=True),
    "c4_small": dict(SB=1, NS=3, W=40, H=30, Hl=15, Wl=20, focal=[36.0, 36.5], c=[20.5, 14.5],
                     z_near=0.1, z_far=5.0, d_hidden=512, n_coarse=96, n_fine=48, n_fine_depth=16,
                     B=16, white_bkgd=False, eval_batch_size=50000, store_weights=False,
                     fine_mlp=True),
}


def case_inputs(name, cs):
    """Deterministic inputs of a case (shared with tests through the same code path:
    tests call tests/golden_util.py which mirrors this using the stored seeds)."""
    seed = sum(ord(ch) for ch in name)  # stable across processes (unlike hash())
    SB, NS = cs["SB"], cs["NS"]
    r = (cs["z_near"] + cs["z_far"]) * 0.5
    src = torch.stack([torch.stack([synth.pose_spherical(40.0 * v + 25.0 * o, -30.0, r)
                                    for v in range(NS)]) for o in range(SB)])  # (SB,NS,4,4)
    latent = synth.make_latent(seed, SB * NS, cs["Hl"], cs["Wl"])
    focal = torch.tensor(cs["focal"], dtype=torch.float32)
    if focal.dim() == 1 and SB == 1:
        focal = focal[None]          # (1,2): one fx,fy pair
    c = None if cs["c"] is None else torch.tensor(cs["c"], dtype=torch.float32)[None]
    # target rays: orbit views, random pixel subset so that off-image projections occur
    tgt = torch.stack([synth.pose_spherical(100.0 + 70.0 * o, -10.0 - 5 * o, r) for o in range(SB)])
    f_scalar = float(torch.as_tensor(cs["focal"]).reshape(-1)[0])
    all_rays = synth.gen_rays(tgt, cs["W"], cs["H"], f_scalar, cs["z_near"], cs["z_far"])
    g = torch.Generator().manual_seed(seed + 1)
    pix = torch.randint(0, cs["W"] * cs["H"], (SB, cs["B"]), generator=g)
    rays = torch.stack([all_rays[o].reshape(-1, 8)[pix[o]] for o in range(SB)])  # (SB,B,8)
    wc = synth.make_mlp_weights(seed + 2, cs["d_hidden"])
    wf = synth.make_mlp_weights(seed + 3, cs["d_hidden"]) if cs["fine_mlp"] else None
    noise = synth.draw_noise(seed + 4, SB * cs["B"], cs["n_coarse"], cs["n_fine"], cs["n_fine_depth"])
    return dict(seed=seed, src_poses=src, latent=latent, focal=focal, c=c, rays=rays, wc=wc, wf=wf,
                noise=noise)


def run_case(name, cs, check):
    inp = case_inputs(name, cs)
    net, renderer = ref_harness.build_reference(
        cs["d_hidden"], inp["wc"], inp["wf"], cs["n_coarse"], cs["n_fine"], cs["n_fine_depth"],
        white_bkgd=cs["white_bkgd"], eval_batch_size=cs["eval_batch_size"])
    focal_arg = inp["focal"]
    ref_harness.set_scene(net, inp["latent"], inp["src_poses"], focal_arg, inp["c"], cs["W"], cs["H"])
    out, zs = ref_harness.run_reference_render(net, renderer, inp["rays"], inp["seed"] + 4)

    # bare field evaluation on scattered points (some behind cameras / far off-image)
    g = torch.Generator().manual_seed(inp["seed"] + 5)
    P = 40
    xyz = (torch.rand(cs["SB"], P, 3, generator=g) - 0.5) * 3.0
    vdir = torch.nn.functional.normalize(torch.randn(cs["SB"], P, 3, generator=g), dim=-1)
    with torch.no_grad():
        f_c = net(xyz, coarse=True, viewdirs=vdir)
        f_f = net(xyz, coarse=False, viewdirs=vdir)

    rec = dict(
        src_poses=inp["src_poses"].numpy(), latent=inp["latent"].numpy(),
        focal=inp["focal"].numpy(), rays=inp["rays"].numpy(),
        has_c=np.array(inp["c"] is not None), c=(inp["c"].numpy() if inp["c"] is not None else np.zeros(1)),
        seed=np.array(inp["seed"]),
        field_xyz=xyz.numpy(), field_dirs=vdir.numpy(), field_coarse=f_c.numpy(), field_fine=f_f.numpy(),
        ref_state_poses=net.poses.numpy(), ref_state_focal=net.focal.numpy(), ref_state_c=net.c.numpy(),
        coarse_rgb=out.coarse.rgb.numpy(), coarse_depth=out.coarse.depth.numpy(),
        coarse_weights=out.coarse.weights.numpy(), z_coarse=zs[0].numpy(),
        wc_checksum=np.array(synth.weights_checksum(inp["wc"])),
        wf_checksum=np.array(synth.weights_checksum(inp["wf"]) if inp["wf"] is not None else 0.0),
    )
    for k, v in inp["noise"].items():
        rec["noise_" + k] = v.numpy()
    if cs["n_fine"] > 0:
        rec.update(fine_rgb=out.fine.rgb.numpy(), fine_depth=out.fine.depth.numpy(),
                   fine_weights=out.fine.weights.numpy(), z_fine=zs[1].numpy())
    if cs["store_weights"]:
        for k, v in inp["wc"].items():
            rec["wc/" + k] = v.numpy()
        if inp["wf"] is not None:
            for k, v in inp["wf"].items():
                rec["wf/" + k] = v.numpy()
    for k, v in cs.items():
        if k in ("focal", "c"):
            continue
        rec["cfg_" + k] = np.array(v)
    path = os.path.join(GOLD, name + ".npz")
    np.savez_compressed(path, **rec)
    print(f"{name}: wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")

    if check:
        state = oracle.encode_state(inp["src_poses"].reshape(-1, 4, 4), inp["focal"], inp["c"],
                                    cs["W"], cs["H"])
        assert torch.equal(state["poses"], net.poses), "poses"
        res = oracle.render(inp["rays"], inp["noise"], state, inp["latent"], inp["wc"], inp["wf"],
                            cs["NS"], cs["n_coarse"], cs["n_fine"], cs["n_fine_depth"],
                            white_bkgd=cs["white_bkgd"], eval_batch_size=cs["eval_batch_size"])
        d = (res["coarse"]["rgb"] - out.coarse.rgb.reshape(-1, 3)).abs().max().item()
        dz = (res["coarse"]["z"] - zs[0]).abs().max().item()
        msg = f"   check: coarse rgb {d:.2e} z {dz:.2e}"
        if cs["n_fine"] > 0:
            d2 = (res["fine"]["rgb"] - out.fine.rgb.reshape(-1, 3)).abs().max().item()
            dz2 = (res["fine"]["z"] - zs[1]).abs().max().item()
            msg += f" | fine rgb {d2:.2e} z {dz2:.2e}"
        fo = oracle.field_eval(xyz, vdir, state, inp["latent"], inp["wc"], cs["NS"])
        msg += f" | field {(fo - f_c).abs().max().item():.2e}"
        print(msg)


def util_fixture(check):
    """Caller-side helpers our drop-in util must reproduce: pose_spherical, gen_rays."""
    _, _, util = ref_harness.import_reference()
    poses = torch.stack([util.pose_spherical(a, p, 1.3) for a, p in ((0, -30), (40, -30), (123.4, -10))])
    rays = util.gen_rays(poses, 12, 9, torch.tensor(13.5), 0.8, 1.8)
    rays_c = util.gen_rays(poses[:1], 12, 9, torch.tensor([13.5, 14.0]), 0.1, 5.0,
                           c=torch.tensor([6.5, 4.0]))
    np.savez_compressed(os.path.join(GOLD, "util_rays.npz"), poses=poses.numpy(), rays=rays.numpy(),
                        rays_c=rays_c.numpy())
    if check:
        p2 = torch.stack([synth.pose_spherical(a, p, 1.3) for a, p in ((0, -30), (40, -30), (123.4, -10))])
        r2 = synth.gen_rays(p2, 12, 9, torch.tensor(13.5), 0.8, 1.8)
        print("   check: pose", (p2 - poses).abs().max().item(), "rays", (r2 - rays).abs().max().item())
    print("util_rays: written")


def grad_fixture(name, check):
    """Gradients of the reference's own training loss (train/train.py:199-215: render with want_weights, MSE coarse
    + MSE fine, loss.backward()) w.r.t. every MLP parameter and the latent, with the reference run in grad mode."""
    cs = CASES[name]
    inp = case_inputs(name, cs)
    net, renderer = ref_harness.build_reference(
        cs["d_hidden"], inp["wc"], inp["wf"], cs["n_coarse"], cs["n_fine"], cs["n_fine_depth"],
        white_bkgd=cs["white_bkgd"], eval_batch_size=cs["eval_batch_size"])
    latent = inp["latent"].clone().requires_grad_(True)
    ref_harness.set_scene(net, latent, inp["src_poses"], inp["focal"], inp["c"], cs["W"], cs["H"])
    g = torch.Generator().manual_seed(inp["seed"] + 6)
    gt = torch.rand(cs["SB"], cs["B"], 3, generator=g)
    torch.manual_seed(inp["seed"] + 4)
    out = renderer(net, inp["rays"], want_weights=True)
    crit = torch.nn.MSELoss()                       # loss.get_rgb_loss(conf["loss.rgb"], ...) with use_l1 = False
    loss = crit(out.coarse.rgb, gt)
    if cs["n_fine"] > 0:
        loss = loss * 1.0 + crit(out.fine.rgb, gt) * 1.0
    loss.backward()
    rec = dict(loss=np.array(loss.item()), rgb_gt=gt.numpy(), g_latent=latent.grad.numpy())
    for k, p in net.mlp_coarse.named_parameters():
        rec["gc/" + k] = p.grad.numpy()
    if net.mlp_fine is not None:
        for k, p in net.mlp_fine.named_parameters():
            rec["gf/" + k] = p.grad.numpy()
    path = os.path.join(GOLD, "grad_" + name + ".npz")
    np.savez_compressed(path, **rec)
    print(f"grad_{name}: wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB), loss {loss.item():.6f}")
    if check:
        state = oracle.encode_state(inp["src_poses"].reshape(-1, 4, 4), inp["focal"], inp["c"], cs["W"], cs["H"])
        lat = inp["latent"].clone().requires_grad_(True)
        wc = {k: v.clone().requires_grad_(True) for k, v in inp["wc"].items()}
        wf = None if inp["wf"] is None else {k: v.clone().requires_grad_(True) for k, v in inp["wf"].items()}
        lo = oracle.train_loss(inp["rays"], gt, inp["noise"], state, lat, wc, wf, cs["NS"], cs["n_coarse"],
                               cs["n_fine"], cs["n_fine_depth"], white_bkgd=cs["white_bkgd"],
                               eval_batch_size=cs["eval_batch_size"])
        lo.backward()
        worst = 0.0
        for k, v in wc.items():
            ref = torch.from_numpy(rec["gc/" + k])
            worst = max(worst, ((v.grad - ref).abs().max() / (ref.abs().max() + 1e-12)).item())
        print(f"   check: loss {abs(lo.item() - loss.item()):.2e}, coarse-grad worst rel {worst:.2e}, latent "
              f"{((lat.grad - latent.grad).abs().max() / latent.grad.abs().max()).item():.2e}")


def frames_fixture():
    """(frames * 255).astype(uint8) exactly as eval/gen_video.py:236 writes it, on colours that include the
    interesting boundaries (0, k/255 +- 1 ulp, 1.0, just above 1.0)."""
    g = torch.Generator().manual_seed(77)
    rgb = torch.rand(2, 5, 7, 3, generator=g)
    edge = torch.tensor([0.0, 1.0, 1.0000001, 0.5, 128 / 255, 127.999 / 255, 254.99999 / 255, 1e-8, 0.99999994,
                         3 / 255, 1 / 255, 0.003921569])
    rgb.view(-1)[: edge.numel()] = edge
    frames = rgb.view(-1, 5, 7, 3)
    u8 = (frames.cpu().numpy() * 255).astype(np.uint8)
    np.savez_compressed(os.path.join(GOLD, "frames_u8.npz"), rgb=rgb.numpy(), u8=u8)
    print("frames_u8: written")


def _flatten_conf(c, prefix=""):
    out = {}
    for k in c.keys():
        v = c[k]
        if hasattr(v, "keys"):
            out.update(_flatten_conf(v, prefix + k + "."))
        else:
            out[prefix + k] = v
    return out


def conf_fixture():
    """The reference's conf/exp/*.conf and expconf.conf as flattened trees, read with this package's HOCON reader (the
    reference's files are the schema the shipped confs must equal)."""
    hocon = _load("pnr_hocon", os.path.join(ROOT, "pixel-nerf_b200", "src", "util", "hocon.py"))
    ref = ref_harness.REF_ROOT
    rec = {"exp/" + name: _flatten_conf(hocon.parse_file(os.path.join(ref, "conf", "exp", name)))
           for name in sorted(os.listdir(os.path.join(ref, "conf", "exp")))}
    rec["expconf.conf"] = _flatten_conf(hocon.parse_file(os.path.join(ref, "expconf.conf")))
    path = os.path.join(GOLD, "ref_confs.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
    print(f"ref_confs: wrote {path} ({len(rec)} files)")


def encode_fixture():
    """The reference's SpatialEncoder.forward / PixelNeRFNet.encode state (src/model/encoder.py:111-164,
    src/model/models.py:89-144) for oracle.seeded_state weights on oracle.encode_scene inputs: the camera state exactly,
    the latent and index() values at oracle.encode_sample_index positions, and their max |value| (tolerance scale)."""
    model, _, _ = ref_harness.import_reference()
    rec = {}
    for name, (use_first_pool, (SB, NS, H, W)) in oracle.ENCODE_CASES.items():
        net = model.make_model(ref_harness.model_conf(64, use_first_pool)).eval()
        net.load_state_dict(oracle.seeded_state(net.state_dict(), 3), strict=True)
        images, poses, focal, c, uv = oracle.encode_scene(7, SB, NS, H, W)
        with torch.no_grad():
            net.encode(images, poses, focal, c=c)
            idx = net.encoder.index(uv, None, net.image_shape)
        lat = net.encoder.latent
        rec[name + "/latent_shape"] = np.array(lat.shape)
        rec[name + "/latent"] = lat.reshape(-1)[oracle.encode_sample_index(lat.numel(), 1)].numpy()
        rec[name + "/latent_absmax"] = np.array(lat.abs().max().item())
        rec[name + "/index_shape"] = np.array(idx.shape)
        rec[name + "/index"] = idx.reshape(-1)[oracle.encode_sample_index(idx.numel(), 2)].numpy()
        rec[name + "/index_absmax"] = np.array(idx.abs().max().item())
        for k in ("latent_scaling", "poses", "focal", "c", "image_shape"):
            v = net.encoder.latent_scaling if k == "latent_scaling" else getattr(net, k)
            rec[name + "/" + k] = v.numpy()
        rec[name + "/num_views_per_obj"] = np.array(net.num_views_per_obj)
    path = os.path.join(GOLD, "encode_state.npz")
    np.savez_compressed(path, **rec)
    print(f"encode_state: wrote {path} ({os.path.getsize(path) / 1e3:.0f} KB)")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    for name, cs in CASES.items():
        if a.only and a.only != name:
            continue
        run_case(name, cs, a.check)
    if not a.only:
        util_fixture(a.check)
    if not a.only or a.only == "frames_u8":
        frames_fixture()
    if not a.only or a.only == "confs":
        conf_fixture()
    if not a.only or a.only == "encode_state":
        encode_fixture()
    if not a.only or a.only == "grad":
        grad_fixture("tiny", a.check)
        grad_fixture("sb2_d", a.check)
