"""Full-size configurations of BASELINE.json (C2 / C3 / C4 shapes, real resnet34 trunk for the latent) checked
through size-independent properties, since the CPU oracle would take minutes there:
  * the tensor engine's fine samples are explained on every ray by its own coarse pass (tests/fine_pass_check.py),
    and its fine rgb equals the fp32 SIMT engine's field composited at those samples (|d rgb| < 1e-4, every ray),
  * batch-split invariance: a ray's result does not depend on which other rays share its call (bit-exact),
  * sample depths are sorted, weights are non-negative and sum to <= 1, white background closes the sum.
"""
import importlib.util
import os
import sys

import pytest
import torch

import fine_pass_check as fpc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _load_bench():
    spec = importlib.util.spec_from_file_location("pnr_bench", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _scene(name, engine):
    bench = _load_bench()
    cfg = bench.synth.CONFIGS[name]
    net, renderer = bench.build_scene(cfg, torch.device("cuda:0"), engine)
    return bench, cfg, net, renderer


def _tc_fine_checked(net, rays, out, noise, cfg, white_bkgd, depth_std=0.01):
    """Layers 1 and 2 of tests/fine_pass_check.py on every ray of a tensor-engine render, and its fine rgb against the
    SIMT engine's fine field at the same samples, composited by pnr_composite, on every ray."""
    pick = lambda o: dict(z=o.z, weights=o.weights, depth=o.depth, rgb=o.rgb)
    return fpc.check_render(rays, pick(out.coarse), pick(out.fine), {k: v.cpu() for k, v in noise.items()},
                            cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"], depth_std,
                            fpc.simt_composite(net, white_bkgd), depth_tol=None, weights_tol=None)


@pytest.mark.parametrize("name,n_rays", [("c2", 3000), ("c3", 3000), ("c4", 1500)])
def test_engines_agree_at_full_config(name, n_rays):
    bench, cfg, net, renderer = _scene(name, "tc")
    rays = bench.synth.make_rays(cfg, n_rays).cuda()[None]
    noise = {k: v.cuda() for k, v in bench.synth.draw_noise(5, n_rays, cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]).items()}
    import pnr_native as pn
    with torch.no_grad():
        a = renderer._forward_fused(net, rays, True, noise_in=noise, want_z=True)
        assert pn.tc_status() == 0
        net.engine = "simt"
        b = renderer._forward_fused(net, rays, True, noise_in=noise, want_z=True)
    assert (a.coarse.rgb - b.coarse.rgb).abs().max() < 1e-4
    assert (a.coarse.depth - b.coarse.depth).abs().max() < 2e-4
    chk = _tc_fine_checked(net, rays, a, noise, cfg, white_bkgd=cfg["white_bkgd"])
    flipped = int(((a.fine.z - b.fine.z).abs() > 2e-4).any(dim=-1).sum())
    print(f"{name}: {chk}, {flipped} of {n_rays} rays merged other samples than the SIMT engine")
    for o in (a, b):
        z, w = o.fine.z, o.fine.weights
        assert torch.all(z[..., 1:] >= z[..., :-1])
        assert torch.all(w >= 0) and torch.all(w.sum(-1) <= 1 + 1e-5)
        assert torch.isfinite(o.fine.rgb).all()
    if cfg["white_bkgd"]:
        # white background: rgb = sum(w * rgb_k) + 1 - sum(w) >= 1 - sum(w)
        assert torch.all(a.fine.rgb.min(-1).values >= 1 - a.fine.weights.sum(-1) - 1e-5)


def test_batch_split_invariance_bit_exact():
    """Rays are independent units: rendering them in one call or in ragged pieces (with the same per-ray noise)
    must give bit-identical pixels -- the property multi-GPU sharding relies on."""
    bench, cfg, net, renderer = _scene("c2", "tc")
    n = 1000
    rays = bench.synth.make_rays(cfg, n).cuda()[None]
    noise = {k: v.cuda() for k, v in bench.synth.draw_noise(9, n, cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]).items()}
    with torch.no_grad():
        full = renderer._forward_fused(net, rays, False, noise_in=noise)
        parts = []
        for a, b in ((0, 137), (137, 640), (640, 1000)):
            sub = {k: v[a:b].contiguous() for k, v in noise.items()}
            parts.append(renderer._forward_fused(net, rays[:, a:b].contiguous(), False, noise_in=sub).fine.rgb)
    assert torch.equal(torch.cat(parts, dim=1), full.fine.rgb)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_render_matches_single_gpu_order():
    """bind_parallel(net, [0, 1]): same ray order as one GPU; per-shard noise differs (as with DataParallel),
    so compare with injected noise through the replicas directly."""
    bench, cfg, net, renderer = _scene("c2", "tc")
    n = 513
    rays = bench.synth.make_rays(cfg, n).cuda()[None]
    par = renderer.bind_parallel(net, [0, 1], simple_output=True)
    with torch.no_grad():
        rgb, depth = par(rays)
    assert rgb.shape == (1, n, 3) and depth.shape == (1, n) and rgb.device.index == 0
    assert torch.isfinite(rgb).all()
    # shard boundaries follow torch.chunk: replica 1 renders rays[257:]
    rep = par._replicas[1]
    copies = rep.refreshes
    assert copies == 3                     # coarse weights, fine weights, scene: one peer copy each
    with torch.no_grad():
        par(rays)
    assert rep.refreshes == copies         # nothing changed -> nothing is re-sent (DataParallel re-broadcasts per call)
    noise = {k: v for k, v in bench.synth.draw_noise(3, n, cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]).items()}
    with torch.no_grad():
        whole = renderer._forward_fused(net, rays, False, noise_in={k: v.cuda(0) for k, v in noise.items()}).fine.rgb
        second = renderer._forward_fused(rep, rays[:, 257:].to("cuda:1"), False,
                                         noise_in={k: v[257:].contiguous().cuda(1) for k, v in noise.items()}).fine.rgb
    assert torch.equal(second.cpu(), whole[:, 257:].cpu())
    # an in-place weight update (optimizer.step) and a new encode() each invalidate exactly their part
    with torch.no_grad():
        net.mlp_fine.lin_out.bias.add_(0.25)
        par(rays)
        assert rep.refreshes == copies + 2          # fine weights + scene (its P maps depend on the weights)
        whole2 = renderer._forward_fused(net, rays, False, noise_in={k: v.cuda(0) for k, v in noise.items()}).fine.rgb
        second2 = renderer._forward_fused(rep, rays[:, 257:].to("cuda:1"), False,
                                          noise_in={k: v[257:].contiguous().cuda(1) for k, v in noise.items()}).fine.rgb
    assert torch.equal(second2.cpu(), whole2[:, 257:].cpu()) and not torch.equal(whole2, whole)


@pytest.mark.parametrize("name", ["c2", "c3", "c4"])
def test_oracle_parity_at_true_shapes(name):
    """The product default (engine auto -> tensor engine) against the CPU ORACLE at the true C2 / C3 / C4 shapes (real
    resnet34 latent: 2x512x64x64, 1x512x32x32, 3x512x150x200), 256 rays spread over a frame, injected noise --
    the same `parity` block bench.py prints."""
    bench, cfg, net, renderer = _scene(name, "auto")
    rays = bench.synth.make_rays(cfg, bench.WORKLOADS[name]["frame_rays"]).cuda()[None]
    import pnr_native as pn
    par = bench.parity_block(net, renderer, cfg, rays, n=256)
    assert pn.tc_status() == 0
    assert net._fused.mlp["mlp_coarse"][3] is not None                 # the tensor engine did run
    assert par["rays"] == 256
    assert par["max_abs_drgb_coarse"] < 1e-4, par
    assert par["max_abs_drgb"] < 1e-4, par
    assert par["psnr_db"] > 50 if par["flipped_rays"] else par["psnr_db"] > 80, par
    # the same rays and noise, every ray's fine pass checked against the oracle at the kernel's own samples
    chk = fpc.check_true_shape(bench, net, renderer, cfg, rays, n=256, depth_tol=2e-4)
    assert pn.tc_status() == 0
    print(f"{name} tc: {chk}, {par['flipped_rays']} rays merged other samples than the oracle")
    lat = net.encoder.latent
    assert lat.shape[0] * lat.shape[2] * lat.shape[3] * 512 < 2 ** 32   # 32-bit tap offsets (pnr_field_tc.cu geo[])


@pytest.mark.parametrize("SB,NS", [(2, 2), (1, 6), (3, 1)])
def test_tensor_engine_multi_object_and_many_views(SB, NS):
    """Super-batches (train.py uses SB=4) and the C5 sweep's NS=6: tensor engine vs SIMT engine on synthetic
    latents, per-object focal lengths, through NeRFRenderer's fused path."""
    import gpu_util
    import golden_util as gu
    from model import make_model
    from render import NeRFRenderer
    import pnr_native as pn
    dev = torch.device("cuda:0")
    W = H = 32
    net = make_model(gpu_util.model_conf(512))
    net.mlp_coarse.load_state_dict(gu.synth.make_mlp_weights(21, 512))
    net.mlp_fine.load_state_dict(gu.synth.make_mlp_weights(22, 512))
    net = net.to(dev).eval()
    latent = gu.synth.make_latent(7, SB * NS, 16, 16).to(dev)
    poses = torch.stack([torch.stack([gu.synth.pose_spherical(40.0 * v + 25.0 * o, -30.0, 1.3) for v in range(NS)])
                         for o in range(SB)]).to(dev)
    focal = torch.linspace(30.0, 36.0, SB).to(dev)          # one focal length per object
    net.set_scene(latent, poses, focal, None, W, H)
    renderer = NeRFRenderer(n_coarse=32, n_fine=16, n_fine_depth=8, white_bkgd=True).eval()
    B = 200
    tgt = torch.stack([gu.synth.pose_spherical(100.0 + 50.0 * o, -15.0, 1.3) for o in range(SB)])
    rays = gu.synth.gen_rays(tgt, W, H, 32.0, 0.8, 1.8).reshape(SB, -1, 8)[:, :B].contiguous().to(dev)
    noise = {k: v.to(dev) for k, v in gu.synth.draw_noise(4, SB * B, 32, 16, 8).items()}
    with torch.no_grad():
        net.engine = "tc"
        a = renderer._forward_fused(net, rays, True, noise_in=noise, want_z=True)
        assert pn.tc_status() == 0
        net.engine = "simt"
        b = renderer._forward_fused(net, rays, True, noise_in=noise, want_z=True)
    assert a.fine.rgb.shape == (SB, B, 3)
    assert (a.coarse.rgb - b.coarse.rgb).abs().max() < 1e-4
    chk = _tc_fine_checked(net, rays, a, noise, dict(n_coarse=32, n_fine=16, n_fine_depth=8), white_bkgd=True)
    print(f"SB={SB} NS={NS}: {chk}")
