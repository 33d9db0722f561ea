"""Training through `bind_parallel(net, gpus)` on the GPU: the sharded fused node (render/fused_train.py,
`_ShardedFusedRender`: pnr_mgpu_render + pnr_mgpu_render_backward) against the single-GPU node on the same draws.
`[0, 0]` runs the whole sharded path -- two shards, a replica, the staged reduction -- on one device; `[0, 1]` and the
unmodified train.py with --gpu_id "0 1" need two GPUs and are skipped otherwise."""
import warnings

import pytest
import torch

import aux_grad_util as au
import golden_util as gu

pytestmark = pytest.mark.gpu
rel = au.rel


def _two_gpus():
    return torch.cuda.is_available() and torch.cuda.device_count() >= 2


DEVICES = [pytest.param([0, 0], id="one_gpu_two_shards"),
           pytest.param([0, 1], id="two_gpus", marks=pytest.mark.skipif(not _two_gpus(), reason="needs 2 GPUs"))]


def _draws(R, Kc, Kf, Kfd, seed, dev):
    g = torch.Generator().manual_seed(seed)
    nz = {"u_coarse": torch.rand(R, Kc, generator=g)}
    if Kf - Kfd > 0:
        nz["u_fine"], nz["u_fine_jit"] = torch.rand(R, Kf - Kfd, generator=g), torch.rand(R, Kf - Kfd, generator=g)
    if Kfd > 0:
        nz["n_depth"] = torch.randn(R, Kfd, generator=g)
    return {k: v.to(dev) for k, v in nz.items()}


def _flat_outputs(res, want_weights=True, fine=True):
    names = [o for o in au.OUTPUTS if (fine or o.startswith("coarse")) and (want_weights or "weights" not in o)]
    return names, [res[o.split(".")[0]][o.split(".")[1]] for o in names]


def _grads(net):
    out = {} if net.encoder.latent.grad is None else {"latent": net.encoder.latent.grad.clone()}
    for pre, m in (("coarse.", net.mlp_coarse), ("fine.", net.mlp_fine)):
        if m is not None:
            out.update({pre + k: p.grad.clone() for k, p in m.named_parameters()})
    return out


def _zero(net):
    for p in list(net.parameters()) + [net.encoder.latent]:
        p.grad = None


def _step(net, renderer, rays, noise, ups, par, want_weights=True):
    """One grad-mode render + backward with the given draws and upstream gradients -> (outputs, gradients).  par None:
    the single-GPU node; else the sharded node of `par` = bind_parallel(net, gpus)."""
    from render.fused_train import fused_render_train, sharded_render_train
    _zero(net)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        if par is None:
            res = fused_render_train(renderer, net, rays, want_weights, noise_in=noise)
        else:
            res = sharded_render_train(par, rays, want_weights, noise_in=noise)
    assert not [w for w in caught if "bind_parallel" in str(w.message)]
    fine = "fine" in res and len(res["fine"]) > 0
    names, outs = _flat_outputs(res, want_weights, fine)
    torch.autograd.backward(outs, grad_tensors=[ups[n].reshape(t.shape) for n, t in zip(names, outs)])
    torch.cuda.synchronize()
    return [t.detach().clone() for t in outs], _grads(net)


def _random_ups(SB, B, Kc, K, seed, dev):
    g = torch.Generator().manual_seed(seed)
    shapes = {"coarse.rgb": (SB, B, 3), "coarse.depth": (SB, B), "coarse.weights": (SB, B, Kc),
              "fine.rgb": (SB, B, 3), "fine.depth": (SB, B), "fine.weights": (SB, B, K)}
    return {k: (torch.randn(s, generator=g) / (SB * B)).to(dev) for k, s in shapes.items()}


def _compare(single, sharded, bound):
    (o1, g1), (o2, g2) = single, sharded
    for a, b in zip(o1, o2):
        assert torch.equal(a, b)
    assert g1.keys() == g2.keys()
    err = {k: rel(g2[k], g1[k]) for k in g1}
    worst = max(err.values())
    print(f"\nsharded vs single-GPU gradients: worst max-norm relative difference {worst:.3e} "
          f"({max(err, key=err.get)})")
    assert worst <= bound, sorted(err.items(), key=lambda kv: -kv[1])[:5]
    return worst


@pytest.mark.parametrize("gpus", DEVICES)
def test_sharded_step_matches_one_gpu_at_c2_train_shape(gpus):
    """C2 model at train.py's batch (SB = 4, B = 128, tensor engine) with injected draws: the sharded node's outputs
    are bit-identical to the single-GPU node's, and every weight and latent gradient agrees to <= 1e-4 relative
    (the float atomics of the backward make two runs of either node agree only to rounding).  Then an optimizer step
    and a new scene, as on every training step: the next sharded step refreshes the replica and still agrees."""
    from test_gpu_aux_grad import _c2_train_scene
    dev = torch.device("cuda:0")
    net, renderer, rays = _c2_train_scene(dev)
    SB, B = rays.shape[:2]
    Kc, Kf, Kfd = renderer.n_coarse, renderer.n_fine, renderer.n_fine_depth
    ups = _random_ups(SB, B, Kc, Kc + Kf, 9, dev)
    par = renderer.bind_parallel(net, gpus).train()
    noise = _draws(SB * B, Kc, Kf, Kfd, 7, dev)
    _compare(_step(net, renderer, rays, noise, ups, None), _step(net, renderer, rays, noise, ups, par), 1e-4)
    rep = par._replicas[gpus[1]]
    refreshes = rep.refreshes
    torch.optim.SGD(net.parameters(), lr=1e-1).step()          # with the sharded step's gradients
    lat = (net.encoder.latent.detach() * 0.9 + 0.01).clone().requires_grad_(True)
    net.set_scene(lat, _poses(net), net.focal[:, 0].clone(), None, *net._image_wh)
    noise = _draws(SB * B, Kc, Kf, Kfd, 8, dev)
    _compare(_step(net, renderer, rays, noise, ups, None), _step(net, renderer, rays, noise, ups, par), 1e-4)
    assert rep.refreshes >= refreshes + 2                    # weights and scene


def _poses(net):
    """Camera-to-world poses [SB][NS][4][4] back from the world-to-camera ones set_cameras stored."""
    w2c = net.poses
    rot, t = w2c[:, :3, :3], w2c[:, :3, 3:]
    c2w = torch.eye(4, device=w2c.device).repeat(w2c.shape[0], 1, 1)
    c2w[:, :3, :3] = rot.transpose(1, 2)
    c2w[:, :3, 3:] = -torch.bmm(rot.transpose(1, 2), t)
    return c2w.reshape(net.num_objs, net.num_views_per_obj, 4, 4)


@pytest.mark.parametrize("gpus", DEVICES)
@pytest.mark.parametrize("name", au.CASE_NAMES)
def test_sharded_node_matches_reference_gradients_of_all_outputs(name, gpus):
    """The fixture's upstream gradients of the six outputs through the sharded node: every weight and latent gradient
    equals what the unmodified reference computed to <= 1e-3 relative, the bar of the single-GPU node."""
    import gpu_util
    from render.fused_train import sharded_render_train
    case, aux = gu.load_case(name), au.load(name)
    net = gpu_util.build_net(case, device="cuda:0", engine="auto").train()
    net.encoder.latent = case["latent"].cuda().clone().requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    par = renderer.bind_parallel(net, gpus).train()
    res = sharded_render_train(par, case["rays"].cuda(), True, noise_in={k: v.cuda() for k, v in case["noise"].items()})
    names, outs = _flat_outputs(res)
    torch.autograd.backward(outs, grad_tensors=[aux["up"][o].cuda().reshape(t.shape) for o, t in zip(names, outs)])
    assert rel(net.encoder.latent.grad.cpu(), aux["g_latent"]) < 1e-3
    for k, p in net.mlp_coarse.named_parameters():
        assert rel(p.grad.cpu(), aux["gc"][k]) < 1e-3, ("coarse", k)
    for k, p in net.mlp_fine.named_parameters():
        assert rel(p.grad.cpu(), aux["gf"][k]) < 1e-3, ("fine", k)


@pytest.mark.parametrize("variant", ["no_weights", "simple_output", "stop_encoder_grad", "no_fine_mlp", "eight_shards"])
def test_sharded_step_variants_match_one_gpu(variant):
    """want_weights=False, simple_output (the best pass only), stop_encoder_grad (no latent gradient), mlp_fine None,
    and eight shards on one GPU of which the last two get no rays (B = 12): the same outputs and gradients as the
    single-GPU node."""
    import gpu_util
    from render.fused_train import sharded_render_train
    case = gu.load_case("sb2_d")
    net = gpu_util.build_net(case, device="cuda:0", engine="auto").train()
    if variant == "no_fine_mlp":
        net.mlp_fine = None
    net.encoder.latent = case["latent"].cuda().clone().requires_grad_(variant != "stop_encoder_grad")
    net.stop_encoder_grad = variant == "stop_encoder_grad"
    renderer = gpu_util.build_renderer(case).train()
    cfg = case["cfg"]
    SB, B, Kc, Kf = cfg["SB"], cfg["B"], cfg["n_coarse"], cfg["n_fine"]
    rays = case["rays"].cuda()
    noise = {k: v.cuda() for k, v in case["noise"].items()}
    ups = _random_ups(SB, B, Kc, Kc + Kf, 3, "cuda:0")
    gpus = [0] * 8 if variant == "eight_shards" else [0, 0]
    if variant == "simple_output":     # the wrapper returns (rgb, depth) of the fine pass only
        import render.nerf as rn
        zero_coarse = {k: (v * 0 if k.startswith("coarse") else v) for k, v in ups.items()}
        outs1, g1 = _step(net, renderer, rays, noise, zero_coarse, None, want_weights=False)
        par = renderer.bind_parallel(net, gpus, simple_output=True).train()
        _zero(net)
        rgb, depth = rn._wrapper_output(renderer, sharded_render_train(par, rays, False, noise_in=noise), True)
        torch.autograd.backward([rgb, depth], grad_tensors=[ups["fine.rgb"], ups["fine.depth"]])
        torch.cuda.synchronize()
        assert torch.equal(rgb.detach(), outs1[2]) and torch.equal(depth.detach(), outs1[3])
        _compare((outs1[2:], g1), ([rgb.detach(), depth.detach()], _grads(net)), 1e-4)
        return
    ww = variant != "no_weights"
    single = _step(net, renderer, rays, noise, ups, None, want_weights=ww)
    sharded = _step(net, renderer, rays, noise, ups, renderer.bind_parallel(net, gpus).train(), want_weights=ww)
    _compare(single, sharded, 1e-4)
    if variant == "stop_encoder_grad":
        assert "latent" not in sharded[1]


def test_bind_parallel_grad_mode_uses_the_sharded_node():
    """Through the wrapper's own forward (the call train.py makes): outputs require grad, no fallback warning, the
    gradients reach every parameter and the latent on gpus[0]."""
    import gpu_util
    case = gu.load_case("sb2_d")
    net = gpu_util.build_net(case, device="cuda:0", engine="auto").train()
    net.encoder.latent = case["latent"].cuda().clone().requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    par = renderer.bind_parallel(net, [0, 0]).train()
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        out = par(case["rays"].cuda(), want_weights=True)
    loss = out["coarse"]["rgb"].square().mean() + out["fine"]["weights"].sum(-1).mean() + out["fine"]["depth"].mean()
    loss.backward()
    assert net.encoder.latent.grad is not None and net.encoder.latent.grad.abs().max() > 0
    assert all(p.grad is not None for p in net.parameters() if p.requires_grad and p is not net.encoder.latent
               and any(p is q for m in (net.mlp_coarse, net.mlp_fine) for q in m.parameters()))
    assert par._replicas[0].refreshes > 0


@pytest.mark.skipif(not _two_gpus(), reason="needs 2 GPUs")
def test_train_main_runs_unmodified_on_two_gpus(tmp_path):
    """The reference's unmodified train/train.py with --gpu_id "0 1" through the overlay tree."""
    import numpy as np
    import dropin_util as du
    if du.reference_root() is None:
        pytest.skip("no reference checkout (oracle/_ref)")
    overlay = du.make_overlay(tmp_path)
    data = du.make_srn_dataset(str(tmp_path / "data" / "cars"), n_obj=4, n_views=5, size=128)
    conf = du.write_test_conf(overlay, str(tmp_path / "test.conf"),
                              extra="train {\n  print_interval = 1\n  save_interval = 2\n  vis_interval = 2\n  eval_interval = 2\n}\n")
    r = du.run_script(overlay, "train/train.py",
                      ["-n", "dropin_train2", "-c", conf, "-D", data, "-F", "srn", "-B", "2", "-V", "2", "--epochs", "2",
                       "--gpu_id", "0 1", "--lr", "1e-4"], cwd=tmp_path, timeout=1500)
    assert r.returncode == 0, (r.stderr[-3000:], r.stdout[-1000:])
    assert "gradients are required" not in r.stderr
    losses = [float(l.split("t:")[1].split()[0]) for l in r.stdout.splitlines() if l.startswith("E ") and " t:" in l]
    assert len(losses) == 4 and all(np.isfinite(losses))
