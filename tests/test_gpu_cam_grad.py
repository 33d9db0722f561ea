"""Gradients w.r.t. the rays and the source cameras through the default CUDA training path on one GPU
(render/fused_train.py: pnr_render forward, pnr_render_backward_cam backward), through the bare field node and through
util.gen_rays: against torch autograd of the oracle's forward (which restates the reference's graph), against the
composed-torch path at the train.py shape, and for pose refinement with a frozen network."""
import os
import warnings

import pytest
import torch

import aux_grad_util as au
import golden_util as gu

pytestmark = pytest.mark.gpu
rel = au.rel
OUTS = [("coarse", "rgb"), ("coarse", "depth"), ("coarse", "weights"), ("fine", "rgb"), ("fine", "depth"),
        ("fine", "weights")]


def _cameras(case, dev):
    """Leaf camera tensors requiring grad: c2w source poses, focal and c as given to encode()."""
    cfg = case["cfg"]
    poses = case["src_poses"].clone().to(dev).requires_grad_(True)
    focal = case["focal"].clone().to(dev).requires_grad_(True)
    c = case["c"] if case["c"] is not None else torch.tensor([[cfg["W"] * 0.5, cfg["H"] * 0.5]])   # one (cx, cy) row
    c = c.clone().to(dev).requires_grad_(True)
    return poses, focal, c


def _oracle_grads(case, up):
    """Autograd of the oracle's forward on the CPU -> gradients of rays, c2w poses, focal and c."""
    cfg = case["cfg"]
    poses, focal, c = _cameras(case, "cpu")
    rays = case["rays"].clone().requires_grad_(True)
    state = gu.oracle.encode_state(poses.reshape(-1, 4, 4), focal, c, cfg["W"], cfg["H"])
    res = gu.oracle.render(rays, case["noise"], state, case["latent"], case["wc"], case["wf"], cfg["NS"],
                           cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"], white_bkgd=bool(cfg["white_bkgd"]),
                           eval_batch_size=cfg["eval_batch_size"])
    outs = [res[p][q] for p, q in OUTS]
    torch.autograd.backward(outs, grad_tensors=[up[f"{p}.{q}"].reshape(t.shape) for (p, q), t in zip(OUTS, outs)])
    return dict(rays=rays.grad, poses=poses.grad, focal=focal.grad, c=c.grad)


def _fused_step(case, engine, up, frozen=True):
    import gpu_util
    from render.fused_train import fused_render_train
    dev = torch.device("cuda:0")
    net = gpu_util.build_net(case, device=dev, engine=engine).train()
    if frozen:
        net.requires_grad_(False)
    poses, focal, c = _cameras(case, dev)
    cfg = case["cfg"]
    net.set_scene(case["latent"].to(dev), poses, focal, c, cfg["W"], cfg["H"])
    rays = case["rays"].clone().to(dev).requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    noise = {k: v.cuda() for k, v in case["noise"].items()}
    out = fused_render_train(renderer, net, rays, True, noise_in=noise)
    outs = [out[p][q] for p, q in OUTS]
    torch.autograd.backward(outs, grad_tensors=[up[f"{p}.{q}"].to(dev).reshape(t.shape)
                                                for (p, q), t in zip(OUTS, outs)])
    return dict(rays=rays.grad, poses=poses.grad, focal=focal.grad, c=c.grad), net


@pytest.mark.parametrize("engine", ["auto", "simt"])
@pytest.mark.parametrize("name", au.CASE_NAMES)
def test_fused_node_ray_and_camera_gradients_match_the_oracle(name, engine):
    """The reference's upstream gradients of all six outputs (tests/golden/grad_aux_*.npz) through the fused node of a
    frozen network: rays, c2w source poses, focal and c against autograd of the oracle's forward, <= 1e-3."""
    case, aux = gu.load_case(name), au.load(name)
    got, _ = _fused_step(case, engine, aux["up"])
    ref = _oracle_grads(case, aux["up"])
    for k in ("rays", "poses", "focal", "c"):
        assert ref[k].abs().max() > 0, k
        assert rel(got[k].cpu(), ref[k]) < 1e-3, (k, rel(got[k].cpu(), ref[k]))


@pytest.mark.parametrize("engine", ["auto", "simt"])
@pytest.mark.parametrize("fixture", ["tiny", "sb2_d", "sb2_d_clamp"])
def test_fused_node_matches_the_reference_camera_gradients(fixture, engine):
    """tests/golden/grad_cam_*.npz (the unmodified reference with rays, c2w poses, focal and c requiring grad) replayed
    through the fused node: every ray / camera gradient and the MLP gradients to <= 1e-3."""
    import test_golden_cam_grad as gc
    fx = gc.load(fixture)
    case = gu.load_case(gc.FIXTURES[fixture])
    case["c"] = fx["c"]
    import gpu_util
    from render.fused_train import fused_render_train
    dev = torch.device("cuda:0")
    net = gpu_util.build_net(case, device=dev, engine=engine).train()
    poses, focal, c = _cameras(case, dev)
    cfg = case["cfg"]
    net.set_scene(case["latent"].to(dev), poses, focal, c, cfg["W"], cfg["H"])
    rays = case["rays"].clone().to(dev).requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    renderer.depth_std = fx["depth_std"]
    out = fused_render_train(renderer, net, rays, True, noise_in={k: v.cuda() for k, v in case["noise"].items()})
    outs = [out[p][q] for p, q in OUTS]
    torch.autograd.backward(outs, [fx["up"][f"{p}.{q}"].to(dev).reshape(t.shape) for (p, q), t in zip(OUTS, outs)])
    for got, ref in ((rays.grad, fx["rays"]), (poses.grad, fx["poses"]), (focal.grad, fx["focal"]),
                     (c.grad, fx["g_c"])):
        assert rel(got.cpu().reshape(ref.shape), ref) < 1e-3
    for k, p in net.mlp_coarse.named_parameters():
        assert rel(p.grad.cpu(), fx["gc"][k]) < 1e-3, k


def test_trainable_network_still_gets_the_reference_weight_gradients():
    """Camera gradients requested alongside trainable MLPs: the MLP gradients still match the reference's."""
    case, aux = gu.load_case("sb2_d"), au.load("sb2_d")
    _, net = _fused_step(case, "auto", aux["up"], frozen=False)
    for k, p in net.mlp_coarse.named_parameters():
        assert rel(p.grad.cpu(), aux["gc"][k]) < 1e-3, ("coarse", k)
    for k, p in net.mlp_fine.named_parameters():
        assert rel(p.grad.cpu(), aux["gf"][k]) < 1e-3, ("fine", k)


def test_nothing_requested_launches_what_it_launched_before(monkeypatch):
    """No ray / camera gradient asked for: the node calls pnr_render_backward_ex as before, with the same launches."""
    import gpu_util
    import pnr_native as pn
    from render.fused_train import fused_render_train
    case, aux = gu.load_case("sb2_d"), au.load("sb2_d")
    net = gpu_util.build_net(case, device="cuda:0", engine="auto").train()
    net.encoder.latent = net.encoder.latent.clone().requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    noise = {k: v.cuda() for k, v in case["noise"].items()}
    L = pn.lib()
    calls = []
    orig_ex, orig_cam = L.pnr_render_backward_ex, L.pnr_render_backward_cam
    monkeypatch.setattr(L, "pnr_render_backward_ex", lambda *a: calls.append("ex") or orig_ex(*a))
    monkeypatch.setattr(L, "pnr_render_backward_cam", lambda *a: calls.append("cam") or orig_cam(*a))
    counts = []
    for cam_arg in (False, True):
        rays = case["rays"].cuda()
        out = fused_render_train(renderer, net, rays, True, noise_in=noise)
        outs = [out[p][q] for p, q in OUTS]
        n0 = pn.launch_count()
        torch.autograd.backward(outs, grad_tensors=[aux["up"][f"{p}.{q}"].cuda().reshape(t.shape)
                                                    for (p, q), t in zip(OUTS, outs)])
        torch.cuda.synchronize()
        counts.append(pn.launch_count() - n0)
        if not cam_arg:
            ref = [net.encoder.latent.grad.clone()] + [p.grad.clone() for p in net.mlp_coarse.parameters()]
            net.zero_grad()
            net.encoder.latent.grad = None
            net.poses.requires_grad_(True)
    assert calls == ["ex", "cam"]
    assert counts[1] > counts[0]
    # the weight-gradient GEMMs (split-K) and the latent scatter accumulate with float atomics: on the GPU two runs agree
    # to the rounding of the accumulation order; bit equality of the two entry points is checked on the emulator
    got = [net.encoder.latent.grad] + [p.grad for p in net.mlp_coarse.parameters()]
    for a, b in zip(ref, got):
        assert rel(b, a) < 1e-4


def test_field_node_view_direction_and_camera_gradients():
    """net(xyz, viewdirs=...) in grad mode (model/fused_field.py) against autograd of the oracle's field."""
    import gpu_util
    case = gu.load_case("sb2_d")
    cfg = case["cfg"]
    dev = torch.device("cuda:0")
    net = gpu_util.build_net(case, device=dev, engine="auto").train().requires_grad_(False)
    poses, focal, c = _cameras(case, dev)
    net.set_scene(case["latent"].to(dev), poses, focal, c, cfg["W"], cfg["H"])
    g = torch.Generator().manual_seed(2)
    r = case["rays"][:, :10]
    xyz0 = (r[..., :3] + (0.8 + torch.rand(cfg["SB"], 10, 1, generator=g)) * r[..., 3:6]).contiguous()
    d_out = torch.randn(cfg["SB"], 10, 4, generator=g) * 1e-2
    xyz, dirs = xyz0.cuda().requires_grad_(True), r[..., 3:6].cuda().requires_grad_(True)
    net(xyz, coarse=True, viewdirs=dirs).backward(d_out.cuda())
    p2, f2, c2 = _cameras(case, "cpu")
    x2, d2 = xyz0.clone().requires_grad_(True), r[..., 3:6].clone().requires_grad_(True)
    state = gu.oracle.encode_state(p2.reshape(-1, 4, 4), f2, c2, cfg["W"], cfg["H"])
    gu.oracle.field_eval(x2, d2, state, case["latent"], case["wc"], cfg["NS"]).backward(d_out)
    for a, b in ((xyz, x2), (dirs, d2), (poses, p2), (focal, f2), (c, c2)):
        assert rel(a.grad.cpu(), b.grad) < 1e-3


def test_gen_rays_pose_gradient():
    import util
    g = torch.Generator().manual_seed(4)
    poses = gu.synth.pose_spherical(30.0, -20.0, 1.3)[None].repeat(2, 1, 1)
    poses[1, :3, 3] += 0.1
    W, H, f = 20, 14, torch.tensor(18.0)
    d_rays = torch.randn(2, H, W, 8, generator=g)
    p_gpu = poses.cuda().requires_grad_(True)
    rays = util.gen_rays(p_gpu, W, H, f.cuda(), 0.5, 2.5)
    rays.backward(d_rays.cuda())
    with torch.no_grad():
        assert torch.equal(rays.detach(), util.gen_rays(poses.cuda(), W, H, f.cuda(), 0.5, 2.5))
    p_cpu = poses.clone().requires_grad_(True)
    util.gen_rays(p_cpu, W, H, f, 0.5, 2.5).backward(d_rays)
    assert rel(p_gpu.grad.cpu(), p_cpu.grad) < 1e-5


def _c2_pose_scene(dev, perturb):
    """C2 model (d_hidden 512, tensor engine) at train.py's batch (SB = 4 objects, B = 128 rays), frozen; source poses
    (c2w) perturbed by `perturb` and requiring grad, target rays from util.gen_rays of poses requiring grad."""
    import gpu_util
    import util
    from model import make_model
    from render import NeRFRenderer
    c2 = gu.synth.CONFIGS["c2"]
    SB, NS, B = 4, c2["NS"], 128
    net = make_model(gpu_util.model_conf(512))
    net.mlp_coarse.load_state_dict(gu.synth.make_mlp_weights(31, 512))
    net.mlp_fine.load_state_dict(gu.synth.make_mlp_weights(32, 512))
    net = net.to(dev).train().requires_grad_(False)
    net.engine = "tc"
    r = (c2["z_near"] + c2["z_far"]) * 0.5
    src = torch.stack([torch.stack([gu.synth.pose_spherical(40.0 * v + 25.0 * o, -30.0, r) for v in range(NS)])
                       for o in range(SB)]).to(dev)
    src = (src + perturb).requires_grad_(True)
    latent = gu.synth.make_latent(5, SB * NS, 32, 32).to(dev)
    tgt = torch.stack([gu.synth.pose_spherical(100.0 + 70.0 * o, -10.0 - 5 * o, r) for o in range(SB)]).to(dev)
    tgt = tgt.requires_grad_(True)
    renderer = NeRFRenderer(n_coarse=c2["n_coarse"], n_fine=c2["n_fine"], n_fine_depth=c2["n_fine_depth"],
                            depth_std=0.01, white_bkgd=c2["white_bkgd"]).train()
    pix = torch.randint(0, c2["W"] * c2["H"], (SB, B), generator=torch.Generator().manual_seed(3)).to(dev)

    def rays_of(src_, tgt_):
        net.set_scene(latent, src_, torch.tensor([c2["focal"]]).to(dev), None, c2["W"], c2["H"])
        all_rays = util.gen_rays(tgt_, c2["W"], c2["H"], torch.tensor(c2["focal"]).to(dev), c2["z_near"],
                                 c2["z_far"]).reshape(SB, -1, 8)
        return torch.gather(all_rays, 1, pix[..., None].expand(-1, -1, 8))
    return net, renderer, src, tgt, rays_of


def _render_grads(net, renderer, src, tgt, rays_of, mode, target):
    """One render with PNR_FUSED_BACKWARD=mode and seeded RNG; rgb MSE against `target` -> (loss, grads of src, tgt)."""
    os.environ["PNR_FUSED_BACKWARD"] = mode
    try:
        torch.manual_seed(12)
        out = renderer.bind_parallel(net, None).train()(rays_of(src, tgt), want_weights=True)
        loss = ((out["fine"]["rgb"] - target) ** 2).mean() + ((out["coarse"]["rgb"] - target) ** 2).mean()
        gs, gt = torch.autograd.grad(loss, (src, tgt))
    finally:
        os.environ.pop("PNR_FUSED_BACKWARD", None)
    return loss.item(), gs, gt


def test_frozen_network_pose_refinement_at_train_shape():
    """Encoder and MLPs frozen, one source pose perturbed and the target poses trainable.  At every one of 20 Adam
    steps the fused node, the composed-torch path (PNR_FUSED_BACKWARD=0) and the field node under the torch renderer
    (=1, pnr_field_backward_cam on the tensor engine) compute the pose gradients at the same poses and agree within
    5e-2 (max-norm relative; the tensor-engine recompute and split-bf16 backward GEMMs already make the MLP gradients
    differ by up to 3.9e-2 at this shape; measured on an H100: 2.0e-2; the field backward alone, pose gradients
    included, stays within 8.4e-4 of float64 even with every point kept (tests/test_gpu_backward_wide.py), so it does
    not explain this gap, which is not explained yet); the step uses the fused gradients and the
    render loss against the unperturbed render decreases (measured: 0.193 -> 0.177; the synthetic field varies fast,
    so the loss is far from quadratic and 20 small steps do not close the gap)."""
    dev = torch.device("cuda:0")
    perturb = torch.zeros(4, gu.synth.CONFIGS["c2"]["NS"], 4, 4, device=dev)
    perturb[1, 0, :3, 3] = torch.tensor([0.03, -0.02, 0.025], device=dev)
    net, renderer, src, tgt, rays_of = _c2_pose_scene(dev, perturb)
    with torch.no_grad():
        torch.manual_seed(12)
        ref = renderer.bind_parallel(net, None)(rays_of(src - perturb, tgt), want_weights=True)
        target = ref["fine"]["rgb"].clone()
    opt = torch.optim.Adam([src, tgt], lr=2e-3)
    losses, worst = [], 0.0
    for _ in range(20):
        loss, gs, gt = _render_grads(net, renderer, src, tgt, rays_of, "auto", target)
        _, gs0, gt0 = _render_grads(net, renderer, src, tgt, rays_of, "0", target)
        _, gs1, gt1 = _render_grads(net, renderer, src, tgt, rays_of, "1", target)    # field node, torch renderer
        err = max(rel(gs, gs0), rel(gt, gt0), rel(gs, gs1), rel(gt, gt1))
        worst = max(worst, err)
        assert err < 5e-2, err
        losses.append(loss)
        opt.zero_grad()
        src.grad, tgt.grad = gs, gt
        opt.step()
    print(f"pose refinement: loss {losses[0]:.3e} -> {losses[-1]:.3e}, worst gradient gap {worst:.2e}")
    assert losses[-1] < losses[0], losses


def test_sharded_node_gives_the_single_gpu_ray_and_camera_gradients(monkeypatch):
    """bind_parallel(net, [0, 0]) with trainable rays and cameras: two shards on one GPU through
    pnr_mgpu_render_backward_cam, no fallback warning.  With the same full-ray draws injected into both (each shard
    otherwise draws its own, as under DataParallel), its gradients equal the single-GPU node's to <= 1e-4."""
    import gpu_util
    import pnr_native as pn
    from render.fused_train import fused_render_train, sharded_render_train
    case, aux = gu.load_case("sb2_d"), au.load("sb2_d")
    cfg = case["cfg"]
    L = pn.lib()
    calls = []
    orig = L.pnr_mgpu_render_backward_cam
    monkeypatch.setattr(L, "pnr_mgpu_render_backward_cam", lambda *a: calls.append(1) or orig(*a))
    noise = {k: v.cuda() for k, v in case["noise"].items()}
    res = []
    for gpus in (None, [0, 0], [0, 0]):
        net = gpu_util.build_net(case, device="cuda:0", engine="auto").train().requires_grad_(False)
        poses, focal, c = _cameras(case, "cuda:0")
        net.set_scene(case["latent"].cuda(), poses, focal, c, cfg["W"], cfg["H"])
        renderer = gpu_util.build_renderer(case).train()
        rays = case["rays"].cuda().requires_grad_(True)
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            if gpus is None:
                out = fused_render_train(renderer, net, rays, True, noise_in=noise)
            elif not res[1:]:      # through the public wrapper: it must take the sharded node, not the fallback
                out = renderer.bind_parallel(net, gpus).train()(rays, want_weights=True)
            else:
                out = sharded_render_train(renderer.bind_parallel(net, gpus).train(), rays, True, noise_in=noise)
        assert not [w for w in caught if "bind_parallel" in str(w.message)], [str(w.message) for w in caught]
        outs = [out[p][q] for p, q in OUTS]
        torch.autograd.backward(outs, grad_tensors=[aux["up"][f"{p}.{q}"].cuda().reshape(t.shape)
                                                    for (p, q), t in zip(OUTS, outs)])
        res.append([rays.grad, poses.grad, focal.grad, c.grad])
    assert calls == [1, 1]                    # both sharded steps ran the sharded backward
    for a, b in zip(res[0], res[2]):
        assert a.abs().max() > 0
        assert rel(b, a) < 1e-4
