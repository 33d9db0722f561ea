"""Gradients of every output of the default CUDA training path (render/fused_train.py: pnr_render forward,
pnr_render_backward_ex backward) on one GPU: against the reference's own gradients for a loss on rgb, depth and weights
(tests/golden/grad_aux_*.npz), against the composed-torch grad path at the train.py shape on the tensor engine, and
the rgb-only step against the rgb-only entry point."""
import os

import pytest
import torch

import aux_grad_util as au
import golden_util as gu

pytestmark = pytest.mark.gpu
rel = au.rel


def _outputs(out, fine=True, want_weights=True):
    names = [o for o in au.OUTPUTS if (fine or o.startswith("coarse")) and (want_weights or "weights" not in o)]
    return names, [out[o.split(".")[0]][o.split(".")[1]] for o in names]


def _fixture_step(case, engine):
    import gpu_util
    from render.fused_train import fused_render_train
    net = gpu_util.build_net(case, device="cuda:0", engine=engine).train()
    net.encoder.latent = case["latent"].cuda().clone().requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    noise = {k: v.cuda() for k, v in case["noise"].items()}
    out = fused_render_train(renderer, net, case["rays"].cuda(), True, noise_in=noise)
    return net, out


@pytest.mark.parametrize("engine", ["auto", "simt"])
@pytest.mark.parametrize("name", au.CASE_NAMES)
def test_fused_node_matches_reference_gradients_of_all_outputs(name, engine):
    """The fixture's upstream gradients of the six outputs fed to the fused node: every weight and latent gradient
    equals what the unmodified reference computed to <= 1e-3 relative."""
    case, aux = gu.load_case(name), au.load(name)
    net, out = _fixture_step(case, engine)
    names, outs = _outputs(out)
    for t in outs:
        assert t.requires_grad
    torch.autograd.backward(outs, grad_tensors=[aux["up"][o].cuda().reshape(t.shape) for o, t in zip(names, outs)])
    assert rel(net.encoder.latent.grad.cpu(), aux["g_latent"]) < 1e-3
    for k, p in net.mlp_coarse.named_parameters():
        assert rel(p.grad.cpu(), aux["gc"][k]) < 1e-3, ("coarse", k)
    for k, p in net.mlp_fine.named_parameters():
        assert rel(p.grad.cpu(), aux["gf"][k]) < 1e-3, ("fine", k)


def _c2_train_scene(dev, engine="tc"):
    """C2 model (d_hidden 512, 2 source views, 64 + 32 samples of which 16 depth-centred) at train.py's batch: SB = 4
    objects, B = 128 rays each, on synthetic weights, latents and cameras."""
    import gpu_util
    from model import make_model
    from render import NeRFRenderer
    c2 = gu.synth.CONFIGS["c2"]
    SB, NS, B = 4, c2["NS"], 128
    net = make_model(gpu_util.model_conf(512))
    net.mlp_coarse.load_state_dict(gu.synth.make_mlp_weights(31, 512))
    net.mlp_fine.load_state_dict(gu.synth.make_mlp_weights(32, 512))
    net = net.to(dev).train()
    net.engine = engine
    r = (c2["z_near"] + c2["z_far"]) * 0.5
    poses = torch.stack([torch.stack([gu.synth.pose_spherical(40.0 * v + 25.0 * o, -30.0, r) for v in range(NS)])
                         for o in range(SB)]).to(dev)
    latent = gu.synth.make_latent(5, SB * NS, 32, 32).to(dev)
    net.set_scene(latent, poses, torch.tensor([c2["focal"]]).to(dev), None, c2["W"], c2["H"])
    net.encoder.latent = net.encoder.latent.clone().requires_grad_(True)
    renderer = NeRFRenderer(n_coarse=c2["n_coarse"], n_fine=c2["n_fine"], n_fine_depth=c2["n_fine_depth"],
                            depth_std=0.01, white_bkgd=c2["white_bkgd"]).train()
    tgt = torch.stack([gu.synth.pose_spherical(100.0 + 70.0 * o, -10.0 - 5 * o, r) for o in range(SB)])
    all_rays = gu.synth.gen_rays(tgt, c2["W"], c2["H"], c2["focal"], c2["z_near"], c2["z_far"]).reshape(SB, -1, 8)
    pix = torch.randint(0, all_rays.shape[1], (SB, B), generator=torch.Generator().manual_seed(3))
    rays = torch.stack([all_rays[o][pix[o]] for o in range(SB)]).contiguous().to(dev)
    return net, renderer, rays


def _c2_step(mode, up_fn, engine="tc"):
    """One grad-mode render at the C2 train shape with PNR_FUSED_BACKWARD=mode, seeded device RNG; records the fine
    sample depths each path used.  -> (outputs, z_fine, net) after backward with up_fn(outputs, z_fine)."""
    dev = torch.device("cuda:0")
    net, renderer, rays = _c2_train_scene(dev, engine)
    zs = []
    if mode == "0":
        orig = renderer.composite

        def spy(model, rays_, z_samp, coarse=True, sb=0):
            if not coarse:
                zs.append(z_samp.detach())
            return orig(model, rays_, z_samp, coarse=coarse, sb=sb)
        renderer.composite = spy
    else:
        orig = renderer._forward_fused

        def spy(*a, **kw):
            res = orig(*a, **kw)
            zs.append(res.fine.z.reshape(-1, res.fine.z.shape[-1]).detach())
            return res
        renderer._forward_fused = spy
    os.environ["PNR_FUSED_BACKWARD"] = mode
    try:
        render_par = renderer.bind_parallel(net, None).train()
        torch.manual_seed(12)
        out = render_par(rays, want_weights=True)
        names, outs = _outputs(out)
        torch.autograd.backward(outs, grad_tensors=up_fn(names, outs, zs[0]))
    finally:
        os.environ.pop("PNR_FUSED_BACKWARD", None)
    return outs, zs[0], net


def _c2_errors(rgb_only):
    """Fused node (tensor engine) vs composed torch at the C2 train shape for seeded random upstream gradients of all
    six outputs (rgb_only: of the two rgb outputs only) -> (max-norm relative error per gradient tensor, fraction of
    rays with a flipped fine sample).  Both runs draw the same samples from the same seeded device RNG, except where
    the tensor engine's coarse weights put an importance sample in a neighbouring CDF bin: those rays get zero upstream
    gradient in both runs."""
    saved = {}

    def up_fn_ref(names, outs, z):
        saved["z0"] = z
        return [torch.zeros_like(t) for t in outs]    # this run only learns the composed path's fine samples

    _c2_step("0", up_fn_ref)
    g = torch.Generator().manual_seed(21)

    def up_fn_fused(names, outs, z):
        flipped = ((z - saved["z0"]).abs() > 2e-4).any(-1)
        saved["flipped"] = flipped
        keep = (~flipped).float().reshape(outs[0].shape[0], outs[0].shape[1])
        ups = []
        for n, t in zip(names, outs):
            u = torch.randn(t.shape, generator=g).to(t.device) / t.numel()
            if rgb_only and "rgb" not in n:
                u = torch.zeros_like(u)
            ups.append(u * keep.reshape(*keep.shape, *([1] * (t.dim() - 2))))
        saved["up"] = ups
        return ups

    outs1, _, net1 = _c2_step("auto", up_fn_fused)
    outs0, _, net0 = _c2_step("0", lambda names, outs, z: [u.clone() for u in saved["up"]])
    kept = ~saved["flipped"].reshape(outs1[0].shape[:2])
    for a, b in zip(outs1, outs0):
        assert (a.detach() - b.detach())[kept].abs().max() < 1e-3
    err = {"latent": rel(net1.encoder.latent.grad, net0.encoder.latent.grad)}
    for pre, m1, m0 in (("coarse ", net1.mlp_coarse, net0.mlp_coarse), ("fine ", net1.mlp_fine, net0.mlp_fine)):
        for (k, p), (_, q) in zip(m1.named_parameters(), m0.named_parameters()):
            err[pre + k] = rel(p.grad, q.grad)
    return err, saved["flipped"].float().mean().item()


def test_fused_node_matches_composed_torch_at_train_shape_on_the_tensor_engine():
    """Gradients of all six outputs through the fused node against the composed-torch path on the same device.  At this
    shape the two already differ by up to ~4e-2 (max-norm relative) for an rgb-only upstream, the existing behaviour:
    the backward recomputes the field with the tensor engine (sigma values near zero can land on the other side of the
    ReLU) and runs its GEMMs on split-bf16 operands, and random-sign upstream gradients cancel in the weight gradients.
    Measured on an H100: <= 1.4e-2 with all six outputs, <= 3.9e-2 rgb-only.  A dropped depth or weights term would give
    errors of order one, since those upstream gradients are as large as the rgb ones.  The field backward alone does
    not account for this gap: at width 512 it stays within 8.4e-4 of float64 on c2_small even with every point kept,
    ReLU arguments near zero included (tests/test_gpu_backward_wide.py, H100), so the rest of the ~1e-2 lies on the
    render or composed-torch side and is not explained yet."""
    err_all, flipped = _c2_errors(rgb_only=False)
    err_rgb, _ = _c2_errors(rgb_only=True)
    assert flipped < 0.05
    worst = max(err_all.values())
    assert worst < 5e-2, sorted(err_all.items(), key=lambda kv: -kv[1])[:5]
    assert worst <= 2.0 * max(err_rgb.values()), (worst, max(err_rgb.values()))


def _grads(net):
    return [net.encoder.latent.grad.clone()] + [p.grad.clone() for _, p in net.mlp_coarse.named_parameters()] + \
        [p.grad.clone() for _, p in net.mlp_fine.named_parameters()]


@pytest.mark.parametrize("name", au.CASE_NAMES)
def test_rgb_only_step_same_through_old_and_new_entry_points(name, monkeypatch):
    """An rgb-only loss reaches the library with NULL depth / weights gradients.  Routing the node to the rgb-only entry
    point pnr_render_backward instead runs the same arithmetic.  The weight-gradient GEMMs (split-K) and the latent
    scatter accumulate with float atomics, so on the GPU two runs of either entry point agree to the rounding of the
    accumulation order, not bit for bit; tests/test_emu_aux_grad.py checks bit equality on the sequential emulator."""
    import pnr_native as pn
    case, aux = gu.load_case(name), au.load(name)
    gt = aux["rgb_gt"].cuda()

    def step():
        net, out = _fixture_step(case, "auto")
        crit = torch.nn.MSELoss()
        (crit(out.coarse.rgb, gt) + crit(out.fine.rgb, gt)).backward()
        torch.cuda.synchronize()
        return _grads(net)

    new = step()
    L = pn.lib()
    calls = []

    def old_entry(scene, mc, mf, cfg, rays, noise, fwd, ug, gc, gf, dlat, B, ws, nbytes, stream):
        calls.append(1)
        assert not (ug.d_depth_coarse or ug.d_weights_coarse or ug.d_depth_fine or ug.d_weights_fine)
        return L.pnr_render_backward(scene, mc, mf, cfg, rays, noise, fwd, ug.d_rgb_coarse, ug.d_rgb_fine, gc, gf,
                                     dlat, B, ws, nbytes, stream)
    monkeypatch.setattr(L, "pnr_render_backward_ex", old_entry)
    old = step()
    assert len(calls) == 1
    assert new[0].abs().max() > 0
    for a, c in zip(old, new):
        assert rel(c, a) < 1e-4


def test_grad_mode_outputs_all_require_grad_and_no_grad_outputs_unchanged():
    import gpu_util
    case = gu.load_case("sb2_d")
    net = gpu_util.build_net(case, device="cuda:0", engine="auto").train()
    renderer = gpu_util.build_renderer(case).train()
    rays = case["rays"].cuda()
    for want_weights in (True, False):
        torch.manual_seed(5)
        out = renderer(net, rays, want_weights=want_weights)
        names, outs = _outputs(out, want_weights=want_weights)
        assert ("weights" in out["coarse"]) == want_weights and ("weights" in out["fine"]) == want_weights
        assert all(t.requires_grad for t in outs), names
        torch.manual_seed(5)
        with torch.no_grad():
            ref = renderer(net, rays, want_weights=want_weights)
        _, refs = _outputs(ref, want_weights=want_weights)
        for n, a, b in zip(names, outs, refs):
            assert not b.requires_grad
            assert (a.detach() - b).abs().max() < 1e-6, n
