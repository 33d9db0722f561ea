"""Fused forward + `pnr_render_backward` for a training step (SURVEY 8f-1).

The default grad-mode path on CUDA (`PNR_FUSED_BACKWARD` unset / auto / 2): `NeRFRenderer.forward` becomes ONE autograd
node whose forward is the fused `pnr_render` (any engine, incl. the tensor engine) and whose backward is
`pnr_render_backward` (fp32 recompute-in-backward).  Validated on H100 against the composed-torch path on the same
device and against the gradients the reference computed itself (tests/test_gpu_backward.py), and on the host emulator
(tests/test_emu_kernels.py).

Every returned output is differentiable, as in the reference: `rgb`, `depth` and (with `want_weights`) `weights` of
both passes.  A loss may so add e.g. the alpha loss of model/loss.py on `fine.weights.sum(-1)` or a depth term to the
rgb losses of train/train.py:199-212; the backward is `pnr_render_backward_ex` with the upstream gradient of each
output.  Outputs the loss does not use reach the backward as None and go to the library as NULL, so an rgb-only step
runs the same arithmetic as the rgb-only entry point `pnr_render_backward`.
"""
import torch

import pnr_native as pn

from .dotmap_compat import DotMap


class _FusedRender(torch.autograd.Function):
    @staticmethod
    def forward(ctx, renderer, model, want_weights, noise_in, rays, latent, *params):
        dev = rays.device
        SB, B, _ = rays.shape
        R = SB * B
        Kc, Kf, Kfd = int(renderer.n_coarse), int(renderer.n_fine), int(renderer.n_fine_depth)
        fine = bool(renderer.using_fine) and Kf > 0
        if not fine:
            Kf = Kfd = 0
        f32 = dict(dtype=torch.float32, device=dev)
        if noise_in is not None:          # parity tests replay a fixture's draws
            noise = {k: v.to(**f32).contiguous() for k, v in noise_in.items()}
        else:
            noise = {"u_coarse": torch.rand(R, Kc, **f32)}      # the reference's draw order (nerf.py:111,135,141,158)
            if fine and Kf - Kfd > 0:
                noise["u_fine"] = torch.rand(R, Kf - Kfd, **f32)
                noise["u_fine_jit"] = torch.rand(R, Kf - Kfd, **f32)
            if fine and Kfd > 0:
                noise["n_depth"] = torch.randn(R, Kfd, **f32)
        with torch.no_grad():
            res = renderer._forward_fused(model, rays, want_weights, noise_in=noise, want_z=True)
        ctx.renderer, ctx.model, ctx.noise = renderer, model, noise
        ctx.cfg = (Kc, Kf, Kfd, fine, float(renderer.depth_std), bool(renderer.white_bkgd))
        ctx.rays = rays.detach().contiguous().float()
        ctx.fwd = (res.coarse.z.reshape(R, Kc), res.fine.z.reshape(R, Kc + Kf) if fine else None,
                   res.coarse.depth.reshape(R))
        outs = [res.coarse.rgb, res.coarse.depth]
        if want_weights:
            outs.append(res.coarse.weights)
        if fine:
            outs += [res.fine.rgb, res.fine.depth]
            if want_weights:
                outs.append(res.fine.weights)
        ctx.set_materialize_grads(False)     # unused outputs arrive as None -> NULL (zero) in PnrRenderGrad
        ctx.layout = (want_weights, fine)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        renderer, model = ctx.renderer, ctx.model
        Kc, Kf, Kfd, fine, depth_std, white = ctx.cfg
        want_weights, _ = ctx.layout
        rays = ctx.rays
        dev = rays.device
        SB, B, _ = rays.shape
        R = SB * B
        names =["d_rgb_coarse", "d_depth_coarse"] + (["d_weights_coarse"] if want_weights else [])
        if fine:
            names += ["d_rgb_fine", "d_depth_fine"] + (["d_weights_fine"] if want_weights else [])
        widths = dict(d_rgb_coarse=3, d_depth_coarse=1, d_weights_coarse=Kc, d_rgb_fine=3, d_depth_fine=1,
                      d_weights_fine=Kc + Kf)
        up = {}          # the upstream tensors must outlive the library call
        for name, gr in zip(names, grads):
            if gr is not None:
                up[name] = gr.reshape(R, widths[name]).to(torch.float32).contiguous()
        scene, mc, mf, keep = model._scene_struct(want_fine=fine)
        mlps = [model.mlp_coarse] + ([model.mlp_fine] if (fine and model.mlp_fine is not None) else [])
        gdicts, gstructs = [], []
        for mlp in mlps:
            g = {k: torch.zeros_like(p, dtype=torch.float32, memory_format=torch.contiguous_format)
                 for k, p in mlp.named_parameters()}
            gdicts.append(g)
            gstructs.append(pn.make_mlp_struct(g, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                               mlp.combine_layer))
        V, C, Hl, Wl = model.encoder.latent.shape
        want_latent = ctx.needs_input_grad[5]
        d_latent = torch.zeros(V, Hl, Wl, C, dtype=torch.float32, device=dev) if want_latent else None
        noise = pn.PnrNoise()
        lin = renderer._lin_steps(Kc, dev)
        noise.lin_steps, noise.u_coarse = pn.dptr(lin), pn.dptr(ctx.noise["u_coarse"])
        if "n_depth" in ctx.noise:
            noise.n_depth = pn.dptr(ctx.noise["n_depth"])
        z_c, z_f, depth_c = ctx.fwd
        fwd = pn.PnrRenderOut()
        fwd.z_coarse, fwd.depth_coarse = pn.dptr(z_c.contiguous()), pn.dptr(depth_c.contiguous())
        if fine:
            fwd.z_fine = pn.dptr(z_f.contiguous())
        cfg = pn.PnrRenderCfg(Kc, Kf, Kfd, depth_std, 1 if white else 0, pn.ENGINES[model.engine])
        L = pn.lib()
        ug = pn.PnrRenderGrad()
        for name, t in up.items():
            setattr(ug, name, pn.dptr(t, name))
        nbytes = L.pnr_render_backward_workspace_bytes(scene, mc, mf, cfg, B)
        ws = pn.workspace(dev, nbytes)
        with torch.cuda.device(dev):
            pn.check(L.pnr_render_backward_ex(scene, mc, mf, cfg, pn.dptr(rays, "rays"), noise, fwd, ug, gstructs[0],
                                              gstructs[1] if len(gstructs) > 1 else None, pn.dptr(d_latent), B,
                                              ws.data_ptr(), ws.numel(), pn.stream_ptr(dev)))
        g_latent = d_latent.permute(0, 3, 1, 2) if want_latent else None
        flat = []
        for mlp, g in zip(mlps, gdicts):
            flat += [g[k] for k, _ in mlp.named_parameters()]
        return (None, None, None, None, None, g_latent) + tuple(flat)


def fused_render_train(renderer, model, rays, want_weights, noise_in=None):
    fine = bool(renderer.using_fine) and int(renderer.n_fine) > 0
    mlps = [model.mlp_coarse] + ([model.mlp_fine] if (fine and model.mlp_fine is not None) else [])
    params = [p for mlp in mlps for _, p in mlp.named_parameters()]
    latent = model.encoder.latent.detach() if model.stop_encoder_grad else model.encoder.latent
    outs = list(_FusedRender.apply(renderer, model, want_weights, noise_in, rays, latent, *params))
    res = DotMap()
    res.coarse = DotMap(rgb=outs.pop(0), depth=outs.pop(0))
    if want_weights:
        res.coarse.weights = outs.pop(0)
    if fine:
        res.fine = DotMap(rgb=outs.pop(0), depth=outs.pop(0))
        if want_weights:
            res.fine.weights = outs.pop(0)
    return res
