"""Fused forward + `pnr_render_backward` for a training step (SURVEY 8f-1), on one GPU or sharded over several.

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

The inputs are differentiable as in the reference's graph too: the rays (origin, direction, near, far) and the source
cameras `net.poses` / `net.focal` / `net.c` that encode() derived with torch ops from the poses, focal and c it was
given.  When any of them requires grad the backward is `pnr_render_backward_cam`, which also returns those gradients;
autograd carries the pose gradient on to the camera-to-world poses given to encode() (and, through `util.gen_rays`, to
the target poses of the rays).  So a frozen network can refine noisy poses.  Only the gradients autograd asks for are
computed; with none of them asked for the call is `pnr_render_backward_ex`, unchanged.  `image_shape` and
`latent_scaling` are buffers and get no gradient, as in the reference.

`bind_parallel(net, gpus)` with several GPUs trains through `_ShardedFusedRender` below: the rays are sharded as by
the reference's DataParallel(dim=1), every GPU renders and differentiates its shard, and the shards' gradients are
summed onto gpus[0] (pnr_mgpu_render / pnr_mgpu_render_backward, csrc/pnr_mgpu.cu); with ray or camera gradients
pnr_mgpu_render_backward_cam, whose camera gradients sit in the same per-shard arenas and are reduced with them.
"""
import torch

import pnr_native as pn

from .dotmap_compat import DotMap


class _FusedRender(torch.autograd.Function):
    @staticmethod
    def forward(ctx, renderer, model, want_weights, noise_in, rays, latent, poses, focal, c, *params):
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
        d_rays = torch.empty(SB, B, 8, dtype=torch.float32, device=dev) if ctx.needs_input_grad[4] else None
        cam, d_cam = pn.camera_grad(model, ctx.needs_input_grad[6:9], dev)
        pn.sync_deterministic()
        nbytes = L.pnr_render_backward_workspace_bytes(scene, mc, mf, cfg, B)
        ws = pn.workspace(dev, nbytes)
        gfine = gstructs[1] if len(gstructs) > 1 else None
        with torch.cuda.device(dev):
            if d_rays is None and cam is None:
                pn.check(L.pnr_render_backward_ex(scene, mc, mf, cfg, pn.dptr(rays, "rays"), noise, fwd, ug,
                                                  gstructs[0], gfine, pn.dptr(d_latent), B, ws.data_ptr(), ws.numel(),
                                                  pn.stream_ptr(dev)))
            else:
                pn.check(L.pnr_render_backward_cam(scene, mc, mf, cfg, pn.dptr(rays, "rays"), noise, fwd, ug,
                                                   gstructs[0], gfine, pn.dptr(d_latent), pn.dptr(d_rays), cam, B,
                                                   ws.data_ptr(), ws.numel(), pn.stream_ptr(dev)))
        g_latent = d_latent.permute(0, 3, 1, 2) if want_latent else None
        flat = []
        for mlp, g in zip(mlps, gdicts):
            flat += [g[k] for k, _ in mlp.named_parameters()]
        return (None, None, None, None, d_rays, g_latent) + d_cam + tuple(flat)



def fused_render_train(renderer, model, rays, want_weights, noise_in=None):
    pn.check_trainable(model.engine)
    fine = bool(renderer.using_fine) and int(renderer.n_fine) > 0
    mlps = [model.mlp_coarse] + ([model.mlp_fine] if (fine and model.mlp_fine is not None) else [])
    params = [p for mlp in mlps for _, p in mlp.named_parameters()]
    latent = model.encoder.latent.detach() if model.stop_encoder_grad else model.encoder.latent
    outs = list(_FusedRender.apply(renderer, model, want_weights, noise_in, rays, latent, model.poses, model.focal,
                                   model.c, *params))
    res = DotMap()
    res.coarse = DotMap(rgb=outs.pop(0), depth=outs.pop(0))
    if want_weights:
        res.coarse.weights = outs.pop(0)
    if fine:
        res.fine = DotMap(rgb=outs.pop(0), depth=outs.pop(0))
        if want_weights:
            res.fine.weights = outs.pop(0)
    return res


# ------------------------------------------------------------------------------------------
# several GPUs: bind_parallel(net, gpus) in grad mode
# ------------------------------------------------------------------------------------------
_WIDTHS = ("d_rgb_coarse", "d_depth_coarse", "d_weights_coarse", "d_rgb_fine", "d_depth_fine", "d_weights_fine")


def _grad_arena(mlps, latent_shape, dev, cam_shapes=(None, None, None)):
    """One zeroed fp32 buffer on `dev` holding every parameter gradient of `mlps`, (latent_shape not None) the
    channels-last latent gradient and the camera gradients of `cam_shapes` (poses, focal, c; None = not wanted), so
    that one kernel reduces a shard's whole gradient -> (flat, [dict per mlp], [PnrMlp per mlp], latent view or None,
    (d_poses, d_focal, d_c) views or None).  Every device gets the same layout."""
    sizes = [p.numel() for mlp in mlps for _, p in mlp.named_parameters()]
    lat_n = 0 if latent_shape is None else torch.Size(latent_shape).numel()
    cam_n = [0 if sh is None else torch.Size(sh).numel() for sh in cam_shapes]
    flat = torch.zeros(sum(sizes) + lat_n + sum(cam_n), dtype=torch.float32, device=dev)
    dicts, structs, off = [], [], 0
    for mlp in mlps:
        g = {}
        for k, p in mlp.named_parameters():
            g[k] = flat[off:off + p.numel()].view(p.shape)
            off += p.numel()
        dicts.append(g)
        structs.append(pn.make_mlp_struct(g, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                          mlp.combine_layer))
    lat = flat[off:off + lat_n].view(latent_shape) if latent_shape is not None else None
    off += lat_n
    cams = []
    for sh, k in zip(cam_shapes, cam_n):
        cams.append(flat[off:off + k].view(sh) if sh is not None else None)
        off += k
    return flat, dicts, structs, lat, tuple(cams)


class _ShardedFusedRender(torch.autograd.Function):
    """The training step of `bind_parallel(net, gpus)` (the reference's DataParallel(dim=1) over the rays,
    train/train.py): pnr_mgpu_render over the shards, then pnr_mgpu_render_backward, which runs every shard's backward
    on its own GPU and sums the shards' gradients onto gpus[0].  Inputs and outputs live on gpus[0], so autograd
    continues into the encoder there."""

    @staticmethod
    def forward(ctx, sharded, want_weights, noise_in, rays, latent, poses, focal, c, *params):
        import ctypes as C
        net, renderer = sharded.module.net, sharded.module.renderer
        L = pn.lib()
        Kc, Kf, Kfd = int(renderer.n_coarse), int(renderer.n_fine), int(renderer.n_fine_depth)
        fine = bool(renderer.using_fine) and Kf > 0
        if not fine:
            Kf = Kfd = 0
        gpus, n = sharded.gpus, len(sharded.gpus)
        dev0 = torch.device("cuda", gpus[0])
        rays0 = rays.detach().to(dev0).contiguous().float()
        SB, B, _ = rays0.shape
        R = SB * B
        cfg = pn.PnrRenderCfg(Kc, Kf, Kfd, float(renderer.depth_std), 1 if renderer.white_bkgd else 0,
                              pn.ENGINES[net.engine])
        f32 = dict(dtype=torch.float32, device=dev0)
        out0 = pn.PnrRenderOut()
        names = [("coarse", "rgb", 3), ("coarse", "depth", 0)] + ([("coarse", "weights", Kc)] if want_weights else [])
        if fine:
            names += [("fine", "rgb", 3), ("fine", "depth", 0)] + ([("fine", "weights", Kc + Kf)] if want_weights else [])
        outs = []
        for p, q, w in names:
            t = torch.empty(SB, B, w, **f32) if w else torch.empty(SB, B, **f32)
            setattr(out0, f"{q}_{p}", pn.dptr(t))
            outs.append(t)
        shards = (pn.PnrShard * n)()
        keep, stages = [rays0], {}
        per = -(-B // n)
        bounds = [(min(B, per * i), min(B, per * (i + 1))) for i in range(n)]
        for i, g in enumerate(gpus):
            a, b = bounds[i]
            Bi = b - a
            if Bi <= 0:
                continue
            dev = torch.device("cuda", g)
            model = net
            if i > 0:
                model = sharded._replicas[g]
                sharded._refresh(model, fine)
            with torch.cuda.device(dev):
                scene, mc, mf, keep2 = model._scene_struct(want_fine=fine)
                Ri = SB * Bi
                f32i = dict(dtype=torch.float32, device=dev)
                if noise_in is not None:      # tests replay full-ray draws: each shard takes its rays' rows
                    nz = {k: v.reshape(SB, B, -1)[:, a:b].reshape(Ri, -1).to(**f32i).contiguous()
                          for k, v in noise_in.items()}
                else:                         # device i's own generator, in the reference's draw order
                    nz = {"u_coarse": torch.rand(Ri, Kc, **f32i)}
                    if fine and Kf - Kfd > 0:
                        nz["u_fine"] = torch.rand(Ri, Kf - Kfd, **f32i)
                        nz["u_fine_jit"] = torch.rand(Ri, Kf - Kfd, **f32i)
                    if fine and Kfd > 0:
                        nz["n_depth"] = torch.randn(Ri, Kfd, **f32i)
                noise = pn.PnrNoise()
                lin = renderer._lin_steps(Kc, dev)
                noise.lin_steps, noise.u_coarse = pn.dptr(lin), pn.dptr(nz["u_coarse"])
                if fine and Kf - Kfd > 0:
                    noise.u_fine, noise.u_fine_jit = pn.dptr(nz["u_fine"]), pn.dptr(nz["u_fine_jit"])
                if fine and Kfd > 0:
                    noise.n_depth = pn.dptr(nz["n_depth"])
                # local outputs; the samples stay here for the backward
                st = {"rgb_coarse": torch.empty(Ri, 3, **f32i), "depth_coarse": torch.empty(Ri, **f32i),
                      "z_coarse": torch.empty(Ri, Kc, **f32i)}
                if want_weights:
                    st["weights_coarse"] = torch.empty(Ri, Kc, **f32i)
                if fine:
                    st.update(rgb_fine=torch.empty(Ri, 3, **f32i), depth_fine=torch.empty(Ri, **f32i),
                              z_fine=torch.empty(Ri, Kc + Kf, **f32i))
                    if want_weights:
                        st["weights_fine"] = torch.empty(Ri, Kc + Kf, **f32i)
                stage = pn.PnrRenderOut()
                for k, t in st.items():
                    setattr(stage, k, pn.dptr(t))
                ws = pn.workspace(dev, L.pnr_render_workspace_bytes(scene, mc, mf, cfg, Bi))
                sh = shards[i]
                sh.scene, sh.mlp_coarse = C.pointer(scene), C.pointer(mc)
                sh.mlp_fine = C.pointer(mf) if mf is not None else None
                sh.noise = C.pointer(noise)
                sh.workspace, sh.workspace_bytes = ws.data_ptr(), ws.numel()
                rays_i = rays0
                if i > 0 or SB > 1:
                    rays_i = torch.empty(SB, Bi, 8, **f32i)
                    sh.rays_stage = pn.dptr(rays_i)
                sh.stage = stage
                sh.stream = pn.stream_ptr(dev)
                stages[i] = (st, rays_i)
                keep += [lin, nz, keep2, scene, mc, mf, noise, ws]
        with torch.cuda.device(dev0):
            pn.check(L.pnr_mgpu_render(sharded._mgpu(), shards, cfg, pn.dptr(rays0, "rays"), out0, B,
                                       pn.stream_ptr(dev0)))
        ctx.sharded, ctx.shards, ctx.keep, ctx.stages, ctx.bounds = sharded, shards, keep, stages, bounds
        ctx.cfg, ctx.dims, ctx.rays_device = cfg, (SB, B, Kc, Kf, fine), rays.device
        ctx.layout = [f"d_{q}_{p}" for p, q, _ in names]
        ctx.set_materialize_grads(False)     # unused outputs arrive as None -> NULL (zero) in PnrRenderGrad
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        import ctypes as C
        sharded, (SB, B, Kc, Kf, fine) = ctx.sharded, ctx.dims
        net = sharded.module.net
        gpus, n = sharded.gpus, len(sharded.gpus)
        dev0 = torch.device("cuda", gpus[0])
        L = pn.lib()
        R = SB * B
        up, ug = {}, pn.PnrRenderGrad()       # the upstream tensors must outlive the library call
        for name, gr in zip(ctx.layout, grads):
            if gr is not None:
                up[name] = gr.to(device=dev0, dtype=torch.float32).reshape(R, -1).contiguous()
                setattr(ug, name, pn.dptr(up[name], name))
        mlps = [net.mlp_coarse] + ([net.mlp_fine] if (fine and net.mlp_fine is not None) else [])
        V, Cc, Hl, Wl = net.encoder.latent.shape
        lat_shape = (V, Hl, Wl, Cc) if ctx.needs_input_grad[4] else None
        cam_shapes = tuple(t.shape if need else None
                           for t, need in zip((net.poses, net.focal, net.c), ctx.needs_input_grad[5:8]))
        flat0, gdicts, gstructs, d_lat0, d_cam0 = _grad_arena(mlps, lat_shape, dev0, cam_shapes)
        want_rays = ctx.needs_input_grad[3]
        d_rays0 = torch.empty(SB, B, 8, dtype=torch.float32, device=dev0) if want_rays else None
        cam0 = None
        if any(t is not None for t in d_cam0):
            cam0 = pn.PnrCameraGrad(*(pn.dptr(t) for t in d_cam0))
        scs = (pn.PnrShardCam * n)()
        sgs = (pn.PnrShardGrad * n)()
        keep = [up, flat0]
        h = sharded._mgpu()
        ws_bytes = {}
        pn.sync_deterministic()
        for i, (a, b) in enumerate(ctx.bounds):      # one workspace per device, sized for its largest shard
            if b - a > 0:
                sh = ctx.shards[i]
                nb = L.pnr_render_backward_workspace_bytes(sh.scene, sh.mlp_coarse, sh.mlp_fine, ctx.cfg, b - a)
                ws_bytes[gpus[i]] = max(ws_bytes.get(gpus[i], 0), nb)
        wss = {g: pn.workspace(torch.device("cuda", g), nb) for g, nb in ws_bytes.items()}
        for i, (a, b) in enumerate(ctx.bounds):
            Bi = b - a
            if Bi <= 0:
                continue
            dev = torch.device("cuda", gpus[i])
            st, rays_i = ctx.stages[i]
            sg = sgs[i]
            with torch.cuda.device(dev):
                sg.rays, sg.z_coarse, sg.depth_coarse = pn.dptr(rays_i), pn.dptr(st["z_coarse"]), pn.dptr(st["depth_coarse"])
                sg.z_fine = pn.dptr(st.get("z_fine"))
                if up and (i > 0 or SB > 1):
                    stage = torch.empty(SB * Bi * (8 + 2 * Kc + Kf), dtype=torch.float32, device=dev)
                    sg.up_stage = pn.dptr(stage)
                    keep.append(stage)
                ws = wss[gpus[i]]
                sg.workspace, sg.workspace_bytes = ws.data_ptr(), ws.numel()
                sg.stream = pn.stream_ptr(dev)
                if want_rays and (i > 0 or SB > 1):      # the shard's ray gradients, un-staged onto gpus[0]
                    dr = torch.empty(SB, Bi, 8, dtype=torch.float32, device=dev)
                    scs[i].d_rays = pn.dptr(dr)
                    keep.append(dr)
                if i == 0:
                    sg.arena, sg.arena_count = pn.dptr(flat0), flat0.numel()
                    continue
                flat, _, structs, d_lat, d_cam = _grad_arena(mlps, lat_shape, dev, cam_shapes)
                scs[i].cam = pn.PnrCameraGrad(*(pn.dptr(t) for t in d_cam))
                sg.grad_coarse = C.pointer(structs[0])
                sg.grad_fine = C.pointer(structs[1]) if len(structs) > 1 else None
                sg.d_latent_nhwc = pn.dptr(d_lat)
                sg.arena, sg.arena_count = pn.dptr(flat), flat.numel()
                keep += [flat, structs]
            if not L.pnr_mgpu_peer_load(h, i):          # device 0 cannot read device i: stage the arena there
                stage0 = torch.empty_like(flat0)
                sg.arena_stage0 = pn.dptr(stage0)
                keep.append(stage0)
        keep.append(wss)
        gfine = gstructs[1] if len(gstructs) > 1 else None
        with torch.cuda.device(dev0):
            if d_rays0 is None and cam0 is None:
                pn.check(L.pnr_mgpu_render_backward(h, ctx.shards, sgs, ctx.cfg, ug, gstructs[0], gfine,
                                                    pn.dptr(d_lat0), B, pn.stream_ptr(dev0)))
            else:
                pn.check(L.pnr_mgpu_render_backward_cam(h, ctx.shards, sgs, scs, ctx.cfg, ug, gstructs[0], gfine,
                                                        pn.dptr(d_lat0), pn.dptr(d_rays0), cam0, B,
                                                        pn.stream_ptr(dev0)))
        sharded._keep_bwd = keep     # (the driver also orders every shard stream after the reduction)
        g_latent = d_lat0.permute(0, 3, 1, 2) if d_lat0 is not None else None
        flat = []
        for mlp, g in zip(mlps, gdicts):
            flat += [g[k] for k, _ in mlp.named_parameters()]
        g_rays = d_rays0.to(ctx.rays_device) if d_rays0 is not None else None
        return (None, None, None, g_rays, g_latent) + d_cam0 + tuple(flat)


def sharded_render_train(sharded, rays, want_weights, noise_in=None):
    """Grad-mode forward of `_ShardedRender` (render/nerf.py) -> DotMap like NeRFRenderer.forward.  noise_in: optional
    dict(u_coarse, u_fine, u_fine_jit, n_depth) of full-ray draws [SB*B][...]; each shard takes its rays' rows (tests
    compare with the single-GPU node on the same draws)."""
    net, renderer = sharded.module.net, sharded.module.renderer
    pn.check_trainable(net.engine)
    fine = bool(renderer.using_fine) and int(renderer.n_fine) > 0
    mlps = [net.mlp_coarse] + ([net.mlp_fine] if (fine and net.mlp_fine is not None) else [])
    params = [p for mlp in mlps for _, p in mlp.named_parameters()]
    latent = net.encoder.latent.detach() if net.stop_encoder_grad else net.encoder.latent
    outs = list(_ShardedFusedRender.apply(sharded, want_weights, noise_in, rays, latent, net.poses, net.focal, net.c,
                                          *params))
    res = DotMap()
    res.coarse = DotMap(rgb=outs.pop(0), depth=outs.pop(0))
    if want_weights:
        res.coarse.weights = outs.pop(0)
    if fine:
        res.fine = DotMap(rgb=outs.pop(0), depth=outs.pop(0))
        if want_weights:
            res.fine.weights = outs.pop(0)
    return res
