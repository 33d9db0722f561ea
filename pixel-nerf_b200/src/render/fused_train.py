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

Both nodes set up their forward call with render/fused_call.py, take the same inputs after their leading arguments
(`_apply`), and lay out their gradients in one zeroed buffer per device (`_grad_arena`).

Frozen MLP parameters (`requires_grad=False`: pose refinement, fine-tuning only some layers) cost nothing in the
backward.  Each node reads per parameter whether autograd wants its gradient; the arena then holds only the
wanted ones, the frozen ones stay NULL in the gradient structs and get None, and the call goes to the `_sel` entry
point (`pnr_render_backward_sel` / `pnr_mgpu_render_backward_sel`).  That skips a frozen tensor's weight-gradient GEMM,
its transposes and its bias sum, the input-gradient chain below the lowest trainable layer when no input gradient is
wanted, the latent and geometry backward when none of latent, rays or cameras is wanted, and a whole pass with nothing
to train or differentiate.  The wanted gradients are bit-equal to the full call's.  With every parameter trainable the
calls are exactly the ones described above, and so is the sharded node's call for a wholly frozen network (ray and
camera gradients only): that one still runs the full backward and drops the weight gradients.
"""
import ctypes as C

import torch

import pnr_native as pn

from . import fused_call as fc
from .dotmap_compat import DotMap
from .sharding import shard_bounds

_OUTPUTS = (("coarse", "rgb"), ("coarse", "depth"), ("coarse", "weights"),
            ("fine", "rgb"), ("fine", "depth"), ("fine", "weights"))


def _output_names(want_weights, fine):
    """(pass, quantity) of each output of a node, in the order it returns them."""
    return [(p, q) for p, q in _OUTPUTS if (fine or p == "coarse") and (want_weights or q != "weights")]


def _mlps(net, fine):
    return [net.mlp_coarse] + ([net.mlp_fine] if (fine and net.mlp_fine is not None) else [])


def _upstream(names, grads, dev):
    """PnrRenderGrad of the upstream gradients of the outputs `names`, as fp32 [R][width] on `dev`; outputs the loss
    does not use arrive as None and stay NULL.  -> (struct, the tensors it points at: they must outlive the call)."""
    ug, up = pn.PnrRenderGrad(), {}
    for (p, q), gr in zip(names, grads):
        if gr is not None:
            name = f"d_{q}_{p}"
            up[name] = gr.to(device=dev, dtype=torch.float32).flatten(0, 1).contiguous()
            setattr(ug, name, pn.dptr(up[name], name))
    return ug, up


def _grad_arena(net, fine, needs, wanted, dev):
    """One zeroed fp32 buffer on `dev` holding the gradient of every parameter of the MLPs the call runs that `wanted`
    (one bool per parameter, in the node's input order) asks for and, where `needs` (latent, poses, focal, c: four bools)
    asks, the channels-last latent gradient and the camera gradients, so that one kernel reduces a shard's whole
    gradient.  Every device gets the same layout.  -> (flat, [parameter gradient views in the order of the node's inputs,
    None where not wanted], (PnrMlp coarse, PnrMlp fine) with frozen tensors NULL, or None for a wholly frozen or absent
    MLP, latent view or None, (d_poses, d_focal, d_c) views or None, PnrCameraGrad or None when no camera gradient is
    asked for)."""
    mlps = _mlps(net, fine)
    V, Cc, Hl, Wl = net.encoder.latent.shape
    lat_shape = (V, Hl, Wl, Cc) if needs[0] else None
    cam_shapes = [t.shape if need else None for t, need in zip((net.poses, net.focal, net.c), needs[1:])]
    params = [p for mlp in mlps for p in mlp.parameters()]
    sizes = [p.numel() for p, w in zip(params, wanted) if w]
    lat_n = 0 if lat_shape is None else torch.Size(lat_shape).numel()
    cam_n = [0 if sh is None else torch.Size(sh).numel() for sh in cam_shapes]
    flat = torch.zeros(sum(sizes) + lat_n + sum(cam_n), dtype=torch.float32, device=dev)
    grads, structs, off, wanted = [], [], 0, iter(wanted)
    for mlp in mlps:
        g = {}
        for k, p in mlp.named_parameters():
            if next(wanted):
                g[k] = flat[off:off + p.numel()].view(p.shape)
                off += p.numel()
            grads.append(g.get(k))
        structs.append(pn.make_mlp_struct(g, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                          mlp.combine_layer) if g else None)
    lat = flat[off:off + lat_n].view(lat_shape) if lat_shape is not None else None
    off += lat_n
    cams = []
    for sh, k in zip(cam_shapes, cam_n):
        cams.append(flat[off:off + k].view(sh) if sh is not None else None)
        off += k
    cam = pn.PnrCameraGrad(*(pn.dptr(t) for t in cams)) if any(t is not None for t in cams) else None
    return flat, grads, (structs[0], structs[1] if len(structs) > 1 else None), lat, tuple(cams), cam


def _mlp_ref(struct):
    return C.byref(struct) if struct is not None else None


def _apply(node, lead, net, renderer, rays, want_weights, noise_in):
    """Runs autograd Function `node` on (*lead, want_weights, noise_in, rays, latent, poses, focal, c, *MLP parameters)
    -> DotMap like NeRFRenderer.forward."""
    pn.check_trainable(net.engine)
    fine = fc.sample_counts(renderer)[3]
    params = [p for mlp in _mlps(net, fine) for p in mlp.parameters()]
    latent = net.encoder.latent.detach() if net.stop_encoder_grad else net.encoder.latent
    outs = node.apply(*lead, want_weights, noise_in, rays, latent, net.poses, net.focal, net.c, *params)
    res = DotMap()
    for (p, q), t in zip(_output_names(want_weights, fine), outs):
        getattr(res, p)[q] = t
    return res


class _FusedRender(torch.autograd.Function):
    @staticmethod
    def forward(ctx, renderer, model, want_weights, noise_in, rays, latent, poses, focal, c, *params):
        SB, B, _ = rays.shape
        counts = fc.sample_counts(renderer)
        noise = fc.draw_noise(SB * B, counts, rays.device, noise_in)
        with torch.no_grad():
            res = renderer._forward_fused(model, rays, want_weights, noise_in=noise, want_z=True)
        ctx.renderer, ctx.model, ctx.noise, ctx.counts = renderer, model, noise, counts
        ctx.cfg = fc.render_cfg(renderer, model.engine)
        ctx.rays = rays.detach().contiguous().float()
        ctx.fwd = DotMap(coarse=DotMap(z=res.coarse.z, depth=res.coarse.depth))     # what the backward reads
        if counts[3]:
            ctx.fwd.fine = DotMap(z=res.fine.z)
        ctx.names = _output_names(want_weights, counts[3])
        ctx.set_materialize_grads(False)     # unused outputs arrive as None -> NULL (zero) in PnrRenderGrad
        return tuple(res[p][q] for p, q in ctx.names)

    @staticmethod
    def backward(ctx, *grads):
        renderer, model, rays = ctx.renderer, ctx.model, ctx.rays
        Kc, _, _, fine = ctx.counts
        dev = rays.device
        SB, B, _ = rays.shape
        ug, up = _upstream(ctx.names, grads, dev)
        scene, mc, mf, keep = model._scene_struct(want_fine=fine)
        wanted = ctx.needs_input_grad[9:]
        flat, pgrads, (gc, gf), d_latent, d_cam, cam = _grad_arena(model, fine, ctx.needs_input_grad[5:9], wanted, dev)
        noise = fc.bind_noise(renderer._lin_steps(Kc, dev), ctx.noise)
        fwd = fc.bind_outputs(ctx.fwd)
        L = pn.lib()
        d_rays = torch.empty(SB, B, 8, dtype=torch.float32, device=dev) if ctx.needs_input_grad[4] else None
        pn.sync_deterministic()
        ws = pn.workspace(dev, L.pnr_render_backward_workspace_bytes(scene, mc, mf, ctx.cfg, B))
        with torch.cuda.device(dev):
            if not all(wanted):      # part of the network is frozen
                pn.check(L.pnr_render_backward_sel(scene, mc, mf, ctx.cfg, pn.dptr(rays, "rays"), noise, fwd, ug,
                                                   _mlp_ref(gc), _mlp_ref(gf), pn.dptr(d_latent), pn.dptr(d_rays), cam,
                                                   B, ws.data_ptr(), ws.numel(), pn.stream_ptr(dev)))
            elif d_rays is None and cam is None:
                pn.check(L.pnr_render_backward_ex(scene, mc, mf, ctx.cfg, pn.dptr(rays, "rays"), noise, fwd, ug, gc, gf,
                                                  pn.dptr(d_latent), B, ws.data_ptr(), ws.numel(), pn.stream_ptr(dev)))
            else:
                pn.check(L.pnr_render_backward_cam(scene, mc, mf, ctx.cfg, pn.dptr(rays, "rays"), noise, fwd, ug, gc,
                                                   gf, pn.dptr(d_latent), pn.dptr(d_rays), cam, B, ws.data_ptr(),
                                                   ws.numel(), pn.stream_ptr(dev)))
        g_latent = d_latent.permute(0, 3, 1, 2) if d_latent is not None else None
        return (None, None, None, None, d_rays, g_latent) + d_cam + tuple(pgrads)


def fused_render_train(renderer, model, rays, want_weights, noise_in=None):
    return _apply(_FusedRender, (renderer, model), model, renderer, rays, want_weights, noise_in)


# ------------------------------------------------------------------------------------------
# several GPUs: bind_parallel(net, gpus) in grad mode
# ------------------------------------------------------------------------------------------
class _ShardedFusedRender(torch.autograd.Function):
    """The training step of `bind_parallel(net, gpus)` (the reference's DataParallel(dim=1) over the rays,
    train/train.py): pnr_mgpu_render over the shards, then pnr_mgpu_render_backward, which runs every shard's backward
    on its own GPU and sums the shards' gradients onto gpus[0].  Inputs and outputs live on gpus[0], so autograd
    continues into the encoder there."""

    @staticmethod
    def forward(ctx, sharded, want_weights, noise_in, rays, latent, poses, focal, c, *params):
        net, renderer = sharded.module.net, sharded.module.renderer
        counts = fc.sample_counts(renderer)
        dev0 = torch.device("cuda", sharded.gpus[0])
        rays0 = rays.detach().to(dev0).contiguous().float()
        SB, B, _ = rays0.shape
        cfg = fc.render_cfg(renderer, net.engine)
        out0, res0 = fc.render_outputs(SB, B, counts, dev0, want_weights, want_z=False)
        # the samples each shard's forward leaves on its GPU are the backward's input
        shards, stages, keep = fc.setup_shards(sharded, rays0, counts, cfg, want_weights, want_z=True,
                                               noise_in=noise_in)
        with torch.cuda.device(dev0):
            pn.check(pn.lib().pnr_mgpu_render(sharded._mgpu(), shards, cfg, pn.dptr(rays0, "rays"), out0, B,
                                              pn.stream_ptr(dev0)))
        ctx.sharded, ctx.shards, ctx.keep, ctx.stages = sharded, shards, keep, stages
        ctx.cfg, ctx.counts, ctx.dims, ctx.rays_device = cfg, counts, (SB, B), rays.device
        ctx.names = _output_names(want_weights, counts[3])
        ctx.set_materialize_grads(False)     # unused outputs arrive as None -> NULL (zero) in PnrRenderGrad
        return tuple(res0[p][q] for p, q in ctx.names)

    @staticmethod
    def backward(ctx, *grads):
        sharded, (SB, B), (Kc, Kf, _, fine) = ctx.sharded, ctx.dims, ctx.counts
        net = sharded.module.net
        gpus, n = sharded.gpus, len(sharded.gpus)
        dev0 = torch.device("cuda", gpus[0])
        L = pn.lib()
        ug, up = _upstream(ctx.names, grads, dev0)
        needs, wanted = ctx.needs_input_grad[4:8], ctx.needs_input_grad[8:]
        # A partly frozen network takes the selective driver.  A wholly frozen one (sharded pose refinement) keeps the
        # driver call it has always made, pnr_mgpu_render_backward_cam over full arenas, whose weight gradients are
        # then dropped.
        sel = any(wanted) and not all(wanted)
        layout = wanted if sel else (True,) * len(wanted)
        flat0, pgrads, (gc0, gf0), d_lat0, d_cam0, cam0 = _grad_arena(net, fine, needs, layout, dev0)
        want_rays = ctx.needs_input_grad[3]
        d_rays0 = torch.empty(SB, B, 8, dtype=torch.float32, device=dev0) if want_rays else None
        scs = (pn.PnrShardCam * n)()
        sgs = (pn.PnrShardGrad * n)()
        keep = [up, flat0]
        h = sharded._mgpu()
        bounds = shard_bounds(B, n)
        ws_bytes = {}
        pn.sync_deterministic()
        for i, (a, b) in enumerate(bounds):      # one workspace per device, sized for its largest shard
            if b - a > 0:
                sh = ctx.shards[i]
                nb = L.pnr_render_backward_workspace_bytes(sh.scene, sh.mlp_coarse, sh.mlp_fine, ctx.cfg, b - a)
                ws_bytes[gpus[i]] = max(ws_bytes.get(gpus[i], 0), nb)
        wss = {g: pn.workspace(torch.device("cuda", g), nb) for g, nb in ws_bytes.items()}
        for i, (a, b) in enumerate(bounds):
            Bi = b - a
            if Bi <= 0:
                continue
            dev = torch.device("cuda", gpus[i])
            st, rays_i = ctx.stages[i]
            sg = sgs[i]
            with torch.cuda.device(dev):
                sg.rays, sg.z_coarse, sg.depth_coarse = pn.dptr(rays_i), pn.dptr(st.coarse.z), pn.dptr(st.coarse.depth)
                sg.z_fine = pn.dptr(st.fine.z) if fine else None
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
                flat, _, (gc, gf), d_lat, _, cam = _grad_arena(net, fine, needs, layout, dev)
                if cam is not None:
                    scs[i].cam = cam
                sg.grad_coarse = C.pointer(gc) if gc is not None else None
                sg.grad_fine = C.pointer(gf) if gf is not None else None
                sg.d_latent_nhwc = pn.dptr(d_lat)
                sg.arena, sg.arena_count = pn.dptr(flat), flat.numel()
                keep += [flat, gc, gf]
            if not L.pnr_mgpu_peer_load(h, i):          # device 0 cannot read device i: stage the arena there
                stage0 = torch.empty_like(flat0)
                sg.arena_stage0 = pn.dptr(stage0)
                keep.append(stage0)
        keep.append(wss)
        with torch.cuda.device(dev0):
            if sel:
                pn.check(L.pnr_mgpu_render_backward_sel(h, ctx.shards, sgs, scs, ctx.cfg, ug, _mlp_ref(gc0),
                                                        _mlp_ref(gf0), pn.dptr(d_lat0), pn.dptr(d_rays0), cam0, B,
                                                        pn.stream_ptr(dev0)))
            elif d_rays0 is None and cam0 is None:
                pn.check(L.pnr_mgpu_render_backward(h, ctx.shards, sgs, ctx.cfg, ug, gc0, gf0, pn.dptr(d_lat0), B,
                                                    pn.stream_ptr(dev0)))
            else:
                pn.check(L.pnr_mgpu_render_backward_cam(h, ctx.shards, sgs, scs, ctx.cfg, ug, gc0, gf0,
                                                        pn.dptr(d_lat0), pn.dptr(d_rays0), cam0, B,
                                                        pn.stream_ptr(dev0)))
        sharded._keep_bwd = keep     # (the driver also orders every shard stream after the reduction)
        g_latent = d_lat0.permute(0, 3, 1, 2) if d_lat0 is not None else None
        g_rays = d_rays0.to(ctx.rays_device) if d_rays0 is not None else None
        return (None, None, None, g_rays, g_latent) + d_cam0 + tuple(g if w else None for g, w in zip(pgrads, wanted))


def sharded_render_train(sharded, rays, want_weights, noise_in=None):
    """Grad-mode forward of `_ShardedRender` (render/nerf.py) -> DotMap like NeRFRenderer.forward.  noise_in: optional
    dict(u_coarse, u_fine, u_fine_jit, n_depth) of full-ray draws [SB*B][...]; each shard takes its rays' rows (tests
    compare with the single-GPU node on the same draws)."""
    net = sharded.module.net
    return _apply(_ShardedFusedRender, (sharded,), net, sharded.module.renderer, rays, want_weights, noise_in)
