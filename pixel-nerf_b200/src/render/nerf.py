"""
NeRFRenderer with the reference's surface (src/render/nerf.py): `from_conf`, `forward(model,
rays, want_weights)`, `bind_parallel(net, gpus, simple_output)`, `sched_step`, mutable
`n_coarse / n_fine / using_fine / eval_batch_size`, persistent `iter_idx / last_sched`.

Inference with a PixelNeRFNet on CUDA runs the whole sample -> field -> composite ->
resample -> field -> composite chain in one C-ABI call (`pnr_render`, include/pnr.h); the
random draws are made with torch, in the reference's order, and handed to the kernels,
so a seeded run replays the reference's samples.  render/fused_call.py sets up that call (counts,
draws, outputs, shards) for every caller.  With autograd enabled (training) on CUDA the
same fused forward runs inside one autograd node whose backward is `pnr_render_backward_ex`
(render/fused_train.py), differentiable in rgb, depth and weights like the reference; a foreign
`model` callable, CPU tensors in grad mode (host-logic tests) or PNR_FUSED_BACKWARD=0 use the
composed torch path below.  `NeRFRenderer._apply_sched` and `_fused_grad` hold the schedule and
the choice of that node for both `NeRFRenderer.forward` and `_ShardedRender`.

Multi-GPU (`bind_parallel(net, gpus)`): the reference wraps a `DataParallel(dim=1)`, which
re-broadcasts the whole module on every call; `_ShardedRender` instead keeps a `_SceneReplica`
(peer copies of the already-derived device state) per extra GPU, refreshed only when
encode()/weights change, and slices rays with torch.chunk semantics, so ray order in the
gathered output is identical.  In grad mode the shards also run their own backward and their
gradients are summed onto gpus[0] (render/fused_train.py).
"""
import os
import warnings

import torch

import pnr_native as pn

from . import fused_call as fc
from .dotmap_compat import DotMap


# ------------------------------------------------------------------------------------------
# composed torch path (autograd / generic model callables)
# ------------------------------------------------------------------------------------------
def _stratified(rays, n, u):
    near, far = rays[:, 6:7], rays[:, 7:8]
    s = torch.linspace(0, 1 - 1.0 / n, n, device=rays.device).unsqueeze(0).repeat(rays.shape[0], 1)
    s = s + u * (1.0 / n)
    return near * (1 - s) + far * s


def _importance(rays, weights, u, jitter, n_coarse):
    w = weights.detach() + 1e-5
    cdf = torch.cumsum(w / torch.sum(w, -1, keepdim=True), -1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    bins = torch.clamp_min(torch.searchsorted(cdf, u, right=True).float() - 1.0, 0.0)
    s = (bins + jitter) / n_coarse
    near, far = rays[:, 6:7], rays[:, 7:8]
    return near * (1 - s) + far * s


def _around_depth(rays, depth, noise, std):
    z = depth.unsqueeze(1).repeat((1, noise.shape[1])) + noise * std
    return torch.max(torch.min(z, rays[:, 7:8]), rays[:, 6:7])


def _integrate(rays, z, field, white_bkgd):
    delta = torch.cat([z[:, 1:] - z[:, :-1], rays[:, 7:8] - z[:, -1:]], -1)
    alpha = 1 - torch.exp(-delta * torch.relu(field[..., 3]))
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], -1), -1)
    w = alpha * trans[:, :-1]
    rgb = torch.sum(w.unsqueeze(-1) * field[..., :3], -2)
    depth = torch.sum(w * z, -1)
    if white_bkgd:
        rgb = rgb + 1 - w.sum(dim=1).unsqueeze(-1)
    return w, rgb, depth


def _wrapper_output(renderer, outputs, simple_output):
    """(rgb, depth) of the best pass, or the plain nested dict (nerf.py:31-42)."""
    if simple_output:
        best = outputs.fine if renderer.using_fine else outputs.coarse
        return best.rgb, best.depth
    return outputs.toDict()


class _RenderWrapper(torch.nn.Module):
    """Callable returned by bind_parallel (nerf.py:15-42)."""

    def __init__(self, net, renderer, simple_output):
        super().__init__()
        self.net = net
        self.renderer = renderer
        self.simple_output = simple_output

    def forward(self, rays, want_weights=False):
        if rays.shape[0] == 0:
            return torch.zeros(0, 3, device=rays.device), torch.zeros(0, device=rays.device)
        outputs = self.renderer(self.net, rays, want_weights=want_weights and not self.simple_output)
        return _wrapper_output(self.renderer, outputs, self.simple_output)


def broadcast_to(gpus, t, dev, handle):
    """A copy on `dev` of the buffer `t` on gpus[0], through pnr_mgpu_broadcast on the handle `handle()` of `gpus`
    (peer copy over NVLink, enqueued on torch's current streams so the caching allocator's stream ordering holds)."""
    import ctypes as C
    n = len(gpus)
    t = t.contiguous()
    with torch.cuda.device(dev):
        dst = torch.empty_like(t, device=dev)
    ptrs, streams = (C.c_void_p * n)(), (C.c_void_p * n)()
    for i, g in enumerate(gpus):
        streams[i] = torch.cuda.current_stream(torch.device("cuda", g)).cuda_stream
        if g == dev.index:
            ptrs[i] = dst.data_ptr()
    pn.check(pn.lib().pnr_mgpu_broadcast(handle(), C.c_void_p(t.data_ptr()), ptrs, t.numel() * t.element_size(),
                                         streams))
    return dst


class _SceneReplica:
    """Everything the fused render path reads, on ANOTHER GPU of the same process: channels-last latent, cameras, fp32
    weights, packed tensor-engine weights and projected maps.  Filled by peer copies (NVLink) of the primary device's
    ALREADY DERIVED buffers -- no module deepcopy, no re-pack, no re-projection -- and refreshed only when the weights
    (parameter versions) or the scene (`net._scene_epoch`, latent version) change.  The reference's DataParallel
    re-broadcasts the whole module on every forward call instead (src/render/nerf.py:370)."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.engine = "auto"
        self.mlp, self.mlp_key = {}, {}
        self.scene_key = None
        self.refreshes = 0          # (weights, scene) copies made so far: tests and DESIGN.md quote it

    def refresh(self, net, want_fine, send=None):
        """send(tensor, device) -> copy on `device`; default torch's `.to` (a peer copy as well).  `_ShardedRender` passes
        a sender built on pnr_mgpu_broadcast for the large buffers."""
        from model.models import _param_key
        dev = self.device
        if send is None:
            send = lambda t, d: t.to(d, non_blocking=True)
        self.engine = net.engine
        names = ["mlp_coarse"] + (["mlp_fine"] if (want_fine and net.mlp_fine is not None) else [])
        scene0, _, _, (nhwc0, proj0) = net._scene_struct(want_fine=want_fine)   # primary: packs / projects if stale
        for name in names:
            mlp = getattr(net, name)
            key = _param_key(mlp)
            if self.mlp_key.get(name) == key:
                continue
            _, _, sd0, packed0 = net._fused.mlp[name]
            sd = {k: v.to(dev, non_blocking=True) for k, v in sd0.items()}
            packed = send(packed0, dev) if packed0 is not None else None
            struct = pn.make_mlp_struct(sd, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                        mlp.combine_layer, packed=packed)
            self.mlp[name], self.mlp_key[name] = (struct, sd, packed), key
            self.refreshes += 1
        lat = net.encoder.latent
        skey = (net._scene_epoch, lat.data_ptr(), lat._version, tuple(self.mlp_key.get(n) for n in names), want_fine)
        if skey != self.scene_key:
            to = lambda t: None if t is None else t.to(dev, non_blocking=True)
            big = lambda t: None if t is None else send(t, dev)
            self.nhwc = big(nhwc0)
            self.proj = {k: big(v) for k, v in proj0.items()}
            self.poses, self.focal, self.c = to(net.poses), to(net.focal), to(net.c)
            self.meta = (scene0.SB, scene0.NS, scene0.image_w, scene0.image_h, scene0.scale_x, scene0.scale_y)
            self.scene_key = skey
            self.refreshes += 1

    def _scene_struct(self, want_fine):
        SB, NS, w, h, sx, sy = self.meta
        mc = self.mlp["mlp_coarse"][0]
        mf = self.mlp["mlp_fine"][0] if (want_fine and "mlp_fine" in self.mlp) else None
        scene = pn.make_scene_struct(self.nhwc, self.poses, self.focal, self.c, SB, NS, w, h, sx, sy,
                                     proj_coarse=self.proj.get("mlp_coarse"), proj_fine=self.proj.get("mlp_fine"))
        return scene, mc, mf, (self.nhwc, self.proj)


class _ShardedRender(torch.nn.Module):
    """Single-process ray sharding over several GPUs (replaces nn.DataParallel(dim=1), nerf.py:368-370) on the C-ABI
    driver `pnr_mgpu_*` (csrc/pnr_mgpu.cu).  Shard i gets torch.chunk piece i of the rays along dim 1 (same ray order as
    DataParallel); one host thread enqueues, per GPU, the peer copy of its rays, ONE fused render launch and the return
    of its pixels -- for a single object the kernels store the final rgb / depth straight into the output tensors on
    gpus[0] through peer memory.  GPUs other than gpus[0] render from a `_SceneReplica`; every GPU draws its samples
    from its own generator (as under DataParallel).

    Gradient mode (train/train.py with several --gpu_id): one autograd node on gpus[0] (render/fused_train.py,
    `_ShardedFusedRender`) runs the same sharded forward and then `pnr_mgpu_render_backward`: every GPU differentiates
    its own shard from the samples its forward left there, and one kernel on gpus[0] sums the shards' weight and latent
    gradients onto gpus[0]'s, so autograd continues into the encoder there as under DataParallel.  The optimizer step
    and encode() change the weights and the scene on every step, so every step refreshes the replicas.  Other models,
    CPU rays or PNR_FUSED_BACKWARD=0/1 run the step on gpus[0] alone, with a one-time warning.  Gradients of the rays
    and the cameras (poses, focal, c) are sharded too (pnr_mgpu_render_backward_cam)."""

    def __init__(self, wrapped, gpus):
        super().__init__()
        self.module = wrapped
        self.gpus = [int(g) for g in gpus]
        self._replicas = {g: _SceneReplica(torch.device("cuda", g)) for g in self.gpus[1:]}
        self._warned = False
        self._handle = None
        self._keep, self._keep_bwd = [], []
        self.timing = None          # dict: CUDA event pairs of each replica refresh are appended to timing["refresh"]

    def _mgpu(self):
        if self._handle is None:
            import ctypes as C
            h = C.c_void_p()
            ids = (C.c_int32 * len(self.gpus))(*self.gpus)
            pn.check(pn.lib().pnr_mgpu_create(ids, len(self.gpus), C.byref(h)))
            self._handle = h
        return self._handle

    def _send(self, t, dev):
        """One buffer of the primary device to `dev` through pnr_mgpu_broadcast (see `broadcast_to`)."""
        return broadcast_to(self.gpus, t, dev, self._mgpu)

    def __del__(self):
        try:
            if self._handle is not None:
                pn.lib().pnr_mgpu_destroy(self._handle)
        except Exception:
            pass

    def _refresh(self, replica, want_fine):
        """Bring `replica` up to the primary's weights and scene (no-op when neither changed)."""
        t = self.timing
        if t is not None:
            ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev[0].record(torch.cuda.current_stream(torch.device("cuda", self.gpus[0])))
        replica.refresh(self.module.net, want_fine, send=self._send)
        if t is not None:
            ev[1].record(torch.cuda.current_stream(torch.device("cuda", self.gpus[0])))
            t.setdefault("refresh", []).append(ev)

    def forward(self, rays, want_weights=False):
        net, renderer, simple = self.module.net, self.module.renderer, self.module.simple_output
        empty = rays.shape[0] == 0 or rays.shape[1] == 0
        grad = not empty and net._needs_autograd(rays)
        if empty or (grad and not renderer._fused_grad(net, rays)):
            if grad and not self._warned:
                warnings.warn(f"bind_parallel(net, {self.gpus}): gradients are required and this model / setting has "
                              f"no sharded backward (it needs a PixelNeRFNet, CUDA rays and PNR_FUSED_BACKWARD unset, "
                              f"auto or 2), so this call runs on cuda:{self.gpus[0]} only")
                self._warned = True
            return self.module(rays, want_weights=want_weights)
        renderer._apply_sched()
        want_weights = want_weights and not simple
        if grad:
            from .fused_train import sharded_render_train
            return _wrapper_output(renderer, sharded_render_train(self, rays, want_weights), simple)
        counts = fc.sample_counts(renderer)
        dev0 = torch.device("cuda", self.gpus[0])
        rays0 = rays.detach().to(dev0).contiguous().float()
        SB, B, _ = rays0.shape
        cfg = fc.render_cfg(renderer, net.engine)
        out0, res0 = fc.render_outputs(SB, B, counts, dev0, want_weights, want_z=False)
        if simple and counts[3]:          # only the best pass is returned: do not ship the other one back
            out0.rgb_coarse = out0.depth_coarse = None
        shards, _, keep = fc.setup_shards(self, rays0, counts, cfg, want_weights, want_z=False)
        with torch.cuda.device(dev0):
            pn.check(pn.lib().pnr_mgpu_render(self._mgpu(), shards, cfg, pn.dptr(rays0, "rays"), out0, B,
                                              pn.stream_ptr(dev0)))
        self._keep = keep        # staging buffers stay referenced until the next call (their streams are still busy)
        return _wrapper_output(renderer, res0, simple)


class NeRFRenderer(torch.nn.Module):
    def __init__(self, n_coarse=128, n_fine=0, n_fine_depth=0, noise_std=0.0, depth_std=0.01,
                 eval_batch_size=100000, white_bkgd=False, lindisp=False, sched=None):
        super().__init__()
        if lindisp:
            raise NotImplementedError("lindisp = True is not supported (no shipped dataset uses it)")
        self.n_coarse, self.n_fine, self.n_fine_depth = n_coarse, n_fine, n_fine_depth
        self.noise_std, self.depth_std = noise_std, depth_std
        self.eval_batch_size = eval_batch_size
        self.white_bkgd = white_bkgd
        self.lindisp = lindisp
        self.using_fine = n_fine > 0
        self.sched = sched if (sched is not None and len(sched) > 0) else None
        self.register_buffer("iter_idx", torch.tensor(0, dtype=torch.long), persistent=True)
        self.register_buffer("last_sched", torch.tensor(0, dtype=torch.long), persistent=True)
        self._lin_cache = {}

    # -- sampling helpers with the reference's names (used by the torch path and by callers) --
    def sample_coarse(self, rays):
        return _stratified(rays, self.n_coarse, torch.rand(rays.shape[0], self.n_coarse, device=rays.device))

    def sample_fine(self, rays, weights):
        B, n = rays.shape[0], self.n_fine - self.n_fine_depth
        u = torch.rand(B, n, dtype=torch.float32, device=rays.device)
        return _importance(rays, weights, u, torch.rand_like(u), self.n_coarse)

    def sample_fine_depth(self, rays, depth):
        noise = torch.randn(rays.shape[0], self.n_fine_depth, device=rays.device)
        return _around_depth(rays, depth, noise, self.depth_std)

    def composite(self, model, rays, z_samp, coarse=True, sb=0):
        """Query `model` at the samples in point chunks and integrate (nerf.py:163-249)."""
        B, K = z_samp.shape
        pts = rays[:, None, :3] + z_samp.unsqueeze(2) * rays[:, None, 3:6]
        dirs = rays[:, None, 3:6].expand(-1, K, -1)
        if sb > 0:
            pts, dirs, dim, chunk = pts.reshape(sb, -1, 3), dirs.reshape(sb, -1, 3), 1, (self.eval_batch_size - 1) // sb + 1
        else:
            pts, dirs, dim, chunk = pts.reshape(-1, 3), dirs.reshape(-1, 3), 0, self.eval_batch_size
        use_dirs = getattr(model, "use_viewdirs", False)
        vals = []
        for p, d in zip(torch.split(pts, chunk, dim=dim), torch.split(dirs, chunk, dim=dim)):
            vals.append(model(p, coarse=coarse, viewdirs=d) if use_dirs else model(p, coarse=coarse))
        field = torch.cat(vals, dim=dim).reshape(B, K, -1)
        if self.training and self.noise_std > 0.0:
            field = torch.cat((field[..., :3], field[..., 3:4] + torch.randn_like(field[..., 3:4]) * self.noise_std), -1)
        return _integrate(rays, z_samp, field, self.white_bkgd)

    # ------------------------------------------------------------------------------------
    def forward(self, model, rays, want_weights=False):
        """rays (SB,B,8) -> DotMap(coarse=DotMap(rgb,depth[,weights]), fine=...) (nerf.py:251-303)."""
        self._apply_sched()
        assert rays.dim() == 3
        if self._can_fuse(model, rays):
            return self._forward_fused(model, rays, want_weights)
        if self._fused_grad(model, rays):
            from .fused_train import fused_render_train
            return fused_render_train(self, model, rays, want_weights)
        return self._forward_torch(model, rays, want_weights)

    def _apply_sched(self):
        """Sample counts of the schedule step reached so far (nerf.py:265-267)."""
        if self.sched is not None and self.last_sched.item() > 0:
            self.n_coarse = self.sched[1][self.last_sched.item() - 1]
            self.n_fine = self.sched[2][self.last_sched.item() - 1]

    def _fused_grad(self, model, rays):
        """Whether grad mode runs the fused autograd node (render/fused_train.py; the training step of
        train/train.py:199-215, gradients through every output): a PixelNeRFNet, CUDA rays, no sigma noise and
        PNR_FUSED_BACKWARD unset, auto or 2.  =1 keeps the renderer in torch ops with a fused field node
        (model/fused_field.py); =0 is the composed-torch path the gradient tests compare with."""
        return (os.environ.get("PNR_FUSED_BACKWARD", "auto") in ("auto", "2") and rays.is_cuda
                and self._is_pixelnerf(model) and not (self.training and self.noise_std > 0.0))

    @staticmethod
    def _is_pixelnerf(model):
        from model.models import PixelNeRFNet
        return isinstance(model, PixelNeRFNet)

    def _can_fuse(self, model, rays):
        from model.models import PixelNeRFNet
        if not isinstance(model, PixelNeRFNet):
            return False
        if model._needs_autograd(rays):
            return False
        if self.training and self.noise_std > 0.0:
            raise NotImplementedError("noise_std > 0 in training mode is not supported by the fused path")
        return True

    def _forward_torch(self, model, rays, want_weights):
        sb = rays.shape[0]
        flat = rays.reshape(-1, 8)
        z_c = self.sample_coarse(flat)
        comp_c = self.composite(model, flat, z_c, coarse=True, sb=sb)
        out = DotMap(coarse=self._format_outputs(comp_c, sb, want_weights))
        if self.using_fine:
            zs = [z_c]
            if self.n_fine - self.n_fine_depth > 0:
                zs.append(self.sample_fine(flat, comp_c[0].detach()))
            if self.n_fine_depth > 0:
                zs.append(self.sample_fine_depth(flat, comp_c[2]))
            z_all, _ = torch.sort(torch.cat(zs, dim=-1), dim=-1)
            comp_f = self.composite(model, flat, z_all, coarse=False, sb=sb)
            out.fine = self._format_outputs(comp_f, sb, want_weights)
        return out

    def _lin_steps(self, n, device):
        key = (n, str(device))
        t = self._lin_cache.get(key)
        if t is None:
            t = torch.linspace(0, 1 - 1.0 / n, n, device=device)
            self._lin_cache[key] = t
        return t

    def _forward_fused(self, model, rays, want_weights, noise_in=None, want_z=False):
        """noise_in: optional dict(u_coarse, u_fine, u_fine_jit, n_depth) replacing the torch draws
        (parity tests replay a fixture's noise); want_z also returns the sample depths."""
        dev = rays.device
        if not rays.is_cuda:
            raise RuntimeError("the fused render path needs CUDA rays (no CPU fallback); got %s" % dev)
        SB, B, _ = rays.shape
        counts = fc.sample_counts(self)
        rays_c = rays.detach().contiguous().float()
        draws = fc.draw_noise(SB * B, counts, dev, noise_in)
        noise = fc.bind_noise(self._lin_steps(counts[0], dev), draws)
        scene, mc, mf, keep = model._scene_struct(want_fine=counts[3])
        if scene.SB != SB:
            raise RuntimeError(f"rays have {SB} objects but encode() saw {scene.SB}")
        cfg = fc.render_cfg(self, model.engine)
        out, res = fc.render_outputs(SB, B, counts, dev, want_weights, want_z)
        L = pn.lib()
        ws = pn.workspace(dev, L.pnr_render_workspace_bytes(scene, mc, mf, cfg, B))
        with torch.cuda.device(dev):
            pn.check(L.pnr_render(scene, mc, mf, cfg, pn.dptr(rays_c, "rays"), noise, out, B, ws.data_ptr(),
                                  ws.numel(), pn.stream_ptr(dev)))
        return res

    def _format_outputs(self, rendered, sb, want_weights=False):
        w, rgb, depth = rendered
        if sb > 0:
            rgb, depth, w = rgb.reshape(sb, -1, 3), depth.reshape(sb, -1), w.reshape(sb, -1, w.shape[-1])
        d = DotMap(rgb=rgb, depth=depth)
        if want_weights:
            d.weights = w
        return d

    def sched_step(self, steps=1):
        """Advance the sample-count schedule (nerf.py:318-338)."""
        if self.sched is None:
            return
        self.iter_idx += steps
        while (self.last_sched.item() < len(self.sched[0])
               and self.iter_idx.item() >= self.sched[0][self.last_sched.item()]):
            self.n_coarse = self.sched[1][self.last_sched.item()]
            self.n_fine = self.sched[2][self.last_sched.item()]
            print("INFO: NeRF sampling resolution changed on schedule ==> c", self.n_coarse, "f", self.n_fine)
            self.last_sched += 1

    @classmethod
    def from_conf(cls, conf, white_bkgd=False, lindisp=False, eval_batch_size=100000):
        return cls(conf.get_int("n_coarse", 128), conf.get_int("n_fine", 0),
                   n_fine_depth=conf.get_int("n_fine_depth", 0), noise_std=conf.get_float("noise_std", 0.0),
                   depth_std=conf.get_float("depth_std", 0.01), white_bkgd=conf.get_float("white_bkgd", white_bkgd),
                   lindisp=lindisp, eval_batch_size=conf.get_int("eval_batch_size", eval_batch_size),
                   sched=conf.get_list("sched", None))

    def bind_parallel(self, net, gpus=None, simple_output=False):
        """Returns a module: forward(rays (SB,B,8), want_weights) -> (rgb, depth) or nested dict."""
        wrapped = _RenderWrapper(net, self, simple_output=simple_output)
        if gpus is not None and len(gpus) > 1:
            print("Using multi-GPU", gpus)
            wrapped = _ShardedRender(wrapped, gpus)
        return wrapped
