"""
PixelNeRFNet with the reference's surface (src/model/models.py): `encode()` leaves the scene
state in module buffers, `forward(xyz, coarse, viewdirs)` evaluates the conditioned field.

Inference (no autograd) goes to the fused sm_90a kernels through the C ABI
(`pnr_field_eval`, include/pnr.h); there is no CPU fallback on that path.  When gradients are
required on CUDA (train/train.py) the same fused forward runs inside an autograd node whose
backward is `pnr_field_backward` (model/fused_field.py; SURVEY.md section 8f row 1).  The
composed torch ops of `_forward_autograd` remain for CPU tensors in grad mode (host-logic
tests) and as the PNR_FUSED_BACKWARD=0 cross-check of the gradient tests.
"""
import os
import os.path as osp
import warnings

import numpy as np
import torch

import pnr_native as pn
from util import repeat_interleave

from .code import PositionalEncoding
from .model_util import make_encoder, make_mlp


def _param_key(mod):
    return tuple((p.data_ptr(), p._version, str(p.device)) for p in mod.parameters())


class _FusedCache:
    """Device-side derived state: channels-last latent, weight structs, tensor-engine packs.
    Everything is keyed on (data_ptr, _version) so in-place updates and re-encodes invalidate."""

    def __init__(self):
        self.latent_key = None
        self.latent_nhwc = None
        self.mlp = {}      # name -> (key, struct, keepalive tensors, packed)
        self.proj = {}     # name -> (key, tensor)

    def latent(self, latent):
        key = (latent.data_ptr(), latent._version, tuple(latent.shape), str(latent.device))
        if key != self.latent_key:
            self.latent_nhwc = pn.pack_latent(latent.detach().contiguous().float())
            self.latent_key = key
            self.proj = {}
        return self.latent_nhwc


class PixelNeRFNet(torch.nn.Module):
    def __init__(self, conf, stop_encoder_grad=False):
        super().__init__()
        self.encoder = make_encoder(conf["encoder"])
        self.use_encoder = conf.get_bool("use_encoder", True)
        self.use_xyz = conf.get_bool("use_xyz", False)
        self.normalize_z = conf.get_bool("normalize_z", True)
        self.stop_encoder_grad = stop_encoder_grad
        self.use_code = conf.get_bool("use_code", False)
        self.use_code_viewdirs = conf.get_bool("use_code_viewdirs", True)
        self.use_viewdirs = conf.get_bool("use_viewdirs", False)
        self.use_global_encoder = conf.get_bool("use_global_encoder", False)
        # The fused path implements the feature set of every shipped config
        # (conf/default.conf); anything else is refused by name, never silently emulated.
        for flag, ok in (("use_encoder", self.use_encoder), ("use_xyz", self.use_xyz),
                         ("normalize_z", self.normalize_z), ("use_code", self.use_code),
                         ("use_viewdirs", self.use_viewdirs)):
            if not ok:
                raise NotImplementedError(f"model.{flag} = False is not supported")
        if self.use_code_viewdirs:
            raise NotImplementedError("model.use_code_viewdirs = True is not supported")
        if self.use_global_encoder:
            raise NotImplementedError("model.use_global_encoder = True is not supported")

        d_latent = self.encoder.latent_size
        self.code = PositionalEncoding.from_conf(conf["code"], d_in=3)
        # the fused kernels (csrc/pnr_geom.cuh feat_channel, k_geom_bwd) compute THIS code in registers
        if not (self.code.num_freqs == 6 and self.code.include_input and abs(self.code.freq_factor - 1.5) < 1e-12):
            raise NotImplementedError(
                "model.code must be num_freqs = 6, freq_factor = 1.5, include_input = True (every shipped conf); got "
                f"num_freqs = {self.code.num_freqs}, freq_factor = {self.code.freq_factor}, "
                f"include_input = {self.code.include_input}")
        d_in = self.code.d_out + 3  # + un-encoded view directions (models.py:58-60)
        d_out = 4
        self.latent_size = self.encoder.latent_size
        self.mlp_coarse = make_mlp(conf["mlp_coarse"], d_in, d_latent, d_out=d_out)
        self.mlp_fine = make_mlp(conf["mlp_fine"], d_in, d_latent, d_out=d_out, allow_empty=True)
        self.register_buffer("poses", torch.empty(1, 3, 4), persistent=False)
        self.register_buffer("image_shape", torch.empty(2), persistent=False)
        self.register_buffer("focal", torch.empty(1, 2), persistent=False)
        self.register_buffer("c", torch.empty(1, 2), persistent=False)
        self.d_in, self.d_out, self.d_latent = d_in, d_out, d_latent
        self.num_objs = 0
        self.num_views_per_obj = 1
        self._image_wh = (0.0, 0.0)
        self._scene_epoch = 0          # bumped by every encode() / set_scene() / set_cameras(): keys per-GPU replicas
        self._fused = _FusedCache()
        self.engine = os.environ.get("PNR_ENGINE", "auto")  # auto | simt | tc

    # ------------------------------------------------------------------------------
    # encode(): state producer (models.py:89-144)
    # ------------------------------------------------------------------------------
    def encode(self, images, poses, focal, z_bounds=None, c=None):
        """images (SB,NS,3,H,W) or (N,3,H,W) (then every image is its own object);
        poses camera-to-world, same leading dims; focal / c scalar, (n,) or (n,2)."""
        self.num_objs = images.size(0)
        if images.dim() == 5:
            assert poses.dim() == 4 and poses.size(1) == images.size(1)
            self.num_views_per_obj = images.size(1)
            images = images.reshape(-1, *images.shape[2:])
            poses = poses.reshape(-1, 4, 4)
        else:
            self.num_views_per_obj = 1
        self.encoder(images)
        self._fused.latent_key = None     # a new latent may reuse the address (and version 0) of an old one
        self.set_cameras(poses, focal, c, images.shape[-1], images.shape[-2])

    def set_cameras(self, poses, focal, c, width, height):
        """Camera bookkeeping of encode() (models.py:112-141) split out so that a scene can
        also be installed from a precomputed latent (see `set_scene`)."""
        rot = poses[:, :3, :3].transpose(1, 2)
        trans = -torch.bmm(rot, poses[:, :3, 3:])
        self.poses = torch.cat((rot, trans), dim=-1).contiguous()          # world -> camera, (V,3,4)
        self.image_shape[0] = width
        self.image_shape[1] = height
        self._image_wh = (float(width), float(height))
        focal = torch.as_tensor(focal, device=self.poses.device)
        if focal.dim() == 0:
            focal = focal[None, None].repeat((1, 2))
        elif focal.dim() == 1:
            focal = focal.unsqueeze(-1).repeat((1, 2))
        else:
            focal = focal.clone()
        self.focal = focal.float().contiguous()   # _scene_struct hands raw pointers of these buffers to the kernels
        self.focal[..., 1] *= -1.0
        if c is None:
            c = (self.image_shape * 0.5).unsqueeze(0)
        else:
            c = torch.as_tensor(c, device=self.poses.device)
            if c.dim() == 0:
                c = c[None, None].repeat((1, 2))
            elif c.dim() == 1:
                c = c.unsqueeze(-1).repeat((1, 2))
        self.c = c.float().contiguous()
        self._scene_epoch += 1

    def set_scene(self, latent, poses, focal, c, width, height):
        """Install a precomputed latent (V,L,Hl,Wl) with cameras (SB,NS,4,4) -- what encode()
        would leave behind, minus the conv trunk.  Used by tests and benchmarks."""
        assert poses.dim() == 4
        self.num_objs, self.num_views_per_obj = poses.shape[0], poses.shape[1]
        enc = self.encoder
        enc.latent = latent
        self._fused.latent_key = None
        enc.latent_scaling[0] = latent.shape[-1]
        enc.latent_scaling[1] = latent.shape[-2]
        enc.latent_scaling = enc.latent_scaling / (enc.latent_scaling - 1) * 2.0
        self.set_cameras(poses.reshape(-1, 4, 4), focal, c, width, height)

    # ------------------------------------------------------------------------------
    # fused-path plumbing
    # ------------------------------------------------------------------------------
    def _mlp_struct(self, name):
        mlp = getattr(self, name)
        key = _param_key(mlp)
        hit = self._fused.mlp.get(name)
        if hit is not None and hit[0] == key:
            return hit[1]
        sd = {k: v.detach().contiguous().float() for k, v in mlp.state_dict().items()}
        struct = pn.make_mlp_struct(sd, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                    mlp.combine_layer)
        packed = None
        nbytes = pn.lib().pnr_pack_mlp_bytes(struct)
        if nbytes > 0 and self.engine != "simt":
            dev = sd["lin_in.weight"].device
            packed = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                pn.check(pn.lib().pnr_pack_mlp(struct, packed.data_ptr(), nbytes, pn.stream_ptr(dev)))
            struct = pn.make_mlp_struct(sd, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                        mlp.combine_layer, packed=packed)
        self._fused.mlp[name] = (key, struct, sd, packed)
        self._fused.proj.pop(name, None)
        return struct

    def _scene_struct(self, want_fine):
        """PnrScene for the current encode() state (include/pnr.h)."""
        enc = self.encoder
        lat = enc.latent
        if not lat.is_cuda:
            raise RuntimeError("fused render path needs the model on a CUDA device (no CPU fallback); "
                               "got latent on %s" % lat.device)
        nhwc = self._fused.latent(lat)
        Hl, Wl = lat.shape[-2], lat.shape[-1]
        # latent_scaling as encoder.py:161-163 computes it (fp32), without a device sync
        sx = np.float32(Wl) / (np.float32(Wl) - np.float32(1)) * np.float32(2)
        sy = np.float32(Hl) / (np.float32(Hl) - np.float32(1)) * np.float32(2)
        NS = self.num_views_per_obj
        V = self.poses.shape[0]
        assert lat.shape[0] == V, "encode() latent/pose count mismatch"
        SB = V // NS
        mc = self._mlp_struct("mlp_coarse")
        mf = self._mlp_struct("mlp_fine") if (want_fine and self.mlp_fine is not None) else None
        proj = {}
        for name, m in (("mlp_coarse", mc), ("mlp_fine", mf)):
            proj[name] = self._projection(name, m, nhwc, SB, NS) if (m is not None and m.packed) else None
        scene = pn.make_scene_struct(nhwc, self.poses.contiguous(), self.focal.contiguous(), self.c.contiguous(),
                                     SB, NS, self._image_wh[0], self._image_wh[1], sx, sy,
                                     proj_coarse=proj["mlp_coarse"], proj_fine=proj["mlp_fine"])
        keep = (nhwc, proj)
        return scene, mc, mf, keep

    def _projection(self, name, mstruct, nhwc, SB, NS):
        key = (self._fused.latent_key, self._fused.mlp[name][0])
        hit = self._fused.proj.get(name)
        if hit is not None and hit[0] == key:
            return hit[1]
        dev = nhwc.device
        tmp = pn.make_scene_struct(nhwc, self.poses.contiguous(), self.focal.contiguous(), self.c.contiguous(),
                                   SB, NS, self._image_wh[0], self._image_wh[1], 2.0, 2.0)
        nbytes = pn.lib().pnr_project_latent_bytes(tmp, mstruct)
        if nbytes == 0:
            return None
        out = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
        ws_bytes = pn.lib().pnr_field_workspace_bytes(tmp, mstruct, 1, pn.ENGINE_SIMT) + (64 << 20)
        ws = pn.workspace(dev, ws_bytes)
        with torch.cuda.device(dev):
            pn.check(pn.lib().pnr_project_latent(tmp, mstruct, out.data_ptr(), nbytes, ws.data_ptr(), ws.numel(),
                                                 pn.stream_ptr(dev)))
        self._fused.proj[name] = (key, out)
        return out

    def _needs_autograd(self, *tensors):
        if not torch.is_grad_enabled():
            return False
        if any(t is not None and t.requires_grad for t in tensors):
            return True
        if self.encoder.latent.requires_grad:
            return True
        return any(p.requires_grad for p in self.mlp_coarse.parameters())

    # ------------------------------------------------------------------------------
    # forward(): the conditioned field (models.py:146-266)
    # ------------------------------------------------------------------------------
    def forward(self, xyz, coarse=True, viewdirs=None, far=False):
        """xyz (SB,B,3) world points, viewdirs (SB,B,3) -> (SB,B,4) [sigmoid rgb, relu sigma]."""
        assert viewdirs is not None, "use_viewdirs models need viewdirs"
        if self._needs_autograd(xyz, viewdirs):
            if os.environ.get("PNR_FUSED_BACKWARD", "auto") != "0" and xyz.is_cuda:
                # fused forward + pnr_field_backward in one autograd node (model/fused_field.py)
                from .fused_field import fused_field
                return fused_field(self, xyz, coarse, viewdirs)
            return self._forward_autograd(xyz, coarse, viewdirs)
        return self._field_fused(xyz, coarse, viewdirs)

    def _field_fused(self, xyz, coarse, viewdirs):
        """pnr_field_eval on detached inputs (no autograd graph)."""
        SB, B, _ = xyz.shape
        use_fine = (not coarse) and self.mlp_fine is not None
        scene, mc, mf, keep = self._scene_struct(want_fine=use_fine)
        if SB != scene.SB:
            raise RuntimeError(f"xyz has {SB} objects but encode() saw {scene.SB}")
        dev = xyz.device
        xyz_c = xyz.detach().contiguous().float()
        dirs_c = viewdirs.detach().reshape(SB, B, 3).contiguous().float()
        out = torch.empty(SB, B, 4, dtype=torch.float32, device=dev)
        m = mf if use_fine else mc
        if use_fine:
            scene.proj_coarse = scene.proj_fine  # pnr_field_eval reads proj_coarse for its mlp
        eng = pn.ENGINES[self.engine]
        L = pn.lib()
        nbytes = L.pnr_field_workspace_bytes(scene, m, B, eng)
        ws = pn.workspace(dev, nbytes)
        with torch.cuda.device(dev):
            pn.check(L.pnr_field_eval(scene, m, pn.dptr(xyz_c, "xyz"), pn.dptr(dirs_c, "viewdirs"), pn.dptr(out),
                                      B, eng, ws.data_ptr(), ws.numel(), pn.stream_ptr(dev)))
        return out

    def _forward_autograd(self, xyz, coarse, viewdirs):
        """Differentiable composed-torch evaluation (training only)."""
        SB, B, _ = xyz.shape
        NS = self.num_views_per_obj
        R = self.poses[:, None, :3, :3]
        x = repeat_interleave(xyz, NS)
        x_rot = torch.matmul(R, x.unsqueeze(-1))[..., 0]
        x_cam = x_rot + self.poses[:, None, :3, 3]
        feat = self.code(x_rot.reshape(-1, 3))
        d = repeat_interleave(viewdirs.reshape(SB, B, 3, 1), NS)
        feat = torch.cat((feat, torch.matmul(R, d).reshape(-1, 3)), dim=1)
        uv = -x_cam[:, :, :2] / x_cam[:, :, 2:]
        uv = uv * repeat_interleave(self.focal.unsqueeze(1), NS if self.focal.shape[0] > 1 else 1)
        uv = uv + repeat_interleave(self.c.unsqueeze(1), NS if self.c.shape[0] > 1 else 1)
        latent = self.encoder.index(uv, None, self.image_shape)
        if self.stop_encoder_grad:
            latent = latent.detach()
        latent = latent.transpose(1, 2).reshape(-1, self.latent_size)
        mlp = self.mlp_coarse if (coarse or self.mlp_fine is None) else self.mlp_fine
        o = mlp(torch.cat((latent, feat), dim=-1), combine_inner_dims=(NS, B)).reshape(-1, B, self.d_out)
        return torch.cat((torch.sigmoid(o[..., :3]), torch.relu(o[..., 3:4])), dim=-1).reshape(SB, B, -1)

    # ------------------------------------------------------------------------------
    # checkpoints (models.py:268-316): same file names and state_dict keys
    # ------------------------------------------------------------------------------
    def load_weights(self, args, opt_init=False, strict=True, device=None):
        if opt_init and not args.resume:
            return
        ckpt = "pixel_nerf_init" if opt_init or not args.resume else "pixel_nerf_latest"
        path = "%s/%s/%s" % (args.checkpoints_path, args.name, ckpt)
        if device is None:
            device = self.poses.device
        if os.path.exists(path):
            print("Load", path)
            self.load_state_dict(torch.load(path, map_location=device), strict=strict)
        elif not opt_init:
            warnings.warn(f"WARNING: {path} does not exist, not loaded!! Model will be re-initialized. "
                          "If you meant to load a pretrained model, it is not in the right place; "
                          "when training, pass --resume unless this is a new experiment.")
        return self

    def save_weights(self, args, opt_init=False):
        from shutil import copyfile
        name = "pixel_nerf_init" if opt_init else "pixel_nerf_latest"
        backup = "pixel_nerf_init_backup" if opt_init else "pixel_nerf_backup"
        path = osp.join(args.checkpoints_path, args.name, name)
        if osp.exists(path):
            copyfile(path, osp.join(args.checkpoints_path, args.name, backup))
        torch.save(self.state_dict(), path)
        return self
