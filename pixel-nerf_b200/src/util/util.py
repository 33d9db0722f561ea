"""
Caller-side helpers the eval / train scripts expect under `util.*` (reference:
src/util/util.py).  Only the ray / pose / indexing helpers that sit next to the render hot
path are provided; image-io, colour-map and conv-padding utilities of the reference are
outside the hot path (SURVEY.md section 2, row 6) and are not part of this package.
"""
import functools
import math

import numpy as np
import torch
from torch import nn


def repeat_interleave(input, repeats, dim=0):
    """(N, ...) -> (N*repeats, ...) with each row repeated consecutively (util.py:58-65)."""
    assert dim == 0
    return input.unsqueeze(1).expand(-1, repeats, *input.shape[1:]).reshape(-1, *input.shape[1:])


def combine_interleaved(t, inner_dims=(1,), agg_type="average"):
    """Multi-view pooling used by ResnetFC (util.py:461-471)."""
    if len(inner_dims) == 1 and inner_dims[0] == 1:
        return t
    t = t.reshape(-1, *inner_dims, *t.shape[1:])
    if agg_type == "average":
        return torch.mean(t, dim=1)
    if agg_type == "max":
        return torch.max(t, dim=1)[0]
    raise NotImplementedError("Unsupported combine type " + agg_type)


def batched_index_select_nd(t, inds):
    """t (B, N, ...), inds (B, k) -> (B, k, ...) (util.py:32-43)."""
    idx = inds.view(*inds.shape, *([1] * (t.dim() - 2))).expand(-1, -1, *t.shape[2:])
    return t.gather(1, idx)


def _intrinsics(width, height, f, c):
    """(fx, fy, cx, cy) as python floats: scalar or 2-vector focal, optional centre (util.py:124-133)."""
    if c is None:
        cx, cy = width * 0.5, height * 0.5
    else:
        cc = torch.as_tensor(c, dtype=torch.float32).reshape(-1)
        cx, cy = float(cc[0]), float(cc[1])
    ff = torch.as_tensor(f, dtype=torch.float32).reshape(-1)
    fx, fy = (float(ff[0]), float(ff[0])) if ff.numel() == 1 else (float(ff[0]), float(ff[1]))
    return fx, fy, cx, cy


def unproj_map(width, height, f, c=None, device="cpu"):
    """(H, W, 3) unit camera-space ray directions, -z forward, +y up (util.py:113-143)."""
    fx, fy, cx, cy = _intrinsics(width, height, f, c)
    ys = (torch.arange(height, dtype=torch.float32) - cy).to(device) / fy
    xs = (torch.arange(width, dtype=torch.float32) - cx).to(device) / fx
    Y = ys[:, None].expand(height, width)
    X = xs[None, :].expand(height, width)
    d = torch.stack((X, -Y, -torch.ones_like(X)), dim=-1)
    return d / torch.norm(d, dim=-1).unsqueeze(-1)


def gen_rays(poses, width, height, focal, z_near, z_far, c=None, ndc=False):
    """(NV,4,4) camera-to-world -> (NV,H,W,8) [origin, unit dir, near, far] (util.py:238-276).

    Differentiable w.r.t. `poses` as in the reference: on CUDA, with grad mode on and `poses.requires_grad`, the kernel
    runs inside an autograd node whose backward is `pnr_gen_rays_backward`.  The reference reads focal and c as Python
    floats (util.py:134-139), so neither gets a gradient through the rays, here as there."""
    if ndc:
        raise NotImplementedError("NDC rays are not used by any shipped config")
    nv, dev = poses.shape[0], poses.device
    if dev.type == "cuda":     # poses already on the GPU: the pnr_gen_rays kernel (no CPU detour)
        import pnr_native
        fx, fy, cx, cy = _intrinsics(width, height, torch.as_tensor(focal).detach().squeeze(),
                                     c.detach() if torch.is_tensor(c) else c)
        if torch.is_grad_enabled() and poses.requires_grad:
            rays = pnr_native.gen_rays_autograd(poses, width, height, fx, fy, cx, cy, z_near, z_far)
            return rays.view(nv, height, width, 8)
        return pnr_native.gen_rays(poses, width, height, fx, fy, cx, cy, z_near, z_far).view(nv, height, width, 8)
    cam = unproj_map(width, height, torch.as_tensor(focal).squeeze(), c=c, device=dev)
    dirs = torch.matmul(poses[:, None, None, :3, :3], cam[None].expand(nv, -1, -1, -1).unsqueeze(-1))[..., 0]
    origins = poses[:, None, None, :3, 3].expand(-1, height, width, -1)
    near = torch.full((nv, height, width, 1), float(z_near), device=dev)
    far = torch.full((nv, height, width, 1), float(z_far), device=dev)
    return torch.cat((origins, dirs, near, far), dim=-1)


def pose_spherical(theta, phi, radius):
    """Orbit camera pose (degrees), NeRF convention (util.py:309-324)."""
    th, ph = theta / 180.0 * np.pi, phi / 180.0 * np.pi
    t = torch.eye(4, dtype=torch.float32)
    t[2, 3] = radius
    rp = torch.tensor([[1, 0, 0, 0], [0, np.cos(ph), -np.sin(ph), 0],
                       [0, np.sin(ph), np.cos(ph), 0], [0, 0, 0, 1]], dtype=torch.float32)
    rt = torch.tensor([[np.cos(th), 0, -np.sin(th), 0], [0, 1, 0, 0],
                       [np.sin(th), 0, np.cos(th), 0], [0, 0, 0, 1]], dtype=torch.float32)
    flip = torch.tensor([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1]], dtype=torch.float32)
    return flip @ (rt @ (rp @ t))


def coord_from_blender(dtype=torch.float32, device="cpu"):
    return torch.tensor([[1, 0, 0, 0], [0, 0, 1, 0], [0, -1, 0, 0], [0, 0, 0, 1]], dtype=dtype, device=device)


def coord_to_blender(dtype=torch.float32, device="cpu"):
    return torch.tensor([[1, 0, 0, 0], [0, 0, -1, 0], [0, 1, 0, 0], [0, 0, 0, 1]], dtype=dtype, device=device)


def bbox_sample(bboxes, num_pix):
    """Random pixels inside per-image boxes: (N,4) [x0,y0,x1,y1] -> (num_pix,3) [img, y, x] (util.py:220-235)."""
    image_ids = torch.randint(0, bboxes.shape[0], (num_pix,))
    bb = bboxes[image_ids]
    x = (torch.rand(num_pix) * (bb[:, 2] + 1 - bb[:, 0]) + bb[:, 0]).long()
    y = (torch.rand(num_pix) * (bb[:, 3] + 1 - bb[:, 1]) + bb[:, 1]).long()
    return torch.stack((image_ids, y, x), dim=-1)


def get_cuda(gpu_id):
    """cuda:<id> when available else cpu (util.py:205-210)."""
    return torch.device("cuda:%d" % gpu_id) if torch.cuda.is_available() else torch.device("cpu")


def psnr(pred, target):
    """PSNR in dB of two tensors or arrays, as a python float (util.py:474-481)."""
    mse = ((pred - target) ** 2).mean()
    return -10 * math.log10(mse)


def count_parameters(model):
    return sum(p.numel() for p in model.parameters() if p.requires_grad)


def get_norm_layer(norm_type="instance", group_norm_groups=32):
    if norm_type == "batch":
        return functools.partial(nn.BatchNorm2d, affine=True, track_running_stats=True)
    if norm_type == "instance":
        return functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=False)
    if norm_type == "group":
        return functools.partial(nn.GroupNorm, group_norm_groups)
    if norm_type == "none":
        return None
    raise NotImplementedError("normalization layer [%s] is not found" % norm_type)


def get_module(net):
    """Unwrap (Distributed)DataParallel (util.py:531-538)."""
    return net.module if hasattr(net, "module") and isinstance(net.module, nn.Module) else net
