"""Analytic scenes for the TSDF fusion tests: depth and opacity maps of a sphere on the exact rays of util.gen_rays, and
the oracle (oracle/pnr_recon_fuse.py) they are fused with."""
import os

import numpy as np
import torch

import emu_util  # noqa: F401  (puts pixel-nerf_b200/src on sys.path)
from golden_util import ROOT, load_by_path

fuse = load_by_path("pnr_recon_fuse_oracle", os.path.join(ROOT, "oracle", "pnr_recon_fuse.py"))


def views(n_turn, radius, phi=-30.0):
    """(n_turn + 2, 4, 4) fp32 camera-to-world poses: a util.pose_spherical turntable at elevation -phi, then one view
    from straight above and one from straight below."""
    import util
    poses = [util.pose_spherical(float(a), phi, radius) for a in np.linspace(-180, 180, n_turn + 1)[:-1]]
    poses += [util.pose_spherical(0.0, -90.0, radius), util.pose_spherical(0.0, 90.0, radius)]
    return torch.stack(poses)


def sphere_maps(poses, width, height, focal, r, c=None):
    """Depth and opacity maps (V, H, W) fp32 of a sphere of radius r at the origin, by ray-sphere intersection in
    float64 on util.gen_rays' rays: depth = the distance to the first hit and opacity 1 where a ray hits it, 0 and 0
    where it does not (what the renderer's sum(w z) and sum(w) are for an opaque surface)."""
    import util
    rays = util.gen_rays(poses, width, height, torch.tensor(float(focal)), 0.1, 10.0, c=c).numpy().astype(np.float64)
    o, d = rays[..., :3], rays[..., 3:6]
    b = (o * d).sum(-1)
    disc = b * b - ((o * o).sum(-1) - r * r)
    hit = disc >= 0
    t = -b - np.sqrt(np.where(hit, disc, 0.0))
    hit &= t > 0
    return np.where(hit, t, 0.0).astype(np.float32), hit.astype(np.float32)


def index_to_world(verts, lo, hi, reso):
    """fuse_views' vertex positions: lo + v (hi - lo) / (n - 1)."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    return verts * ((hi - lo) / (np.asarray(reso) - 1)) + lo
