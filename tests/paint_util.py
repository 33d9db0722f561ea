"""Analytic scenes for the vertex-painting tests: rendered rgb, depth and opacity maps of coloured spheres on the exact
rays of util.gen_rays, the fused, meshed surface they give through the oracles, and the painting oracle
(oracle/pnr_recon_paint.py) itself."""
import os

import numpy as np
import torch

import emu_util  # noqa: F401  (puts pixel-nerf_b200/src on sys.path)
from fuse_util import fuse, index_to_world
from golden_util import ROOT, load_by_path
from recon_util import recon

paint = load_by_path("pnr_recon_paint_oracle", os.path.join(ROOT, "oracle", "pnr_recon_paint.py"))
attrs = load_by_path("pnr_recon_attrs_oracle", os.path.join(ROOT, "oracle", "pnr_recon_attrs.py"))


def gradient_colour(r):
    """The colour field c(p) = 0.5 + 0.5 p / r, in [0, 1] on a sphere of radius r at the origin."""
    return lambda p: 0.5 + 0.5 * p / r


def sphere_scene_maps(poses, width, height, focal, spheres, c=None, background=1.0):
    """rgb (V, H, W, 3), depth and opacity (V, H, W) fp32 maps of opaque spheres, by ray-sphere intersection in
    float64 on util.gen_rays' rays.  spheres: (centre, radius, colour) with colour an rgb triple or a function of the
    hit points.  A ray that hits takes the nearest hit: depth = its distance, opacity 1, rgb = the colour there.  A ray
    that misses has depth 0, opacity 0 and rgb = background (what the renderer composites for an opaque surface)."""
    import util
    rays = util.gen_rays(torch.as_tensor(poses), width, height, torch.tensor(float(focal)), 0.1, 10.0, c=c)
    rays = rays.numpy().astype(np.float64)
    o, d = rays[..., :3], rays[..., 3:6]
    best = np.full(o.shape[:-1], np.inf)
    rgb = np.full(o.shape, float(background))
    for centre, r, colour in spheres:
        oc = o - np.asarray(centre, dtype=np.float64)
        b = (oc * d).sum(-1)
        disc = b * b - ((oc * oc).sum(-1) - r * r)
        t = -b - np.sqrt(np.where(disc >= 0, disc, 0.0))
        hit = (disc >= 0) & (t > 0) & (t < best)
        best = np.where(hit, t, best)
        p = o + t[..., None] * d
        col = colour(p) if callable(colour) else np.broadcast_to(np.asarray(colour, dtype=np.float64), p.shape)
        rgb = np.where(hit[..., None], col, rgb)
    hit = np.isfinite(best)
    return (rgb.astype(np.float32), np.where(hit, best, 0.0).astype(np.float32), hit.astype(np.float32))


def fused_surface(depth, opacity, poses, focal, cx, cy, lo, hi, reso, trunc, min_opacity=0.5):
    """The oracles' fuse_views geometry: fuse the maps, mesh -tsdf at 0 -> (world-space vertices (N, 3) float64,
    triangles, unit outward normals (N, 3) float64)."""
    tsdf = fuse.tsdf_fuse(depth, opacity, poses, focal, focal, cx, cy, lo, hi, reso, trunc, min_opacity)
    v, t = recon.marching_cubes(-tsdf, 0.0)
    normals = attrs.vertex_attrs(-tsdf, 0.0, lo, hi)[0]
    return index_to_world(v, lo, hi, reso), t, normals
