"""
Mesh reconstruction tools (the reference's src/util/recon.py), on the GPU.

`marching_cubes` evaluates sigma on a grid with the fused field kernels and extracts the isosurface with the
library's own marching cubes (`pnr_grid_points`, `pnr_field_eval`, `pnr_mc_count` / `pnr_mc_emit`, include/pnr.h):
the grid, the sigma volume and the mesh stay on the device, and only the mesh comes back.  With `return_colors`,
`pnr_mc_vertex_attrs` adds normals and the field colours each vertex.  With `block`, sigma is evaluated on a coarse
lattice first and only the blocks the surface crosses are refined and meshed (`pnr_band_*`).  There is no CPU path.
"""
import warnings

import numpy as np
import torch

import pnr_native as pn


def marching_cubes(
    occu_net,
    c1=[-1, -1, -1],
    c2=[1, 1, 1],
    reso=[128, 128, 128],
    isosurface=50.0,
    sigma_idx=3,
    eval_batch_size=100000,
    coarse=True,
    device=None,
    return_colors=False,
    block=None,
):
    """
    Run marching cubes on network.
    WARNING: does not make much sense with viewdirs in current form, since
    sigma depends on viewdirs.
    :param occu_net main NeRF type network, encoded with one object (num_objs == 1), on a CUDA device
    :param c1 corner 1 of marching cube bounds x,y,z
    :param c2 corner 2 of marching cube bounds x,y,z (all > c1)
    :param reso resolutions of marching cubes x,y,z
    :param isosurface sigma-isosurface of marching cubes
    :param sigma_idx index of 'sigma' value in last dimension of occu_net's output
    :param eval_batch_size batch size for evaluation
    :param coarse whether to use coarse NeRF for evaluation
    :param device optionally, device to put points for evaluation.
    By default uses device of occu_net's first parameter.
    :param return_colors also return per-vertex normals and colours (pnr_mc_vertex_attrs, then the field at each
    vertex)
    :return vertices (N, 3) float64 numpy, scaled as vertex index * (c2 - c1) / reso + c1; triangles (M, 3) int64
    numpy of vertex ids, counter-clockwise seen from outside (normals toward decreasing sigma).  With return_colors,
    also normals (N, 3) float64 numpy, unit, toward decreasing sigma (from the sigma grid's gradient), and rgb (N, 3)
    float32 numpy: channels 0-2 of occu_net at the vertex's true position on the surface, seen head-on from outside
    (view direction -normal), in eval_batch_size chunks with occu_net's engine
    :param block None (default): sigma on every grid point and marching cubes over the whole grid.  An int b >= 2
    (at most 256): narrow band.  Sigma is evaluated on the coarse lattice of every b-th grid index per axis (plus the
    last), then only in the blocks of b cells per side whose corners straddle the isosurface, and their 26 neighbours.
    The result is exactly the dense result with every cell outside those blocks treated as empty and the vertices no
    remaining triangle uses dropped; where every cell the surface crosses lies in such a block it is the dense result,
    bit for bit.  A feature smaller than a block that no lattice point sees is missed, and the mesh can be open where
    the surface leaves the band.
    """
    if occu_net.use_viewdirs:
        warnings.warn(
            "Running marching cubes with fake view dirs (pointing to origin), output may be invalid"
        )
    if occu_net.num_objs != 1:
        raise RuntimeError(f"marching_cubes needs a network encoded with one object, got num_objs = {occu_net.num_objs}")
    if device is None:
        device = next(occu_net.parameters()).device
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"marching_cubes runs on CUDA only (no CPU fallback); got device {device}")
    reso = [int(r) for r in reso]
    N = reso[0] * reso[1] * reso[2]
    if block is not None:
        if isinstance(block, bool) or not isinstance(block, (int, np.integer)) or not 2 <= block <= pn.BAND_MAX_BLOCK:
            raise ValueError(f"block must be None or an int in [2, {pn.BAND_MAX_BLOCK}], got {block!r}")
        block = int(block)
    is_train = occu_net.training
    occu_net.eval()
    try:
        with torch.no_grad():
            if block is not None:
                vertices, triangles, *colors = _band(occu_net, c1, c2, reso, isosurface, sigma_idx, eval_batch_size,
                                                     coarse, device, return_colors, block)
                return _scaled(vertices, triangles, c1, c2, reso, *colors)
            print("Evaluating sigma @", N, "points")
            bs = max(1, min(int(eval_batch_size), N))
            sigmas = _sigma(occu_net, N, bs, lambda f, n, p, d: pn.grid_points(c1, c2, reso, f, n, p, d), coarse,
                            sigma_idx, device)

            print("Running marching cubes")
            if not return_colors:
                vertices, triangles = pn.marching_cubes(sigmas.view(*reso), isosurface)
            else:
                # the field is queried where the surface is (xyz), not at the returned vertices, which keep the
                # reference's (c2 - c1) / reso scale below
                vertices, triangles, normals, xyz, vd = pn.marching_cubes(sigmas.view(*reso), isosurface,
                                                                          bounds=(c1, c2))
                print("Evaluating colour @", len(xyz), "vertices")
                rgb = _colours(occu_net, xyz, vd, bs, coarse, device)
                normals, rgb = normals.cpu().numpy(), rgb.cpu().numpy()
            vertices, triangles = vertices.cpu().numpy(), triangles.cpu().numpy()
    finally:
        if is_train:
            occu_net.train()
    if return_colors:
        return _scaled(vertices, triangles, c1, c2, reso, normals, rgb)
    return _scaled(vertices, triangles, c1, c2, reso)


def _scaled(vertices, triangles, c1, c2, reso, *colors):
    # Scale (by reso, not reso - 1, as the reference does)
    c1, c2 = np.array(c1), np.array(c2)
    vertices *= (c2 - c1) / np.array(reso)
    return (vertices + c1, triangles) + colors


def _sigma(occu_net, count, bs, points, coarse, sigma_idx, device):
    """sigma [count] of the points `points(first, n, xyz, viewdirs)` writes, in bs chunks"""
    pts = torch.empty(bs, 3, dtype=torch.float32, device=device)
    vd = torch.empty(bs, 3, dtype=torch.float32, device=device)
    sigmas = torch.empty(count, dtype=torch.float32, device=device)
    for first in range(0, count, bs):
        n = min(bs, count - first)
        points(first, n, pts, vd)
        out = occu_net(pts[None, :n], coarse=coarse, viewdirs=vd[None, :n])
        sigmas[first:first + n] = out[0, :, sigma_idx]
    return sigmas


def _colours(occu_net, xyz, vd, bs, coarse, device):
    rgb = torch.empty(len(xyz), 3, dtype=torch.float32, device=device)
    for first in range(0, len(xyz), bs):
        out = occu_net(xyz[None, first:first + bs], coarse=coarse, viewdirs=vd[None, first:first + bs])
        rgb[first:first + bs] = out[0, :, :3]
    return rgb


def _band(occu_net, c1, c2, reso, isosurface, sigma_idx, eval_batch_size, coarse, device, return_colors, block):
    """The narrow-band path of marching_cubes -> numpy (vertices in grid index units, triangles[, normals, rgb]).
    Nothing on it is sized by the full grid."""
    n_lat = pn.band_lattice_size(reso, block)
    print("Evaluating sigma @", n_lat, "coarse lattice points")
    bs = max(1, min(int(eval_batch_size), n_lat))
    lattice = _sigma(occu_net, n_lat, bs, lambda f, n, p, d: pn.band_lattice_points(c1, c2, reso, block, f, n, p, d),
                     coarse, sigma_idx, device)
    plan = pn.band_plan(lattice, reso, block, isosurface, apron=return_colors)
    del lattice
    M = plan.n_points
    print("Evaluating sigma @", M, "points in", plan.n_active, "active blocks")
    bs = max(1, min(int(eval_batch_size), max(M, 1)))
    sigmas = _sigma(occu_net, M, bs, lambda f, n, p, d: pn.band_points(plan, c1, c2, f, n, p, d), coarse, sigma_idx,
                    device)
    print("Running marching cubes")
    if not return_colors:
        return tuple(t.cpu().numpy() for t in pn.band_marching_cubes(sigmas, plan, isosurface))
    vertices, triangles, normals, xyz, vd = pn.band_marching_cubes(sigmas, plan, isosurface, bounds=(c1, c2))
    print("Evaluating colour @", len(xyz), "vertices")
    bs = max(1, min(int(eval_batch_size), reso[0] * reso[1] * reso[2]))      # the dense path's chunks
    rgb = _colours(occu_net, xyz, vd, bs, coarse, device)
    return tuple(t.cpu().numpy() for t in (vertices, triangles, normals, rgb))


def save_obj(vertices, triangles, path, vert_rgb=None, vert_normals=None):
    """
    Save an OBJ file: one `v x y z` line per vertex (`v x y z r g b` with per-vertex colours), then with normals one
    `vn x y z` line per vertex, then one 1-based `f a b c` line per triangle (`f a//a b//b c//c` with normals); every
    coordinate, colour and normal component with %.4f.
    :param vertices (N, 3)
    :param triangles (M, 3) 0-based vertex ids
    :param vert_rgb (N, 3) rgb, optional
    :param vert_normals (N, 3) normals, optional
    """
    vertices = np.asarray(vertices)
    rows = vertices if vert_rgb is None else np.concatenate([vertices, np.asarray(vert_rgb)], axis=1)
    vfmt = "v" + " %.4f" * rows.shape[1] + "\n"
    with open(path, "w") as f:
        f.writelines(vfmt % tuple(r) for r in rows)
        if vert_normals is None:
            f.writelines("f %d %d %d\n" % (a + 1, b + 1, c + 1) for a, b, c in np.asarray(triangles))
        else:
            f.writelines("vn %.4f %.4f %.4f\n" % tuple(n) for n in np.asarray(vert_normals))
            f.writelines("f %d//%d %d//%d %d//%d\n" % (a + 1, a + 1, b + 1, b + 1, c + 1, c + 1)
                         for a, b, c in np.asarray(triangles))
