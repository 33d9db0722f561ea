"""
Mesh reconstruction tools (the reference's src/util/recon.py), on the GPU.

`marching_cubes` evaluates sigma on a grid with the fused field kernels and extracts the isosurface with the
library's own marching cubes (`pnr_grid_points`, `pnr_field_eval`, `pnr_mc_count` / `pnr_mc_emit`, include/pnr.h):
the grid, the sigma volume and the mesh stay on the device, and only the mesh comes back.  With `return_colors`,
`pnr_mc_vertex_attrs` adds normals and the field colours each vertex.  With `block`, sigma is evaluated on a coarse
lattice first and only the blocks the surface crosses are refined and meshed (`pnr_band_*`).  With `gpus`, every field
pass is sharded over several GPUs (`pnr_mgpu_field_eval`) and the rest stays on the first.  There is no CPU path.

`fuse_views` meshes what the renderer shows instead: it renders depth and opacity maps from camera poses, fuses them
into a TSDF (`pnr_tsdf_fuse`) and meshes that with the same marching cubes.  With `colors="views"` it also paints each
vertex with the rendered pixels of the views that see it (`pnr_paint_vertices`).

`keep_components` drops the floaters either leaves: it labels the mesh's connected components on the GPU
(`pnr_mesh_components`) and keeps the largest (`pnr_mesh_compact_count` / `pnr_mesh_compact_emit`).
`decimate` then reduces the mesh with rounds of independent quadric edge collapses on the GPU (`pnr_decimate_*`).
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
    gpus=None,
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
    :param gpus None (default) or one device: everything on `device`.  A list of CUDA device indices [g0, g1, ...]
    with g0 the extraction device (`device`, or occu_net's): every field evaluation -- the sigma grid, the band's
    lattice and refinement points, the vertex colours -- is cut into the same eval_batch_size chunks as on one GPU and
    the chunks are shared out among the devices in contiguous runs; gpus[i] evaluates its run from a copy of the
    scene and weights and sends the values to g0.  A device may repeat ([0, 0]: two shards on one card).  Marching
    cubes, the band plan and the vertex attributes stay on g0.  The result is bit-equal to the call without gpus.
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
    if gpus is not None:
        gpus = [int(g) for g in gpus]
        if not gpus or gpus[0] != (device.index if device.index is not None else torch.cuda.current_device()):
            raise ValueError(f"gpus[0] must be the extraction device {device}, got gpus = {gpus}")
    is_train = occu_net.training
    occu_net.eval()
    field = None
    try:
        with torch.no_grad():
            if gpus is not None and len(gpus) > 1:
                field = _ShardedField(occu_net, gpus, coarse)
            if block is not None:
                vertices, triangles, *colors = _band(occu_net, c1, c2, reso, isosurface, sigma_idx, eval_batch_size,
                                                     coarse, device, return_colors, block, field)
                return _scaled(vertices, triangles, c1, c2, reso, *colors)
            print("Evaluating sigma @", N, "points")
            bs = max(1, min(int(eval_batch_size), N))
            sigmas = _sigma(occu_net, N, bs, lambda f, n, p, d: pn.grid_points(c1, c2, reso, f, n, p, d), coarse,
                            sigma_idx, device, field, pn.point_source(pn.POINTS_GRID, c1, c2, reso))

            print("Running marching cubes")
            if not return_colors:
                vertices, triangles = pn.marching_cubes(sigmas.view(*reso), isosurface)
            else:
                # the field is queried where the surface is (xyz), not at the returned vertices, which keep the
                # reference's (c2 - c1) / reso scale below
                vertices, triangles, normals, xyz, vd = pn.marching_cubes(sigmas.view(*reso), isosurface,
                                                                          bounds=(c1, c2))
                print("Evaluating colour @", len(xyz), "vertices")
                rgb = _colours(occu_net, xyz, vd, bs, coarse, device, field)
                normals, rgb = normals.cpu().numpy(), rgb.cpu().numpy()
            vertices, triangles = vertices.cpu().numpy(), triangles.cpu().numpy()
    finally:
        if field is not None:
            field.close()
        if is_train:
            occu_net.train()
    if return_colors:
        return _scaled(vertices, triangles, c1, c2, reso, normals, rgb)
    return _scaled(vertices, triangles, c1, c2, reso)


def fuse_views(
    net,
    renderer,
    poses,
    width,
    height,
    focal,
    z_near,
    z_far,
    c=None,
    c1=[-1, -1, -1],
    c2=[1, 1, 1],
    reso=[128, 128, 128],
    trunc=None,
    min_opacity=0.5,
    ray_batch_size=50000,
    gpus=None,
    return_colors=False,
    colors="field",
):
    """
    Mesh the surface the renderer shows: render depth and opacity maps of every view, fuse them into a truncated
    signed distance field (TSDF) on the grid of marching_cubes, and run marching cubes on it.  Unlike the sigma grid
    of marching_cubes, every depth sample comes from a real camera with real view directions, so the mesh follows the
    renders of a model whose sigma depends on the view direction.
    :param net main NeRF type network, encoded with one object (num_objs == 1), on a CUDA device
    :param renderer NeRFRenderer; every pixel of every view is rendered through renderer.bind_parallel(net, gpus)
    with want_weights=True, in ray_batch_size batches in the pixel order of render.render_frames, and the fine pass's
    depth and weights.sum(-1) (the coarse pass's when renderer.using_fine is off) are kept per pixel
    :param poses (V, 4, 4) camera-to-world poses, V >= 1 (util.pose_spherical makes a turntable)
    :param width, height, focal, z_near, z_far, c: the cameras, as util.gen_rays takes them
    :param c1, c2, reso: the TSDF grid, as marching_cubes takes them (pnr_grid_points' points), each reso >= 2
    :param trunc truncation distance (world units); default 3 voxel diagonals of the coarsest axis
    :param min_opacity a pixel of lower opacity saw background, which carves the voxels it sees
    :param gpus None or a list of CUDA device indices with gpus[0] net's device: the rendering is sharded over them
    (bind_parallel); fusion, marching cubes, painting and colours run on gpus[0]
    :param return_colors also return per-vertex normals and colours
    :param colors where the colours come from (needs return_colors for anything but the default):
    "field" (default): channels 0-2 of net at the vertex, seen head-on from outside (view direction -normal), from the
    network of the kept pass, as marching_cubes colours its vertices.
    "views": the rendered pixels of the views that see the vertex (pnr_paint_vertices, include/pnr.h), from the kept
    pass's rgb of the same renders, so no extra rendering.  Per view, the vertex's pixel must be a surface pixel
    (opacity >= min_opacity) whose depth lies within trunc of the vertex (not occluded), and the view must face the
    surface; the pixel's colour, with the renderer's background un-mixed ((rgb - bkgd (1 - opacity)) / opacity, bkgd = 1
    for renderer.white_bkgd, else 0), counts with weight cos(normal, direction to the camera).  A vertex no view paints
    falls back to its "field" colour.  The colours are what the renders show, including any view dependence.
    :return vertices (N, 3) float64 numpy in world coordinates at their true positions, lo + v (hi - lo) / (n - 1)
    for index coordinate v (unlike marching_cubes, which keeps the reference's (c2 - c1) / reso scale); triangles
    (M, 3) int64 numpy, counter-clockwise seen from outside.  With return_colors, also normals (N, 3) float64 numpy,
    unit, outward (pnr_mc_vertex_attrs on the fused volume), and rgb (N, 3) float32 numpy in [0, 1], from `colors`.
    The fusion rule is pnr_tsdf_fuse's (include/pnr.h): the renderer's depth is sum(w z), so the surface distance of a
    pixel is depth / opacity.

    Example, a turntable at 30 degrees elevation around an object at the origin::

        poses = torch.stack([util.pose_spherical(a, -30.0, 1.3) for a in np.linspace(-180, 180, 65)[:-1]]).cuda()
        verts, tris = util.recon.fuse_views(net, renderer, poses, 128, 128, focal, 0.8, 1.8, reso=[256] * 3)

    and coloured from those renders::

        verts, tris, normals, rgb = util.recon.fuse_views(net, renderer, poses, 128, 128, focal, 0.8, 1.8,
                                                          reso=[256] * 3, return_colors=True, colors="views")
    """
    from util.util import _intrinsics
    device = next(net.parameters()).device
    if device.type != "cuda":
        raise RuntimeError(f"fuse_views runs on CUDA only (no CPU fallback); got device {device}")
    if net.num_objs != 1:
        raise RuntimeError(f"fuse_views needs a network encoded with one object, got num_objs = {net.num_objs}")
    if gpus is not None:
        gpus = [int(g) for g in gpus]
        if not gpus or gpus[0] != (device.index if device.index is not None else torch.cuda.current_device()):
            raise ValueError(f"gpus[0] must be the network's device {device}, got gpus = {gpus}")
    poses = torch.as_tensor(poses)
    if poses.dim() != 3 or tuple(poses.shape[1:]) != (4, 4) or poses.shape[0] < 1:
        raise ValueError(f"poses must be (V, 4, 4) with V >= 1, got {tuple(poses.shape)}")
    reso = [int(r) for r in reso]
    if len(reso) != 3 or min(reso) < 2:
        raise ValueError(f"reso must be 3 sizes >= 2, got {reso}")
    lo, hi = np.array(c1, dtype=np.float64), np.array(c2, dtype=np.float64)
    h = (hi - lo) / (np.array(reso) - 1)
    if trunc is None:
        trunc = 3.0 * np.sqrt(3.0) * float(np.abs(h).max())
    if not 0 < trunc < np.inf:
        raise ValueError(f"trunc must be positive and finite, got {trunc}")
    if not 0 < min_opacity <= 1:
        raise ValueError(f"min_opacity must be in (0, 1], got {min_opacity}")
    if colors not in ("field", "views"):
        raise ValueError(f'colors must be "field" or "views", got {colors!r}')
    if colors == "views" and not return_colors:
        raise ValueError('colors="views" needs return_colors=True')
    paint = colors == "views"
    V, W, H = poses.shape[0], int(width), int(height)
    fx, fy, cx, cy = _intrinsics(W, H, torch.as_tensor(focal).squeeze(), c)
    bs = max(1, int(ray_batch_size))
    is_train, renderer_train = net.training, renderer.training
    net.eval()
    renderer.eval()
    try:
        with torch.no_grad():
            poses32 = poses.to(device=device, dtype=torch.float32).contiguous()
            render_par = renderer.bind_parallel(net, gpus)
            total = V * H * W
            print("Rendering", V, "views @", total, "rays")
            depth = torch.empty(V, H, W, dtype=torch.float32, device=device)
            opacity = torch.empty(V, H, W, dtype=torch.float32, device=device)
            rgb_map = torch.empty(V, H, W, 3, dtype=torch.float32, device=device) if paint else None
            rays = torch.empty(min(bs, total), 8, dtype=torch.float32, device=device)
            for first in range(0, total, bs):
                count = min(bs, total - first)
                batch = rays[:count]
                pn.gen_rays(poses32, W, H, fx, fy, cx, cy, z_near, z_far, first, count, out=batch)
                out = render_par(batch[None], want_weights=True)
                kept = out["fine"] if renderer.using_fine else out["coarse"]
                depth.view(-1)[first:first + count] = kept["depth"][0]
                opacity.view(-1)[first:first + count] = kept["weights"][0].sum(-1)
                if paint:
                    rgb_map.view(-1, 3)[first:first + count] = kept["rgb"][0]
            del render_par, rays
            print("Fusing", V, "views into", reso)
            tsdf = pn.tsdf_fuse(depth, opacity, poses32, fx, fy, cx, cy, lo, hi, reso, trunc, min_opacity)
            print("Running marching cubes")
            vol = -tsdf                                          # inside is positive, as marching cubes takes it
            if not return_colors:
                vertices, triangles = pn.marching_cubes(vol, 0.0)
            else:
                vertices, triangles, normals, xyz, vd = pn.marching_cubes(vol, 0.0, bounds=(lo, hi))
            vertices, triangles = vertices.cpu().numpy() * h + lo, triangles.cpu().numpy()
            if return_colors:
                coarse = not renderer.using_fine
                if not paint:
                    print("Evaluating colour @", len(xyz), "vertices")
                    rgb = _colours(net, xyz, vd, bs, coarse, device)
                else:
                    # the returned world-space vertices; the rows no view paints take the field colour
                    rgb, weight = pn.paint_vertices(torch.from_numpy(vertices).to(device), normals, rgb_map, depth,
                                                    opacity, poses32, fx, fy, cx, cy, trunc, min_opacity,
                                                    1.0 if renderer.white_bkgd else 0.0)
                    rest = torch.nonzero(weight == 0).view(-1)
                    print("Painted", len(xyz) - len(rest), "vertices from the views;", len(rest),
                          "seen by none take the field's colour")
                    if len(rest):
                        rgb[rest] = _colours(net, xyz[rest], vd[rest], bs, coarse, device)
                normals, rgb = normals.cpu().numpy(), rgb.cpu().numpy()
    finally:
        net.train(is_train)
        renderer.train(renderer_train)
    if return_colors:
        return vertices, triangles, normals, rgb
    return vertices, triangles


def keep_components(vertices, triangles, *vertex_attrs, largest=1, min_triangles=1, device=None):
    """
    Keep the largest connected pieces of a mesh and drop the rest (the floaters of a NeRF field or a fusion), on the
    GPU.  Composes with both extractors, whatever they return::

        verts, tris, normals, rgb = util.recon.keep_components(
            *util.recon.fuse_views(net, renderer, poses, ..., return_colors=True, colors="views"), largest=1)

    :param vertices (N, 3) array-like
    :param triangles (M, 3) array-like of integer vertex ids
    :param vertex_attrs array-likes with a first dimension of N and any trailing shape and dtype (normals, rgb, ...)
    :param largest keep at most this many components (>= 1); None keeps every component with min_triangles
    :param min_triangles keep only components with at least this many triangles (>= 1)
    :param device the CUDA device to run on (default: the current one); there is no CPU path
    :return (vertices, triangles, *vertex_attrs) numpy arrays with the input dtypes.
    Two vertices are connected when some triangle uses both; a component is a maximal connected set of vertices with
    its triangles (two pieces that touch at one vertex are one component).  A vertex no triangle uses is a component
    with 0 triangles and is never kept.  Components are ranked by triangle count, descending, ties going to the
    component whose smallest vertex id is smaller; the first `largest` of that ranking with at least `min_triangles`
    triangles are kept.  The kept vertices and triangles keep their relative order, the triangles are renumbered to
    the kept vertices and every attribute is compacted by the same rows; values are copied bit for bit.  So when
    everything is kept, a mesh without unused vertices (every mesh marching_cubes and fuse_views return) comes back
    bit-equal.  The labelling is pnr_mesh_components and the compaction pnr_mesh_compact_* (include/pnr.h).
    Raises ValueError for largest or min_triangles below 1, wrong shapes, an attribute whose first dimension is not N
    and a triangle id outside [0, N).
    """
    for name, v in (("largest", largest), ("min_triangles", min_triangles)):
        if v is None and name == "largest":
            continue
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
            raise ValueError(f"{name} must be an int >= 1{' or None' if name == 'largest' else ''}, got {v!r}")
    vertices, triangles = np.asarray(vertices), np.asarray(triangles)
    if vertices.ndim != 2 or vertices.shape[1] != 3:
        raise ValueError(f"vertices must be (N, 3), got {vertices.shape}")
    if triangles.ndim != 2 or triangles.shape[1] != 3 or not np.issubdtype(triangles.dtype, np.integer):
        raise ValueError(f"triangles must be (M, 3) integer vertex ids, got {triangles.dtype} {triangles.shape}")
    N, M = len(vertices), len(triangles)
    attrs = [np.asarray(a) for a in vertex_attrs]
    for i, a in enumerate(attrs):
        if a.ndim < 1 or a.shape[0] != N:
            raise ValueError(f"vertex_attrs[{i}] must have a first dimension of {N}, got shape {a.shape}")
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"keep_components runs on CUDA only (no CPU fallback); got device {device}")
    with torch.cuda.device(device):
        tris = torch.from_numpy(np.ascontiguousarray(triangles, dtype=np.int64)).to(device)
        label, tri_count, n_comp = pn.mesh_components(tris, N)
        roots = torch.nonzero(tri_count).view(-1)                       # ascending: ties go to the smaller root
        counts = tri_count[roots]
        order = torch.sort(counts, descending=True, stable=True).indices
        ranked, ranked_counts = roots[order], counts[order]
        kept = ranked[ranked_counts >= int(min_triangles)]
        if largest is not None:
            kept = kept[:int(largest)]
        keep_root = torch.zeros(N, dtype=torch.uint8, device=device)
        keep_root[kept] = 1
        vert_ids, tris_out = pn.mesh_compact(tris, N, label, keep_root)
        del label, tri_count, keep_root, tris
        out = [_gather(a, vert_ids) for a in [vertices] + attrs]
        tris_out = tris_out.cpu().numpy().astype(triangles.dtype, copy=False)
    sep = lambda n: f"{n:,}".replace(",", " ")        # noqa: E731
    print(f"Kept {len(kept)} of {n_comp} components: {sep(len(tris_out))} of {sep(M)} triangles")
    return (out[0], tris_out, *out[1:])


def decimate(vertices, triangles, *vertex_attrs, target_triangles=None, max_error=None, device=None):
    """
    Reduce a mesh on the GPU with quadric edge collapses, keeping a subset of its vertices.  Composes with the
    extractors and keep_components, whatever they return::

        verts, tris, normals, rgb = util.recon.decimate(
            *util.recon.keep_components(*util.recon.fuse_views(..., return_colors=True, colors="views"), largest=1),
            target_triangles=200_000)

    :param vertices (N, 3) array-like
    :param triangles (M, 3) array-like of integer vertex ids
    :param vertex_attrs array-likes with a first dimension of N and any trailing shape and dtype (normals, rgb, ...)
    :param target_triangles stop once the mesh has at most this many triangles (>= 0)
    :param max_error make no collapse whose error exceeds this world length (finite, >= 0); at least one of the two
        bounds is needed, and with both the call stops at whichever binds first
    :param device the CUDA device to run on (default: the current one); there is no CPU path
    :return (vertices, triangles, *vertex_attrs) numpy arrays with the input dtypes.
    Each collapse removes one vertex c and rewrites its triangles to a neighbour d, which does not move; its error is
    the area-weighted RMS distance of d from the planes of the triangles merged into it (Garland-Heckbert quadrics).
    Only interior manifold vertices are removed, so boundaries and non-manifold parts come through unchanged, and no
    collapse flips a triangle.  A vertex with more than 64 incident triangles (a cone tip, a pole) is always kept.  Each round applies a set of collapses far enough apart not to interact, chosen by
    smallest error (pnr_decimate_select); a round that would overshoot the target keeps its cheapest collapses, so
    the result has target - 1 or target triangles unless no valid collapse is left.  The output vertices are input
    rows in their input order, with every attribute copied bit for bit; the triangles keep their relative order,
    renumbered to the vertices they use, and unused vertices are dropped.  The rule is in include/pnr.h.
    Raises ValueError without a bound, for a negative target_triangles, a negative or non-finite max_error, wrong
    shapes, an attribute whose first dimension is not N and a triangle id outside [0, N).
    """
    if target_triangles is None and max_error is None:
        raise ValueError("decimate needs target_triangles or max_error")
    if target_triangles is not None and (isinstance(target_triangles, bool) or
                                         not isinstance(target_triangles, (int, np.integer)) or target_triangles < 0):
        raise ValueError(f"target_triangles must be an int >= 0, got {target_triangles!r}")
    if max_error is not None:
        if isinstance(max_error, bool) or not isinstance(max_error, (int, float, np.integer, np.floating)) or \
                not np.isfinite(max_error) or max_error < 0:
            raise ValueError(f"max_error must be a finite number >= 0, got {max_error!r}")
    vertices, triangles = np.asarray(vertices), np.asarray(triangles)
    if vertices.ndim != 2 or vertices.shape[1] != 3 or not (np.issubdtype(vertices.dtype, np.floating) or
                                                             np.issubdtype(vertices.dtype, np.integer)):
        raise ValueError(f"vertices must be (N, 3) real numbers, got {vertices.dtype} {vertices.shape}")
    if triangles.ndim != 2 or triangles.shape[1] != 3 or not np.issubdtype(triangles.dtype, np.integer):
        raise ValueError(f"triangles must be (M, 3) integer vertex ids, got {triangles.dtype} {triangles.shape}")
    N, M = len(vertices), len(triangles)
    attrs = [np.asarray(a) for a in vertex_attrs]
    for i, a in enumerate(attrs):
        if a.ndim < 1 or a.shape[0] != N:
            raise ValueError(f"vertex_attrs[{i}] must have a first dimension of {N}, got shape {a.shape}")
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise RuntimeError(f"decimate runs on CUDA only (no CPU fallback); got device {device}")
    with torch.cuda.device(device):
        xyz = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float64)).to(device)
        tris = torch.from_numpy(np.ascontiguousarray(triangles, dtype=np.int64)).to(device)
        dec = pn.Decimator(xyz, tris)
        rounds, m = 0, M
        while True:
            if target_triangles is not None and m <= target_triangles:
                reason = "target reached"
                break
            c, d, err, held_back = dec.select(max_error)
            if len(c) == 0:
                reason = "error bound" if held_back else "no valid collapse left"
                break
            if target_triangles is not None and len(c) > -(-(m - target_triangles) // 2):
                keep = -(-(m - target_triangles) // 2)
                # the smallest keys (err, min id, max id); the selected edges share no vertex, so min id decides ties
                order = torch.sort(torch.minimum(c, d), stable=True).indices
                order = order[torch.sort(err[order], stable=True).indices[:keep]]
                order = torch.sort(order).values
                c, d = c[order], d[order]
            m = dec.apply(c, d)
            rounds += 1
        tris = dec.tris
        used = torch.zeros(N, dtype=torch.uint8, device=device)
        used[tris.reshape(-1)] = 1
        del dec, xyz
        vert_ids, tris_out = pn.mesh_compact(tris, N, torch.arange(N, device=device), used)
        out = [_gather(a, vert_ids) for a in [vertices] + attrs]
        tris_out = tris_out.cpu().numpy().astype(triangles.dtype, copy=False)
    sep = lambda n: f"{n:,}".replace(",", " ")        # noqa: E731
    print(f"Decimated in {rounds} rounds: {sep(M)} to {sep(len(tris_out))} triangles ({reason})")
    return (out[0], tris_out, *out[1:])


def _gather(a, rows):
    """a[rows] for a numpy array a and int64 rows on a CUDA device, gathered there bit for bit, dtype kept."""
    if len(rows) == 0:
        return a[:0].copy()
    if not a.flags.writeable:
        a = a.copy()
    t = torch.from_numpy(np.ascontiguousarray(a)).to(rows.device)
    return t.index_select(0, rows).cpu().numpy()


def _scaled(vertices, triangles, c1, c2, reso, *colors):
    # Scale (by reso, not reso - 1, as the reference does)
    c1, c2 = np.array(c1), np.array(c2)
    vertices *= (c2 - c1) / np.array(reso)
    return (vertices + c1, triangles) + colors


def _sigma(occu_net, count, bs, points, coarse, sigma_idx, device, field=None, src=None):
    """sigma [count] of the points `points(first, n, xyz, viewdirs)` writes, in bs chunks (with `field`, a
    _ShardedField: the same points, as the PnrPointSource `src` describes them, over its GPUs)"""
    if field is not None:
        return field.eval(src, count, bs, sigma_idx, 1).view(-1)
    pts = torch.empty(bs, 3, dtype=torch.float32, device=device)
    vd = torch.empty(bs, 3, dtype=torch.float32, device=device)
    sigmas = torch.empty(count, dtype=torch.float32, device=device)
    for first in range(0, count, bs):
        n = min(bs, count - first)
        points(first, n, pts, vd)
        out = occu_net(pts[None, :n], coarse=coarse, viewdirs=vd[None, :n])
        sigmas[first:first + n] = out[0, :, sigma_idx]
    return sigmas


def _colours(occu_net, xyz, vd, bs, coarse, device, field=None):
    if field is not None:
        return field.eval(pn.point_source(pn.POINTS_LIST, xyz0=xyz, viewdirs0=vd), len(xyz), bs, 0, 3)
    rgb = torch.empty(len(xyz), 3, dtype=torch.float32, device=device)
    for first in range(0, len(xyz), bs):
        out = occu_net(xyz[None, first:first + bs], coarse=coarse, viewdirs=vd[None, first:first + bs])
        rgb[first:first + bs] = out[0, :, :3]
    return rgb


def _band(occu_net, c1, c2, reso, isosurface, sigma_idx, eval_batch_size, coarse, device, return_colors, block,
          field=None):
    """The narrow-band path of marching_cubes -> numpy (vertices in grid index units, triangles[, normals, rgb]).
    Nothing on it is sized by the full grid."""
    n_lat = pn.band_lattice_size(reso, block)
    print("Evaluating sigma @", n_lat, "coarse lattice points")
    bs = max(1, min(int(eval_batch_size), n_lat))
    lattice = _sigma(occu_net, n_lat, bs, lambda f, n, p, d: pn.band_lattice_points(c1, c2, reso, block, f, n, p, d),
                     coarse, sigma_idx, device, field, pn.point_source(pn.POINTS_LATTICE, c1, c2, reso, block))
    plan = pn.band_plan(lattice, reso, block, isosurface, apron=return_colors)
    del lattice
    M = plan.n_points
    print("Evaluating sigma @", M, "points in", plan.n_active, "active blocks")
    bs = max(1, min(int(eval_batch_size), max(M, 1)))
    if field is not None:
        field.set_plan(plan)
    sigmas = _sigma(occu_net, M, bs, lambda f, n, p, d: pn.band_points(plan, c1, c2, f, n, p, d), coarse, sigma_idx,
                    device, field, pn.point_source(pn.POINTS_BAND, c1, c2, reso, block, plan.apron, M))
    print("Running marching cubes")
    if not return_colors:
        return tuple(t.cpu().numpy() for t in pn.band_marching_cubes(sigmas, plan, isosurface))
    vertices, triangles, normals, xyz, vd = pn.band_marching_cubes(sigmas, plan, isosurface, bounds=(c1, c2))
    print("Evaluating colour @", len(xyz), "vertices")
    bs = max(1, min(int(eval_batch_size), reso[0] * reso[1] * reso[2]))      # the dense path's chunks
    rgb = _colours(occu_net, xyz, vd, bs, coarse, device, field)
    return tuple(t.cpu().numpy() for t in (vertices, triangles, normals, rgb))


class _ShardedField:
    """occu_net's field over several GPUs for one marching_cubes call: a pnr_mgpu handle over `gpus`, a
    render.nerf._SceneReplica of the scene and weights for the shards after the first (peer copies through
    pnr_mgpu_broadcast; one per device, gpus[0] included when it repeats, as bind_parallel does), and
    pnr_mgpu_field_eval for every field pass.  `close()` destroys the handle and drops the replicas."""

    def __init__(self, occu_net, gpus, coarse):
        import ctypes as C
        from render.nerf import _SceneReplica, broadcast_to
        self.gpus = gpus
        self.engine = pn.ENGINES[occu_net.engine]
        use_fine = (not coarse) and occu_net.mlp_fine is not None
        self.handle = C.c_void_p()
        pn.check(pn.lib().pnr_mgpu_create((C.c_int32 * len(gpus))(*gpus), len(gpus), C.byref(self.handle)))
        send = lambda t, d: broadcast_to(gpus, t, d, lambda: self.handle)    # noqa: E731
        try:
            self.replicas = {}
            self.shards = (pn.PnrFieldShard * len(gpus))()
            self.keep = []
            for i, g in enumerate(gpus):
                dev = torch.device("cuda", g)
                if i == 0:
                    model = occu_net
                else:
                    model = self.replicas.get(g)
                    if model is None:
                        model = self.replicas[g] = _SceneReplica(dev)
                        model.refresh(occu_net, use_fine, send=send)
                with torch.cuda.device(dev):
                    scene, mc, mf, keep = model._scene_struct(want_fine=use_fine)
                mlp = mf if use_fine else mc
                if use_fine:
                    scene.proj_coarse = scene.proj_fine      # pnr_field_eval reads proj_coarse for its mlp
                sh = self.shards[i]
                sh.scene, sh.mlp = C.pointer(scene), C.pointer(mlp)
                sh.stream = pn.stream_ptr(dev)
                self.keep += [scene, mlp, keep]
        except BaseException:
            self.close()
            raise

    def set_plan(self, plan):
        """The band plan on every device: the buffer itself on gpus[0]'s, a peer copy elsewhere."""
        from render.nerf import broadcast_to
        bufs = {self.gpus[0]: plan.buf}
        for i, g in enumerate(self.gpus):
            if g not in bufs:
                bufs[g] = broadcast_to(self.gpus, plan.buf, torch.device("cuda", g), lambda: self.handle)
            self.shards[i].plan, self.shards[i].plan_bytes = bufs[g].data_ptr(), bufs[g].numel()
        self.keep.append(bufs)

    def eval(self, src, count, chunk, channel, n_channels):
        """-> [count, n_channels] fp32 on gpus[0]: channels [channel, channel + n_channels) of the field at the points
        [0, count) of the PnrPointSource src, in chunks of `chunk` points"""
        dev0 = torch.device("cuda", self.gpus[0])
        channel = range(4)[channel]                      # (a negative index counts from the end, as in out[..., idx])
        need = {}                                        # the shards of a device run in turn: they share one workspace
        for i, g in enumerate(self.gpus):
            sh = self.shards[i]
            need[g] = max(need.get(g, 0), pn.lib().pnr_mgpu_field_workspace_bytes(sh.scene, sh.mlp, chunk, self.engine))
        ws = {g: pn.workspace(torch.device("cuda", g), n) for g, n in need.items()}
        for i, g in enumerate(self.gpus):
            self.shards[i].workspace, self.shards[i].workspace_bytes = ws[g].data_ptr(), ws[g].numel()
        out = torch.empty(count, n_channels, dtype=torch.float32, device=dev0)
        return pn.mgpu_field_eval(self.handle, self.shards, src, count, chunk, self.engine, channel, out)

    def close(self):
        if self.handle:
            pn.check(pn.lib().pnr_mgpu_destroy(self.handle))
            self.handle = None
        self.replicas, self.keep = {}, []


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
