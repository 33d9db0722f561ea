#!/usr/bin/env python
"""Connected components of extracted meshes (util.recon.keep_components) on the C2 scene (SRN-car shape: 2 source
views, ResnetFC d=512 with synth.bench_mlp_weights, tensor engine).  The meshes: dense marching cubes of the sigma grid
over [-0.6, 0.6]^3 at each --reso, the narrow band (block 4) at --band (its sigma takes tens of seconds), and a
fuse_views mesh (a turntable of 64 views of 128^2 fused at 256^3; --no-fuse skips it).  Per mesh: vertices, triangles, components,
the triangles largest=1 keeps; device ms of pnr_mesh_components (with its count download) and of pnr_mesh_compact_count
+ _emit (with theirs), best of --reps on the same mesh by CUDA events; wall ms of keep_components(v, t, largest=1) end
to end, host<->device copies included; and host ms of scipy's connected_components on the same vertex graph, for
scale.  Prints one JSON line with the GPU's name and power limit.

    python scripts/bench_recon_components.py [--reso 256 512] [--band 1024] [--no-fuse] [--reps 5]
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch
from scipy.sparse.csgraph import connected_components

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_recon import c2_net, sigma_grid, synth  # noqa: E402
from bench_recon_mgpu import gpu_info  # noqa: E402

C1, C2 = [-0.6] * 3, [0.6] * 3


def device_ms(fn, reps):
    """best CUDA-event ms of fn() over reps calls, and its last result"""
    best, out = float("inf"), None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b))
    return best, out


def measure(verts, tris, reps):
    import pnr_native as pn
    from util import recon as urecon
    n, m = len(verts), len(tris)
    t_d = torch.from_numpy(np.ascontiguousarray(tris, dtype=np.int64)).cuda()
    cc_ms, (label, tri_count, n_comp) = device_ms(lambda: pn.mesh_components(t_d, n), reps)
    roots = torch.nonzero(tri_count).view(-1)
    top = roots[torch.sort(tri_count[roots], descending=True, stable=True).indices[:1]]
    keep_root = torch.zeros(n, dtype=torch.uint8, device="cuda")
    keep_root[top] = 1
    compact_ms, (vert_ids, _) = device_ms(lambda: pn.mesh_compact(t_d, n, label, keep_root), reps)
    del t_d, label, tri_count, keep_root, vert_ids
    walls = []
    for _ in range(max(1, reps // 2)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            kv, kt = urecon.keep_components(verts, tris, largest=1)
        walls.append((time.perf_counter() - t0) * 1e3)
    t0 = time.perf_counter()
    rows = np.concatenate([tris[:, 0], tris[:, 0]])
    graph = sp.coo_matrix((np.ones(2 * m, dtype=np.int8), (rows, np.concatenate([tris[:, 1], tris[:, 2]]))),
                          shape=(n, n)).tocsr()
    t1 = time.perf_counter()
    n_scipy, _ = connected_components(graph, directed=False)
    t2 = time.perf_counter()
    unused = n - len(np.unique(tris))
    return {"vertices": n, "triangles": m, "components": n_comp, "largest_kept_triangles": len(kt),
            "largest_kept_vertices": len(kv), "components_device_ms": cc_ms, "compact_device_ms": compact_ms,
            "keep_components_wall_ms": min(walls), "scipy_graph_ms": (t1 - t0) * 1e3,
            "scipy_connected_components_ms": (t2 - t1) * 1e3, "agrees_with_scipy": n_scipy - unused == n_comp}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reso", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--band", type=int, nargs="*", default=[], help="band meshes (block 4) at these resolutions")
    ap.add_argument("--no-fuse", action="store_true", help="skip the fuse_views mesh (64 views of 128^2 at 256^3)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--engine", default="tc")
    ap.add_argument("--eval-batch-size", type=int, default=100000)
    a = ap.parse_args()
    import pnr_native as pn
    from util import recon as urecon
    net = c2_net(a.engine)
    bs = a.eval_batch_size
    iso = float(sigma_grid(net, C1, C2, [32] * 3, bs).median())          # a level the field crosses
    res = {"metric": "util.recon.keep_components (C2 scene)", **gpu_info(), "engine": a.engine, "iso": iso,
           "reps": a.reps, "meshes": {}}
    measure(np.zeros((3, 3)), np.array([[0, 1, 2]]), 2)                   # warm-up
    for r in a.reso:
        v, t = pn.marching_cubes(sigma_grid(net, C1, C2, [r] * 3, bs).view(r, r, r), iso)
        res["meshes"][f"dense_{r}"] = measure(v.cpu().numpy(), t.cpu().numpy(), a.reps)
        del v, t
        torch.cuda.empty_cache()
    for r in a.band:
        with contextlib.redirect_stdout(io.StringIO()):
            v, t = urecon.marching_cubes(net, C1, C2, [r] * 3, isosurface=iso, eval_batch_size=bs, block=4)
        res["meshes"][f"band_{r}_b4"] = measure(v, t, a.reps)
        torch.cuda.empty_cache()
    if not a.no_fuse:
        import util
        from render import NeRFRenderer
        cfg = synth.CONFIGS["c2"]
        rad = (cfg["z_near"] + cfg["z_far"]) / 2
        poses = torch.stack([util.pose_spherical(float(p), -10.0, rad) for p in np.linspace(-180, 180, 65)[:-1]])
        renderer = NeRFRenderer(n_coarse=cfg["n_coarse"], n_fine=cfg["n_fine"], n_fine_depth=cfg["n_fine_depth"],
                                white_bkgd=cfg["white_bkgd"]).cuda()
        with contextlib.redirect_stdout(io.StringIO()):
            v, t = urecon.fuse_views(net, renderer, poses.cuda(), 128, 128, cfg["focal"] * 128 / cfg["W"],
                                     cfg["z_near"], cfg["z_far"], c1=C1, c2=C2, reso=[256] * 3)
        res["meshes"]["fuse_256_64x128"] = measure(v, t, a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
