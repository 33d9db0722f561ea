#!/usr/bin/env python
"""Decimation of extracted meshes (util.recon.decimate) on the C2 scene (as scripts/bench_recon_components.py): dense
marching cubes at each --reso and the narrow band (block 4) at --band, each after keep_components(largest=1), and the
fuse_views mesh (64 views of 128^2 at 256^3; --no-fuse skips it), each decimated to every --fractions of its
triangles.  Per run: rounds, the fraction of the live vertices each round collapses (first, median, last), device ms
per round (select + apply, each ending in its synchronise, by the host clock) and in total, and the wall ms of
decimate() end to end with its copies and compaction.  Prints one JSON line with the GPU's name and power limit.

    python scripts/bench_recon_decimate.py [--reso 512] [--band 1024] [--fractions 0.1 0.01] [--no-fuse]

The band mesh's sigma alone takes about 25 s; --band with no value skips it.
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_recon import c2_net, sigma_grid, synth  # noqa: E402
from bench_recon_mgpu import gpu_info  # noqa: E402

C1, C2 = [-0.6] * 3, [0.6] * 3


def rounds(verts, tris, target):
    """decimate()'s round loop, timed per round"""
    import pnr_native as pn
    xyz = torch.from_numpy(np.ascontiguousarray(verts, dtype=np.float64)).cuda()
    d = pn.Decimator(xyz, torch.from_numpy(np.ascontiguousarray(tris, dtype=np.int64)).cuda())
    live, m, ms, frac = len(np.unique(tris)), len(tris), [], []
    while m > target:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c, dd, err, _ = d.select()
        if len(c) == 0:
            break
        need = -(-(m - target) // 2)
        if len(c) > need:
            o = torch.sort(torch.minimum(c, dd), stable=True).indices
            o = torch.sort(o[torch.sort(err[o], stable=True).indices[:need]]).values
            c, dd = c[o], dd[o]
        m = d.apply(c, dd)
        ms.append((time.perf_counter() - t0) * 1e3)
        frac.append(len(c) / live)
        live -= len(c)
    return ms, frac, m


def measure(verts, tris, fractions):
    from util import recon as urecon
    out = {"vertices": len(verts), "triangles": len(tris)}
    for f in fractions:
        target = int(len(tris) * f)
        ms, frac, m = rounds(verts, tris, target)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            got = urecon.decimate(verts, tris, target_triangles=target)
        wall = (time.perf_counter() - t0) * 1e3
        assert len(got[1]) == m
        out[f"to_{f:g}"] = {"target": target, "triangles": m, "rounds": len(ms),
                            "collapsed_fraction_first_median_last": [frac[0], float(np.median(frac)), frac[-1]]
                            if frac else [], "round_ms_median": float(np.median(ms)) if ms else 0.0,
                            "round_ms_max": max(ms) if ms else 0.0, "device_ms_total": sum(ms),
                            "decimate_wall_ms": wall}
        print(json.dumps({"progress": out}), file=sys.stderr, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reso", type=int, nargs="*", default=[512])
    ap.add_argument("--band", type=int, nargs="*", default=[1024], help="band meshes (block 4) at these resolutions")
    ap.add_argument("--fractions", type=float, nargs="*", default=[0.1, 0.01])
    ap.add_argument("--no-fuse", action="store_true")
    ap.add_argument("--engine", default="tc")
    ap.add_argument("--eval-batch-size", type=int, default=100000)
    a = ap.parse_args()
    import pnr_native as pn
    from util import recon as urecon
    net = c2_net(a.engine)
    bs = a.eval_batch_size
    iso = float(sigma_grid(net, C1, C2, [32] * 3, bs).median())
    res = {"metric": "util.recon.decimate (C2 scene)", **gpu_info(), "engine": a.engine, "iso": iso, "meshes": {}}
    rounds(np.eye(3), np.array([[0, 1, 2]]), 0)                               # warm-up
    quiet = contextlib.redirect_stdout(io.StringIO())
    for r in a.reso:
        v, t = pn.marching_cubes(sigma_grid(net, C1, C2, [r] * 3, bs).view(r, r, r), iso)
        with quiet:
            v, t = urecon.keep_components(v.cpu().numpy(), t.cpu().numpy(), largest=1)
        torch.cuda.empty_cache()
        res["meshes"][f"dense_{r}_largest"] = measure(v, t, a.fractions)
    for r in a.band:
        with contextlib.redirect_stdout(io.StringIO()):
            v, t = urecon.keep_components(*urecon.marching_cubes(net, C1, C2, [r] * 3, isosurface=iso,
                                                                 eval_batch_size=bs, block=4), largest=1)
        torch.cuda.empty_cache()
        res["meshes"][f"band_{r}_b4_largest"] = measure(v, t, a.fractions)
    if not a.no_fuse:
        import util
        from render import NeRFRenderer
        cfg = synth.CONFIGS["c2"]
        rad = (cfg["z_near"] + cfg["z_far"]) / 2
        poses = torch.stack([util.pose_spherical(float(p), -10.0, rad) for p in np.linspace(-180, 180, 65)[:-1]])
        renderer = NeRFRenderer(n_coarse=cfg["n_coarse"], n_fine=cfg["n_fine"], n_fine_depth=cfg["n_fine_depth"],
                                white_bkgd=cfg["white_bkgd"]).cuda()
        with contextlib.redirect_stdout(io.StringIO()):
            v, t = urecon.keep_components(*urecon.fuse_views(
                net, renderer, poses.cuda(), 128, 128, cfg["focal"] * 128 / cfg["W"], cfg["z_near"], cfg["z_far"],
                c1=C1, c2=C2, reso=[256] * 3), largest=1)
        res["meshes"]["fuse_256_64x128_largest"] = measure(v, t, a.fractions)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
