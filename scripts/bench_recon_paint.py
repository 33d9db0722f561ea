#!/usr/bin/env python
"""Vertex colours from the rendered views (util.recon.fuse_views(..., colors="views")) on the C2 scene (SRN-car shape:
2 source views, ResnetFC d=512 with synth.bench_mlp_weights, 64 + 32 samples per ray): a turntable of V views of
W x W pixels fused into reso^3 TSDFs over [-0.6, 0.6]^3.  Per engine and grid: device ms of pnr_paint_vertices (best
of --repeats launches on the call's own inputs, after the call's launch), device ms of the field colour pass it
replaces (util.recon._colours over every vertex, as colors="field" runs it: best of --repeats), device ms of the
fallback field pass over the vertices no view painted, the painted and fallback vertex counts, and the device ms of
the call's rendering for scale.  Prints one JSON line with the GPU's name and power limit.

    python scripts/bench_recon_paint.py [--views 64] [--res 128] [--resos 128 256] [--engines tc tc_fast]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_recon import c2_net, synth  # noqa: E402
from bench_recon_mgpu import gpu_info  # noqa: E402


def timed(fn, repeats, stream):
    """-> (the first call's result, best device ms over `repeats` calls)"""
    best, out = None, None
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        r = fn()
        b.record(stream)
        b.synchronize()
        out = r if out is None else out
        best = a.elapsed_time(b) if best is None else min(best, a.elapsed_time(b))
    return out, best


def paint_timed(net, renderer, poses, res, reso, bs, repeats):
    """One fuse_views(colors="views") call with its painting and fallback timed, then the field pass over all its
    vertices -> timings and counts"""
    import pnr_native as pn
    from util import recon as urecon
    cfg = synth.CONFIGS["c2"]
    stream = torch.cuda.current_stream()
    seen = {}
    real_paint, real_mc, real_fuse, real_colours = pn.paint_vertices, pn.marching_cubes, pn.tsdf_fuse, urecon._colours
    start = torch.cuda.Event(enable_timing=True)
    fused = torch.cuda.Event(enable_timing=True)

    def paint(*a):
        out, seen["paint_ms"] = timed(lambda: real_paint(*a), repeats, stream)
        seen["painted"] = int((out[1] > 0).sum())
        return out

    def mc(*a, **kw):
        out = real_mc(*a, **kw)
        seen["xyz"], seen["vd"] = out[3], out[4]
        return out

    def fuse(*a):
        fused.record(stream)
        return real_fuse(*a)

    def colours(*a):
        out, seen["fallback_ms"] = timed(lambda: real_colours(*a), 1, stream)
        return out
    pn.paint_vertices, pn.marching_cubes, pn.tsdf_fuse, urecon._colours = paint, mc, fuse, colours
    try:
        seen["fallback_ms"] = 0.0
        torch.cuda.synchronize()
        start.record(stream)
        torch.manual_seed(0)
        verts, tris, normals, rgb = urecon.fuse_views(net, renderer, poses, res, res, cfg["focal"] * res / cfg["W"],
                                                      cfg["z_near"], cfg["z_far"], c1=[-0.6] * 3, c2=[0.6] * 3,
                                                      reso=[reso] * 3, ray_batch_size=bs, return_colors=True,
                                                      colors="views")
        torch.cuda.synchronize()
    finally:
        pn.paint_vertices, pn.marching_cubes, pn.tsdf_fuse, urecon._colours = real_paint, real_mc, real_fuse, \
            real_colours
    with torch.no_grad():
        _, field_ms = timed(lambda: real_colours(net, seen["xyz"], seen["vd"], bs, not renderer.using_fine, "cuda"),
                            repeats, stream)
    n = len(verts)
    return {"render_device_ms": start.elapsed_time(fused), "paint_device_ms": seen["paint_ms"],
            "field_colour_device_ms": field_ms, "fallback_device_ms": seen["fallback_ms"], "vertices": n,
            "painted": seen["painted"], "fallback": n - seen["painted"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--resos", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--engines", nargs="+", default=["tc", "tc_fast"])
    ap.add_argument("--ray-batch-size", type=int, default=50000)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import util
    from render import NeRFRenderer
    cfg = synth.CONFIGS["c2"]
    r = (cfg["z_near"] + cfg["z_far"]) / 2
    poses = torch.stack([util.pose_spherical(float(t), -10.0, r) for t in np.linspace(-180, 180, a.views + 1)[:-1]])
    poses = poses.cuda()
    renderer = NeRFRenderer(n_coarse=cfg["n_coarse"], n_fine=cfg["n_fine"], n_fine_depth=cfg["n_fine_depth"],
                            white_bkgd=cfg["white_bkgd"]).cuda()
    res = {"metric": "util.recon.fuse_views(colors='views') colour stages (C2 scene)", **gpu_info(),
           "views": a.views, "res": a.res, "rays": a.views * a.res * a.res, "ray_batch_size": a.ray_batch_size,
           "repeats": a.repeats, "runs": {}}
    for engine in a.engines:
        net = c2_net(engine)
        paint_timed(net, renderer, poses[:2], 32, 32, a.ray_batch_size, 1)             # warm-up
        res["runs"][engine] = {str(reso): paint_timed(net, renderer, poses, a.res, reso, a.ray_batch_size, a.repeats)
                               for reso in a.resos}
        del net
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
