#!/usr/bin/env python
"""Mesh extraction from rendered depth maps (util.recon.fuse_views) on the C2 scene (SRN-car shape: 2 source views,
ResnetFC d=512 with synth.bench_mlp_weights, 64 + 32 samples per ray): a turntable of V views of W x W pixels fused
into a reso^3 TSDF over [-0.6, 0.6]^3.  Per engine: device ms of the three stages of one fuse_views call on the
device's stream -- rendering (ray generation, the fused render of every pixel, the depth and opacity maps), fusion
(pnr_tsdf_fuse) and marching cubes (pnr_mc_count, the count download, pnr_mc_emit) -- the wall ms of the call, the
vertex and triangle counts and the peak memory torch allocated.  Best of --repeats after a small warm-up call.
Prints one JSON line with the GPU's name and power limit.

    python scripts/bench_recon_fuse.py [--views 64] [--res 128] [--reso 256] [--engines tc tc_fast]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_recon import c2_net, synth  # noqa: E402
from bench_recon_mgpu import gpu_info  # noqa: E402


def fuse_timed(net, renderer, poses, res, reso, bs):
    """One fuse_views call with CUDA events at the stage boundaries -> timings"""
    import pnr_native as pn
    from util import recon as urecon
    cfg = synth.CONFIGS["c2"]
    stream = torch.cuda.current_stream()
    ev = {k: torch.cuda.Event(enable_timing=True) for k in ("start", "fuse0", "fuse1", "mc0", "mc1")}
    real_fuse, real_mc = pn.tsdf_fuse, pn.marching_cubes

    def fuse(*a):
        ev["fuse0"].record(stream)
        out = real_fuse(*a)
        ev["fuse1"].record(stream)
        return out

    def mc(*a, **kw):
        ev["mc0"].record(stream)
        out = real_mc(*a, **kw)
        ev["mc1"].record(stream)
        return out
    pn.tsdf_fuse, pn.marching_cubes = fuse, mc
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        ev["start"].record(stream)
        verts, tris = urecon.fuse_views(net, renderer, poses, res, res, cfg["focal"] * res / cfg["W"], cfg["z_near"],
                                        cfg["z_far"], c1=[-0.6] * 3, c2=[0.6] * 3, reso=[reso] * 3, ray_batch_size=bs)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    finally:
        pn.tsdf_fuse, pn.marching_cubes = real_fuse, real_mc
    return {"render_device_ms": ev["start"].elapsed_time(ev["fuse0"]),
            "fuse_device_ms": ev["fuse0"].elapsed_time(ev["fuse1"]),
            "mc_device_ms": ev["mc0"].elapsed_time(ev["mc1"]), "wall_ms": wall,
            "peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30, "vertices": len(verts), "triangles": len(tris)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--reso", type=int, default=256)
    ap.add_argument("--engines", nargs="+", default=["tc", "tc_fast"])
    ap.add_argument("--ray-batch-size", type=int, default=50000)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    import util
    from render import NeRFRenderer
    cfg = synth.CONFIGS["c2"]
    r = (cfg["z_near"] + cfg["z_far"]) / 2
    poses = torch.stack([util.pose_spherical(float(t), -10.0, r) for t in np.linspace(-180, 180, a.views + 1)[:-1]])
    poses = poses.cuda()
    renderer = NeRFRenderer(n_coarse=cfg["n_coarse"], n_fine=cfg["n_fine"], n_fine_depth=cfg["n_fine_depth"],
                            white_bkgd=cfg["white_bkgd"]).cuda()
    res = {"metric": "util.recon.fuse_views stages (C2 scene)", **gpu_info(), "views": a.views, "res": a.res,
           "reso": a.reso, "rays": a.views * a.res * a.res, "ray_batch_size": a.ray_batch_size, "runs": {}}
    for engine in a.engines:
        net = c2_net(engine)
        fuse_timed(net, renderer, poses[:2], 32, 32, a.ray_batch_size)                 # warm-up
        runs = [fuse_timed(net, renderer, poses, a.res, a.reso, a.ray_batch_size) for _ in range(a.repeats)]
        best = {k: min(run[k] for run in runs) for k in runs[0]}
        best["rays_per_s"] = res["rays"] / (best["render_device_ms"] / 1e3)
        res["runs"][engine] = best
        del net
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
