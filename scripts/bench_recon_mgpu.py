#!/usr/bin/env python
"""Mesh extraction with the field passes sharded over several GPUs (util.recon.marching_cubes(..., gpus=...)) on the
C2 scene (SRN-car shape: 2 source views, ResnetFC d=512 with synth.bench_mlp_weights).  Per device list: the replica
refresh (handle, scene and weight copies; device ms on gpus[0]'s stream and wall ms), then the sigma passes of the
extraction (dense: the grid; block b: the lattice, the plan's count download, the refinement set) and with --colors
the colour pass over the vertices, as device ms on gpus[0]'s stream and wall ms, and whether sigma, mesh and colours
are bit-equal to the first device list's.  On one card "0 0" against "0" is the sharded driver's overhead; scaling
needs several free GPUs.  Prints one JSON line with the GPUs' names and power limits.

    python scripts/bench_recon_mgpu.py --gpus "0" "0 0" [--reso 512] [--block 4] [--colors] [--engine tc]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_recon import c2_net, sigma_grid  # noqa: E402


def gpu_info():
    info = {"gpus": [torch.cuda.get_device_name(i) for i in range(torch.cuda.device_count())]}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limits"] = q.stdout.strip().splitlines() if q.returncode == 0 else None
    except (OSError, subprocess.SubprocessError):
        info["power_limits"] = None
    return info


class Clock:
    """device ms on cuda:g0's current stream and wall ms of a block"""

    def __init__(self, g0):
        self.dev = torch.device("cuda", g0)

    def __enter__(self):
        torch.cuda.synchronize()
        self.ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self.ev[0].record(torch.cuda.current_stream(self.dev))
        self.t = time.perf_counter()
        return self

    def __exit__(self, *exc):
        self.ev[1].record(torch.cuda.current_stream(self.dev))
        torch.cuda.synchronize()
        self.wall_ms = (time.perf_counter() - self.t) * 1e3
        self.device_ms = self.ev[0].elapsed_time(self.ev[1])


def extract(net, gpus, reso, block, iso, bs, colors):
    """util.recon's passes, timed: -> (timings, arrays to compare)"""
    import pnr_native as pn
    from util import recon as urecon
    c1, c2 = [-0.6] * 3, [0.6] * 3
    dev = torch.device("cuda", gpus[0])
    t = {}
    with torch.no_grad():
        with Clock(gpus[0]) as ck:
            field = urecon._ShardedField(net, gpus, True) if len(gpus) > 1 else None
        t["refresh_device_ms"], t["refresh_wall_ms"] = ck.device_ms, ck.wall_ms
        try:
            with Clock(gpus[0]) as ck:
                if block is None:
                    N = int(np.prod(reso))
                    sigma = urecon._sigma(net, N, min(bs, N), lambda f, n, p, d: pn.grid_points(c1, c2, reso, f, n, p, d),
                                          True, 3, dev, field, pn.point_source(pn.POINTS_GRID, c1, c2, reso))
                    arrays = [sigma]
                else:
                    n_lat = pn.band_lattice_size(reso, block)
                    lat = urecon._sigma(net, n_lat, min(bs, n_lat),
                                        lambda f, n, p, d: pn.band_lattice_points(c1, c2, reso, block, f, n, p, d), True,
                                        3, dev, field, pn.point_source(pn.POINTS_LATTICE, c1, c2, reso, block))
                    plan = pn.band_plan(lat, reso, block, iso, apron=colors)
                    if field is not None:
                        field.set_plan(plan)
                    M = plan.n_points
                    sigma = urecon._sigma(net, M, max(1, min(bs, M)),
                                          lambda f, n, p, d: pn.band_points(plan, c1, c2, f, n, p, d), True, 3, dev,
                                          field, pn.point_source(pn.POINTS_BAND, c1, c2, reso, block, plan.apron, M))
                    arrays = [lat, sigma]
            t["sigma_device_ms"], t["sigma_wall_ms"], t["points"] = ck.device_ms, ck.wall_ms, sum(a.numel() for a in arrays)
            if colors:
                if block is None:
                    v, tri, nrm, xyz, vd = pn.marching_cubes(sigma.view(*reso), iso, bounds=(c1, c2))
                else:
                    v, tri, nrm, xyz, vd = pn.band_marching_cubes(sigma, plan, iso, bounds=(c1, c2))
                with Clock(gpus[0]) as ck:
                    rgb = urecon._colours(net, xyz, vd, min(bs, int(np.prod(reso))), True, dev, field)
                t["colour_device_ms"], t["colour_wall_ms"], t["vertices"] = ck.device_ms, ck.wall_ms, len(xyz)
                arrays += [v, tri, nrm, rgb]
        finally:
            if field is not None:
                field.close()
    return t, [a.cpu().numpy() for a in arrays]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", nargs="+", default=["0", "0 0"])
    ap.add_argument("--reso", type=int, default=512)
    ap.add_argument("--block", type=int, default=None)
    ap.add_argument("--colors", action="store_true")
    ap.add_argument("--engine", default="tc")
    ap.add_argument("--eval-batch-size", type=int, default=100000)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    lists = [[int(g) for g in s.split()] for s in a.gpus]
    reso = [a.reso] * 3
    net = c2_net(a.engine)
    iso = float(sigma_grid(net, [-0.6] * 3, [0.6] * 3, [32] * 3, a.eval_batch_size).median())
    res = {"metric": "util.recon.marching_cubes field passes sharded over gpus (C2 scene)", **gpu_info(),
           "engine": a.engine, "reso": a.reso, "block": a.block, "colors": a.colors,
           "eval_batch_size": a.eval_batch_size, "iso": iso, "runs": {}}
    first = None
    for gpus in lists:
        extract(net, gpus, [64] * 3, a.block, iso, a.eval_batch_size, a.colors)       # warm-up
        runs = [extract(net, gpus, reso, a.block, iso, a.eval_batch_size, a.colors) for _ in range(a.repeats)]
        best = {k: min(r[0][k] for r in runs) for k in runs[0][0]}
        arrays = runs[-1][1]
        if first is None:
            first = arrays
        best["bit_equal_to_first"] = all(x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))
                                         for x, y in zip(arrays, first))
        res["runs"][" ".join(map(str, gpus))] = best
        del runs, arrays
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
