#!/usr/bin/env python
"""Mesh extraction (util.recon.marching_cubes) on the C2 scene (SRN-car shape: 2 source views, ResnetFC d=512 with
synth.bench_mlp_weights, tensor engine): device time of the sigma grid (pnr_grid_points + the fused field, chunks of
eval_batch_size points, as util.recon runs it) and of marching cubes (pnr_mc_count, the count download, pnr_mc_emit)
at 128^3 and 256^3.  Prints one JSON line with the GPU's name and power limit.

With --colors it also times what return_colors=True adds: one pnr_mc_vertex_attrs launch (normals, query points and
view directions of every vertex) and the field evaluation at the vertices (chunks of eval_batch_size, as util.recon
runs it), both in device ms, with the vertex count.

    python scripts/bench_recon.py [--reso 128 256] [--reps 5] [--engine tc] [--colors]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pixel-nerf_b200", "src"))
sys.path.insert(0, os.path.join(ROOT, "pixel-nerf_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth  # noqa: E402


def c2_net(engine):
    import gpu_util
    from model import make_model
    cfg = synth.CONFIGS["c2"]
    net = make_model(gpu_util.model_conf(cfg["d_hidden"]))
    net.mlp_coarse.load_state_dict(synth.bench_mlp_weights(11, cfg["d_hidden"]))
    net.mlp_fine.load_state_dict(synth.bench_mlp_weights(12, cfg["d_hidden"]))
    net = net.cuda().eval()
    net.engine = engine
    src, _, focal, c = synth.make_cameras(cfg)
    latent = synth.make_latent(5, cfg["NS"], cfg["H"] // 2, cfg["W"] // 2)
    net.set_scene(latent.cuda(), src[None].cuda(), focal.cuda(), c[None].cuda(), cfg["W"], cfg["H"])
    return net


def sigma_grid(net, c1, c2, reso, bs):
    """util.recon.marching_cubes' evaluation loop."""
    import pnr_native as pn
    N = int(np.prod(reso))
    pts = torch.empty(bs, 3, device="cuda")
    vd = torch.empty(bs, 3, device="cuda")
    sig = torch.empty(N, device="cuda")
    with torch.no_grad():
        for first in range(0, N, bs):
            n = min(bs, N - first)
            pn.grid_points(c1, c2, reso, first, n, pts, vd)
            sig[first:first + n] = net(pts[None, :n], coarse=True, viewdirs=vd[None, :n])[0, :, 3]
    return sig.view(*reso)


def vertex_colours(net, xyz, vd, bs):
    """util.recon.marching_cubes' colour loop."""
    rgb = torch.empty(len(xyz), 3, device="cuda")
    with torch.no_grad():
        for first in range(0, len(xyz), bs):
            out = net(xyz[None, first:first + bs], coarse=True, viewdirs=vd[None, first:first + bs])
            rgb[first:first + bs] = out[0, :, :3]
    return rgb


def attrs_call(vol, iso, c1, c2):
    """pnr_mc_count on a fresh workspace, then a closure that launches pnr_mc_vertex_attrs on it; -> (closure, n_verts,
    (xyz, viewdirs))."""
    import pnr_native as pn
    L = pn.lib()
    nx, ny, nz = vol.shape
    ws = torch.empty(int(L.pnr_mc_workspace_bytes(nx, ny, nz)), dtype=torch.uint8, device="cuda")
    counts = torch.empty(2, dtype=torch.int64, device="cuda")
    s = pn.stream_ptr(vol.device)
    pn.check(L.pnr_mc_count(pn.dptr(vol), nx, ny, nz, iso, C.c_void_p(counts.data_ptr()), C.c_void_p(ws.data_ptr()),
                            ws.numel(), s))
    nv = int(counts[0])
    normals = torch.empty(nv, 3, dtype=torch.float64, device="cuda")
    xyz, vd = torch.empty(nv, 3, device="cuda"), torch.empty(nv, 3, device="cuda")
    lo, hi = (C.c_double * 3)(*c1), (C.c_double * 3)(*c2)

    def launch():
        pn.check(L.pnr_mc_vertex_attrs(pn.dptr(vol), nx, ny, nz, iso, lo, hi, C.c_void_p(normals.data_ptr()),
                                       pn.dptr(xyz), pn.dptr(vd), nv, C.c_void_p(ws.data_ptr()), ws.numel(), s))
        return ws                       # keeps the workspace alive with the closure
    return launch, nv, (xyz, vd)


def timed(fn, reps):
    out, ms = None, []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return out, float(np.median(ms)), float(np.min(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reso", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--engine", default="tc")
    ap.add_argument("--eval-batch-size", type=int, default=100000)
    ap.add_argument("--colors", action="store_true", help="also time the vertex attributes and vertex colours")
    a = ap.parse_args()
    import pnr_native as pn
    net = c2_net(a.engine)
    c1, c2 = [-0.6] * 3, [0.6] * 3
    probe = sigma_grid(net, c1, c2, [32] * 3, a.eval_batch_size)
    iso = float(probe.median())                          # a level the field crosses
    res = {"metric": "util.recon.marching_cubes device ms (C2 scene)", "engine": a.engine, "iso": iso,
           "eval_batch_size": a.eval_batch_size, "gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        res["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else None
    except (OSError, subprocess.SubprocessError, IndexError):
        res["power_limit_and_max_sm_clock"] = None
    for r in a.reso:
        reso = [r] * 3
        sigma_grid(net, c1, c2, reso, a.eval_batch_size)          # warm-up of every chunk shape
        vol, s_med, s_min = timed(lambda: sigma_grid(net, c1, c2, reso, a.eval_batch_size), a.reps)
        pn.marching_cubes(vol, iso)
        (v, t), m_med, m_min = timed(lambda: pn.marching_cubes(vol, iso), a.reps)
        n = r ** 3
        res[str(r)] = {"points": n, "sigma_ms": s_med, "sigma_ms_min": s_min, "points_per_s": n / s_med * 1e3,
                       "mc_ms": m_med, "mc_ms_min": m_min, "verts": int(v.shape[0]), "tris": int(t.shape[0]),
                       "mc_workspace_mb": pn.lib().pnr_mc_workspace_bytes(r, r, r) / 2 ** 20}
        if a.colors:
            launch, nv, (xyz, vd) = attrs_call(vol, iso, c1, c2)
            launch()
            _, a_med, a_min = timed(launch, a.reps)
            vertex_colours(net, xyz, vd, a.eval_batch_size)
            _, f_med, f_min = timed(lambda: vertex_colours(net, xyz, vd, a.eval_batch_size), a.reps)
            res[str(r)].update({"colour_verts": nv, "attrs_ms": a_med, "attrs_ms_min": a_min, "vertex_field_ms": f_med,
                                "vertex_field_ms_min": f_min, "vertex_points_per_s": nv / f_med * 1e3})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
