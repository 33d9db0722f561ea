#!/usr/bin/env python
"""Narrow-band against dense mesh extraction (util.recon.marching_cubes with and without block=) on the C2 scene
(SRN-car shape: 2 source views, ResnetFC d=512 with synth.bench_mlp_weights), per engine: points evaluated, sigma
device ms (every field pass, chunks of eval_batch_size points, as util.recon runs them), marching-cubes device ms
(dense: pnr_mc_count, the count download, pnr_mc_emit; band: pnr_band_plan and its count download,
pnr_band_mc_count, the count download, pnr_band_mc_emit), torch.cuda.max_memory_allocated over the whole extraction,
vertex and triangle counts, whether coverage was complete (every cell the dense surface crosses lies in an active
block; only known where the dense volume was computed) and, beside a dense run, whether the mesh arrays are identical.
Prints one JSON line with the GPU's name, power limit and SM clock.

    python scripts/bench_recon_band.py [--reso 256 512] [--band-only 1024] [--blocks 4 8 16] [--engines tc tc_fast]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_recon import c2_net, sigma_grid, timed  # noqa: E402


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_sm_clock_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else None
    except (OSError, subprocess.SubprocessError, IndexError):
        info["power_limit_sm_clock_max_sm_clock"] = None
    return info


def band_sigma(net, c1, c2, reso, b, bs, iso, apron=False):
    """util.recon's two field passes of the narrow band -> (plan, refinement sigma, lattice points)."""
    import pnr_native as pn
    n_lat = pn.band_lattice_size(reso, b)
    pts = torch.empty(bs, 3, device="cuda")
    vd = torch.empty(bs, 3, device="cuda")
    with torch.no_grad():
        lat = torch.empty(n_lat, device="cuda")
        for first in range(0, n_lat, bs):
            n = min(bs, n_lat - first)
            pn.band_lattice_points(c1, c2, reso, b, first, n, pts, vd)
            lat[first:first + n] = net(pts[None, :n], coarse=True, viewdirs=vd[None, :n])[0, :, 3]
        plan = pn.band_plan(lat, reso, b, iso, apron)
        sig = torch.empty(plan.n_points, device="cuda")
        for first in range(0, plan.n_points, bs):
            n = min(bs, plan.n_points - first)
            pn.band_points(plan, c1, c2, first, n, pts, vd)
            sig[first:first + n] = net(pts[None, :n], coarse=True, viewdirs=vd[None, :n])[0, :, 3]
    return plan, sig, lat


def complete_coverage(vol, lat, reso, b, iso):
    """every non-empty dense cell in an active block, from the dense volume and the lattice sigma (torch, on the GPU)"""
    ins = torch.isfinite(vol) & (vol > iso)
    c = ins[:-1, :-1, :-1]
    mixed = torch.zeros_like(c)
    for k in range(1, 8):
        dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        mixed |= ins[dx:reso[0] - 1 + dx, dy:reso[1] - 1 + dy, dz:reso[2] - 1 + dz] != c
    del ins, c
    m = [(n - 1 + b - 1) // b + 1 for n in reso]
    li = (torch.isfinite(lat) & (lat > iso)).view(*m)
    nb = [x - 1 for x in m]
    seeded = torch.zeros(nb, dtype=torch.bool, device=vol.device)
    for k in range(1, 8):
        dx, dy, dz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        seeded |= li[dx:dx + nb[0], dy:dy + nb[1], dz:dz + nb[2]] != li[:nb[0], :nb[1], :nb[2]]
    active = F.max_pool3d(seeded[None, None].float(), 3, 1, 1)[0, 0] > 0
    cells = active.repeat_interleave(b, 0)[:reso[0] - 1].repeat_interleave(b, 1)[:, :reso[1] - 1]
    cells = cells.repeat_interleave(b, 2)[:, :, :reso[2] - 1]
    return bool((cells | ~mixed).all())


def run(net, reso, b, iso, bs, dense=None):
    import pnr_native as pn
    c1, c2 = [-0.6] * 3, [0.6] * 3
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    if b is None:
        vol, s_ms, _ = timed(lambda: sigma_grid(net, c1, c2, reso, bs), 1)
        (v, t), m_ms, _ = timed(lambda: pn.marching_cubes(vol, iso), 1)
        points, extra = int(np.prod(reso)), {}
        keep = (vol, v.cpu().numpy(), t.cpu().numpy())
    else:
        (plan, sig, lat), s_ms, _ = timed(lambda: band_sigma(net, c1, c2, reso, b, bs, iso), 1)

        def mesh():
            p = pn.band_plan(lat, reso, b, iso)                    # the plan step again, timed with marching cubes
            return pn.band_marching_cubes(sig, p, iso)
        (v, t), m_ms, _ = timed(mesh, 1)
        points = int(lat.numel() + plan.n_points)
        extra = {"lattice_points": int(lat.numel()), "refine_points": plan.n_points, "active_blocks": plan.n_active}
        keep = None
    peak = torch.cuda.max_memory_allocated() - base
    out = {"points": points, "sigma_ms": s_ms, "mc_ms": m_ms, "peak_alloc_mb": peak / 2 ** 20,
           "verts": int(v.shape[0]), "tris": int(t.shape[0]), **extra}
    if b is not None and dense is not None:
        vol, dv, dt = dense
        out["complete_coverage"] = complete_coverage(vol, lat, reso, b, iso)
        out["identical_to_dense"] = bool(np.array_equal(v.cpu().numpy().view(np.int64), dv.view(np.int64))
                                         and np.array_equal(t.cpu().numpy(), dt))
    elif b is not None:
        out["complete_coverage"] = None                  # unknown without the dense volume
    return out, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reso", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--band-only", type=int, nargs="*", default=[1024])
    ap.add_argument("--blocks", type=int, nargs="+", default=[4, 8, 16])
    ap.add_argument("--engines", nargs="+", default=["tc", "tc_fast"])
    ap.add_argument("--eval-batch-size", type=int, default=100000)
    a = ap.parse_args()
    res = {"metric": "util.recon.marching_cubes dense vs narrow band (C2 scene)", **gpu_info(),
           "eval_batch_size": a.eval_batch_size}
    bs = a.eval_batch_size
    for engine in a.engines:
        net = c2_net(engine)
        probe = sigma_grid(net, [-0.6] * 3, [0.6] * 3, [32] * 3, bs)
        iso = float(probe.median())                      # a level the field crosses
        run(net, [64] * 3, None, iso, bs)                # warm-up of both paths
        run(net, [64] * 3, 4, iso, bs)
        rows = res[engine] = {"iso": iso}
        for r in a.reso:
            reso = [r] * 3
            rows[f"{r}/dense"], dense = run(net, reso, None, iso, bs)
            for b in a.blocks:
                rows[f"{r}/b{b}"], _ = run(net, reso, b, iso, bs, dense)
            del dense
            torch.cuda.empty_cache()
        for r in a.band_only:
            for b in a.blocks:
                rows[f"{r}/b{b}"], _ = run(net, [r] * 3, b, iso, bs)
            torch.cuda.empty_cache()
        del net
    res["power_after"] = gpu_info()["power_limit_sm_clock_max_sm_clock"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
