#!/usr/bin/env python
"""The single-pass tensor engine (engine "tc_fast") against the exact one ("tc") in one process, on bench.py's
scenes.

For C2, C3 and C4 (a full frame of bench.py's rays, its L2 flush between steps) the two engines alternate, round after
round, on the same net (same packed weights and projected maps) and the same rays.  Per engine it reports rays/s and the
fused kernel's device time per frame (pnr_profile_begin/end), median over the rounds, and the sm clock nvidia-smi saw.
It then renders the frame once per engine from the same seed (same noise draws) and reports fast against exact:
PSNR, max |d rgb| and p99.9 of the fine rgb on the rays whose importance samples did not flip a bin, the same including
flipped rays, and how many flipped.  Last, the util.recon sigma grid at 128^3 on the C2 scene (scripts/bench_recon.py's
loop), points/s per engine.  One JSON line per workload, then one for the recon grid and one naming the card, its
power limit and max sm clock.

    python scripts/bench_tc_fast.py [--workloads c2,c3,c4] [--rounds 3] [--steps 5]
"""
import argparse
import importlib.util
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
ENGINES = ("tc", "tc_fast")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


bench = _load("pnr_bench", os.path.join(ROOT, "bench.py"))


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def time_engine(net, render, rays, flush, steps, warmup):
    """(ms per frame, kernel ms per frame, median sm MHz) of `steps` frames after `warmup` untimed ones."""
    import pnr_native as pn

    def step():
        flush.zero_()
        with torch.no_grad():
            render(rays)

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    sampler = bench.ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    pn.profile_begin()
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    kern_ms, _ = pn.profile_end()
    sampler.stop_flag = True
    sampler.join()
    return e0.elapsed_time(e1) / steps, kern_ms / steps, sampler.summary().get("sm_mhz")


def compare(net, renderer, rays, z_far_minus_near):
    """Fast against exact on one frame rendered from the same seed: fine rgb errors and flipped rays."""
    out = {}
    for eng in ENGINES:
        net.engine = eng
        torch.manual_seed(11)
        with torch.no_grad():
            r = renderer._forward_fused(net, rays, want_weights=False, want_z=True)
        out[eng] = (r.fine.rgb.reshape(-1, 3).float(), r.fine.z.reshape(rays.shape[1], -1))
    (ra, za), (rb, zb) = out["tc"], out["tc_fast"]
    d = (rb - ra).abs().max(-1).values
    flipped = (zb - za).abs().max(-1).values > 1e-4 * z_far_minus_near
    keep = ~flipped
    mse = ((rb - ra) ** 2).mean().item()
    dk = d[keep]
    return {"rays": int(d.numel()), "psnr_db": -10 * math.log10(mse) if mse > 0 else float("inf"),
            "max_abs_drgb": float(dk.max()) if dk.numel() else None,
            "p999_abs_drgb": float(torch.quantile(dk[:1 << 24], 0.999)) if dk.numel() else None,
            "max_abs_drgb_incl_flipped": float(d.max()), "flipped_rays": int(flipped.sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2,c3,c4")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--steps-c4", type=int, default=2, help="timed frames of C4 (one C4 frame renders 120 000 rays)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--recon-reso", type=int, default=128)
    ap.add_argument("--recon-reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tc_fast.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)    # > 50 MB L2, as bench.py
    for wl in args.workloads.split(","):
        cfg = bench.synth.CONFIGS[wl]
        frame = bench.WORKLOADS[wl]["frame_rays"]
        net, renderer = bench.build_scene(cfg, dev, "tc")
        rays = bench.synth.make_rays(cfg, frame, n_target=max(8, frame // (cfg["W"] * cfg["H"]) + 1))[None].to(dev)
        render = renderer.bind_parallel(net, [0], simple_output=True).eval()
        steps = args.steps_c4 if wl == "c4" else args.steps
        runs = {e: [] for e in ENGINES}
        for _ in range(args.rounds):
            for eng in ENGINES:
                net.engine = eng
                runs[eng].append(time_engine(net, render, rays, flush, steps, args.warmup))
        res = {"workload": wl, "frame_rays": frame, "steps": steps, "rounds": args.rounds}
        for eng in ENGINES:
            ms = [r[0] for r in runs[eng]]
            kms = [r[1] for r in runs[eng]]
            res[eng] = {"rays_per_s": frame / (statistics.median(ms) / 1e3),
                        "ms_per_frame": statistics.median(ms), "kernel_ms_per_frame": statistics.median(kms),
                        "kernel_ms_runs": kms, "sm_mhz": [r[2] for r in runs[eng]]}
        res["speedup_rays_per_s"] = res["tc_fast"]["rays_per_s"] / res["tc"]["rays_per_s"]
        res["speedup_kernel"] = res["tc"]["kernel_ms_per_frame"] / res["tc_fast"]["kernel_ms_per_frame"]
        res["fast_vs_exact"] = compare(net, renderer, rays, cfg["z_far"] - cfg["z_near"])
        print(json.dumps(res), flush=True)
        del net, renderer, render, rays
        torch.cuda.empty_cache()

    import bench_recon
    reso = [args.recon_reso] * 3
    c1, c2 = [-0.6] * 3, [0.6] * 3
    rec = {"recon_sigma_grid": args.recon_reso, "points": args.recon_reso ** 3}
    nets = {e: bench_recon.c2_net(e) for e in ENGINES}
    for e in ENGINES:
        bench_recon.sigma_grid(nets[e], c1, c2, reso, 100000)              # warm-up of every chunk shape
    times = {e: [] for e in ENGINES}
    vols = {}
    for _ in range(args.recon_reps):
        for e in ENGINES:
            vols[e], ms, _ = bench_recon.timed(lambda: bench_recon.sigma_grid(nets[e], c1, c2, reso, 100000), 1)
            times[e].append(ms)
    for e in ENGINES:
        rec[e] = {"sigma_ms": statistics.median(times[e]),
                  "points_per_s": rec["points"] / statistics.median(times[e]) * 1e3}
    a, b = vols["tc"], vols["tc_fast"]
    rec["speedup"] = rec["tc"]["sigma_ms"] / rec["tc_fast"]["sigma_ms"]
    rec["max_abs_dsigma_rel"] = float((b - a).abs().max() / (1 + a.abs().max()))
    print(json.dumps(rec), flush=True)
    print(json.dumps({"card": smi("name,power.limit,clocks.max.sm")}), flush=True)


if __name__ == "__main__":
    main()
