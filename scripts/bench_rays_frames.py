#!/usr/bin/env python
"""HBM roofline of the two caller-side kernels (SURVEY 8f-3): pnr_gen_rays writes 32 B per ray, pnr_frames_u8 reads
4 B and writes 1 B per value.  Buffers are larger than the 50 MB L2; CUDA events, median of 20 after 3 warm-ups."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pixel-nerf_b200", "src"))
sys.path.insert(0, os.path.join(ROOT, "pixel-nerf_b200"))
import pnr_native as pn  # noqa: E402
import synth  # noqa: E402


def timed(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    dev = "cuda:0"
    peak = 6540.5
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    NV, W, H = 100, 400, 300
    poses = torch.stack([synth.pose_spherical(a, -25.0, 2.5) for a in np.linspace(-180, 180, NV + 1)[:-1]]).to(dev)
    rays = torch.empty(NV * W * H, 8, device=dev)
    ms = timed(lambda: pn.gen_rays(poses, W, H, 360.0, 360.0, 200.0, 150.0, 0.1, 5.0, out=rays))
    gb = rays.numel() * 4 / 1e9
    print(json.dumps({"kernel": "k_gen_rays", "rays": NV * W * H, "ms": ms, "GB_written": gb,
                      "GBps": gb / (ms / 1e3), "frac_of_measured_hbm_copy_peak": gb / (ms / 1e3) / peak,
                      "rays_per_s": NV * W * H / (ms / 1e3)}))
    rgb = torch.rand(NV * W * H, 3, device=dev)
    out = torch.empty(NV, H, W, 3, device=dev, dtype=torch.uint8)
    ms = timed(lambda: pn.frames_u8(rgb, out=out.view(-1)))
    gb = rgb.numel() * 5 / 1e9
    print(json.dumps({"kernel": "k_frames_u8", "values": rgb.numel(), "ms": ms, "GB_moved": gb,
                      "GBps": gb / (ms / 1e3), "frac_of_measured_hbm_copy_peak": gb / (ms / 1e3) / peak}))


if __name__ == "__main__":
    main()
