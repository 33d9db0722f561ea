#!/usr/bin/env python
"""Where the tensor engine's time goes: a phase profile of the fused render kernel on bench.py's scenes.

Loads the profile build of the library (`make -C pixel-nerf_b200/csrc prof` -> lib/libpnr_sm90_prof.so, compiled with
-DPNR_TC_PROFILE), renders full frames of bench.py's C2, C3 and C4 rays with the exact ("tc") and the single-pass
("tc_fast") engine, and reads the kernel's 8 phase counters (pnr_tc_counters): clock64() time the first thread of each
warpgroup spent waiting on a weight slot (FULL), in wgmma_wait (retiring the previous step with wait_group 0 before
the next step's FULL wait, and the drains that end an MMA run), in the 256-thread barrier of the consumers, gathering
the projected latent, in geometry and the fine pass's `ready` poll, finishing rays (flush), and in all; and the time
the ring's refills took to issue, counted on the producer lane of each ring (not the time it waits for releases).
They are printed as SM clocks per weight step (a step is one 64-wide k-chunk of 128 weight rows: 9 or 12 wgmma per
warpgroup); "other" is the first thread's total less its own phases (wgmma issue, epilogue arithmetic); the refills
run on the producer warpgroup beside them and are not subtracted.  Each
line names the card, its power limit and the SM clock sampled during the frames.  The counters change the timing a
little; the production library is timed by bench.py.

With --dump DIR each (workload, engine) frame is also rendered once from a fixed seed and its rgb / depth saved as
DIR/<workload>_<engine>_{rgb,depth}.npy, so that two libraries can be compared bit for bit (any library works for
this; only the profile build fills the counters).

    python scripts/tc_phase_profile.py --lib pixel-nerf_b200/lib/libpnr_sm90_prof.so [--workloads c2,c3,c4]
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ("full_wait", "refill", "wgmma_wait", "workers_sync", "gather", "geometry", "flush", "total")
TILE_POINTS = 128


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def smi(query):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def cta_steps(cfg, rays):
    """Weight steps all CTAs of one fused render of `rays` rays run: two CTAs per 128-point tile, NS x (lin_in +
    blocks 0-2) + blocks 3-4 per tile, for the coarse and the fine pass."""
    per_tile = cfg["NS"] * (4 + 3 * 64) + 2 * 64
    kc, kf = cfg["n_coarse"], cfg["n_fine"]
    tiles = -(-rays * kc // TILE_POINTS) + (-(-rays * (kc + kf) // TILE_POINTS) if kf > 0 else 0)
    return 2 * tiles * per_tile


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "pixel-nerf_b200", "lib", "libpnr_sm90_prof.so"))
    ap.add_argument("--workloads", default="c2,c3,c4")
    ap.add_argument("--engines", default="tc,tc_fast")
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--frames-c4", type=int, default=1)
    ap.add_argument("--dump", default=None, help="directory for seeded rgb / depth of every (workload, engine)")
    args = ap.parse_args()
    os.environ["PNR_LIB"] = os.path.abspath(args.lib)    # read when pnr_native is first imported
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tc_phase_profile.py needs a CUDA device")
    bench = _load("pnr_bench", os.path.join(ROOT, "bench.py"))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = smi("name,power.limit,clocks.max.sm")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)    # > 50 MB L2, as bench.py
    for wl in args.workloads.split(","):
        cfg = bench.synth.CONFIGS[wl]
        frame = bench.WORKLOADS[wl]["frame_rays"]
        net, renderer = bench.build_scene(cfg, dev, "tc")
        import pnr_native as pn
        rays = bench.synth.make_rays(cfg, frame, n_target=max(8, frame // (cfg["W"] * cfg["H"]) + 1))[None].to(dev)
        render = renderer.bind_parallel(net, [0], simple_output=True).eval()
        frames = args.frames_c4 if wl == "c4" else args.frames

        def step():
            flush.zero_()
            with torch.no_grad():
                return render(rays)

        for eng in args.engines.split(","):
            net.engine = eng
            step()
            torch.cuda.synchronize()
            pn.tc_counters()                       # clears them
            sampler = bench.ClockSampler(0)
            sampler.start()
            launches0 = pn.launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(frames):
                step()
            e1.record()
            torch.cuda.synchronize()
            cnt = pn.tc_counters()
            launches = pn.launch_count() - launches0
            sampler.stop_flag = True
            sampler.join()
            clk = sampler.summary()
            per = 2 * frames * cta_steps(cfg, frame)    # 2 counted threads per CTA, each through every step
            res = {"workload": wl, "engine": eng, "lib": os.path.basename(args.lib), "frames": frames,
                   "ms_per_frame": e0.elapsed_time(e1) / frames, "launches_per_frame": launches / frames,
                   "counters": dict(zip(PHASES, cnt)), "clocks_per_step": None, "card": card, "sm_mhz": clk.get("sm_mhz"),
                   "power_w": clk.get("power_w"), "power_limit_w": clk.get("power_limit_w"),
                   "clock_reasons": clk.get("reasons")}
            if cnt[-1] > 0:
                cps = {name: c / per for name, c in zip(PHASES, cnt)}
                cps["other"] = cps["total"] - sum(cps[n] for n in PHASES[:-1] if n != "refill")
                res["clocks_per_step"] = {k: round(v, 1) for k, v in cps.items()}
            print(json.dumps(res), flush=True)
            if args.dump:
                os.makedirs(args.dump, exist_ok=True)
                torch.manual_seed(11)
                rgb, depth = step()
                np.save(os.path.join(args.dump, f"{wl}_{eng}_rgb.npy"), rgb.float().cpu().numpy())
                np.save(os.path.join(args.dump, f"{wl}_{eng}_depth.npy"), depth.float().cpu().numpy())
        del net, renderer, render, rays
        torch.cuda.empty_cache()
    print(json.dumps({"card": card}), flush=True)


if __name__ == "__main__":
    main()
