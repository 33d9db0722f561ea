"""A/B timing of two builds of the CUDA library on the flagship benchmark.

Runs `bench.py --no-cpu-baseline` once per (workload, round, library) with PNR_LIB pointing at each library in turn,
alternating A, B, A, B, ... so that both see the same drift of clocks, temperature and neighbours on the card.  For
each workload (C2, then C3 and C4) it prints one JSON line: per library the median and spread of `value` (rays/s), of
`roofline.kernel_ms_per_step` and of `roofline.executed_fp16_mma_tflops`, the clocks and board power bench.py sampled,
and whether the `--dump-outputs` of every run is bit-identical to the first run of library A.  The first round of C2
also keeps bench.py's parity block (CUDA vs the CPU oracle); later runs skip it.  A final line names the card and its
power limit.

    python scripts/bench_tc_ab.py --a old/libpnr_sm90.so --b pixel-nerf_b200/lib/libpnr_sm90.so --out ab_out
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def run_bench(lib, workload, steps, warmup, dump_dir, parity):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu-baseline", "--workload", workload,
           "--steps", str(steps), "--warmup", str(warmup), "--dump-outputs", dump_dir]
    if not parity:
        cmd.append("--no-parity")
    env = dict(os.environ, PNR_LIB=os.path.abspath(lib))
    res = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [l for l in res.stdout.splitlines() if l.startswith("{")]
    if res.returncode != 0 or not lines:
        sys.stderr.write(res.stdout[-3000:] + res.stderr[-3000:])
        raise SystemExit(f"bench.py failed for {lib} ({workload}), exit code {res.returncode}")
    return json.loads(lines[-1])


def same_outputs(d0, d1):
    names = sorted(f for f in os.listdir(d0) if f.endswith(".npy"))
    if names != sorted(f for f in os.listdir(d1) if f.endswith(".npy")):
        return False
    for f in names:
        a, b = np.load(os.path.join(d0, f)), np.load(os.path.join(d1, f))
        if a.shape != b.shape or a.dtype != b.dtype or a.tobytes() != b.tobytes():
            return False
    return True


def stats(xs):
    xs = [x for x in xs if x is not None]
    if not xs:
        return None
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs),
            "spread": (max(xs) - min(xs)) / statistics.median(xs), "runs": xs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True, help="library A (the baseline)")
    ap.add_argument("--b", required=True, help="library B (the candidate)")
    ap.add_argument("--out", required=True, help="directory for the dumped outputs")
    ap.add_argument("--workloads", default="c2,c3,c4")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--steps-c4", type=int, default=3, help="timed steps of C4 (one C4 frame renders 120 000 rays)")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    libs = {"A": args.a, "B": args.b}
    for name, lib in libs.items():
        if not os.path.isfile(lib):
            raise SystemExit(f"library {name} not found: {lib}")
    print(json.dumps({"card": card(), "A": os.path.abspath(args.a), "B": os.path.abspath(args.b)}), flush=True)
    for wl in args.workloads.split(","):
        steps = args.steps_c4 if wl == "c4" else args.steps
        runs = {"A": [], "B": []}
        ref_dump = None
        identical = True
        for rnd in range(args.rounds):
            for name in ("A", "B"):
                dump = os.path.join(os.path.abspath(args.out), f"{wl}_{name}{rnd}")
                line = run_bench(libs[name], wl, steps, args.warmup, dump, parity=(wl == "c2" and rnd == 0))
                runs[name].append(line)
                if ref_dump is None:
                    ref_dump = dump
                else:
                    identical = identical and same_outputs(ref_dump, dump)
                rf = line.get("roofline", {})
                print(json.dumps({"workload": wl, "round": rnd, "lib": name, "value": line["value"],
                                  "kernel_ms_per_step": rf.get("kernel_ms_per_step"),
                                  "executed_fp16_mma_tflops": rf.get("executed_fp16_mma_tflops"),
                                  "gpu_launches": line.get("gpu_launches"), "clocks": line.get("clocks")}), flush=True)
        summary = {"workload": wl, "steps": steps, "rounds": args.rounds, "outputs_bit_identical": identical}
        for name in ("A", "B"):
            ls = runs[name]
            summary[name] = {
                "value": stats([l["value"] for l in ls]),
                "kernel_ms_per_step": stats([l["roofline"]["kernel_ms_per_step"] for l in ls]),
                "executed_fp16_mma_tflops": stats([l["roofline"].get("executed_fp16_mma_tflops") for l in ls]),
                "gpu_launches_per_step": sorted({l["gpu_launches"] / l["steps"] for l in ls}),
                "sm_mhz": stats([l["clocks"].get("sm_mhz") for l in ls]),
                "power_w": stats([l["clocks"].get("power_w") for l in ls]),
                "power_limit_w": ls[0]["clocks"].get("power_limit_w"),
                "clock_reasons": sorted({r for l in ls for r in l["clocks"].get("reasons", [])}),
                "parity": next((l["parity"] for l in ls if "parity" in l), None),
            }
        summary["speedup_median"] = summary["B"]["value"]["median"] / summary["A"]["value"]["median"]
        print(json.dumps(summary), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
