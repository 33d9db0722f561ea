#!/usr/bin/env python
"""Device time of loss.backward() for a partly frozen network at the C2 train shape (SB = 4 objects, B = 128 rays, the
C2 model with d_hidden 512, one GPU, tensor engine): the full backward (everything trainable, rays and cameras too)
alternated in one process with each freeze pattern of tests/frozen_util.py, which runs the selective backward
(pnr_render_backward_sel).  Prints one JSON line per pattern with the median device ms over --rounds rounds, and the
card, power limit and SM clock it ran on.

    python scripts/bench_frozen.py [--rounds 15] [--warmup 3] [--deterministic]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import frozen_util as fu  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        out = torch.cuda.get_device_name(0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--deterministic", action="store_true", help="torch.use_deterministic_algorithms(True)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_frozen.py measures on a CUDA GPU; none is available")
    torch.use_deterministic_algorithms(a.deterministic)
    sc = fu.Scene("c2", torch.device("cuda:0"))
    patterns = dict(full=fu.FULL, **fu.PATTERNS)
    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))

    def timed(p):
        sc.step(p, None, "tc", ev)
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1])

    for _ in range(a.warmup):
        for p in patterns.values():
            timed(p)
    ms = {k: [] for k in patterns}
    for _ in range(a.rounds):
        for k, p in patterns.items():      # full, pattern 1, pattern 2, ...: every round measures every variant
            ms[k].append(timed(p))
    info = card()
    full = float(np.median(ms["full"]))
    for k, v in ms.items():
        med = float(np.median(v))
        print(json.dumps(dict(pattern=k, backward_ms=round(med, 2), spread_ms=round(float(np.ptp(v)), 2),
                              vs_full=round(med / full, 3), rounds=a.rounds, deterministic=a.deterministic,
                              shape="C2 SB=4 B=128", card=info)))


if __name__ == "__main__":
    main()
