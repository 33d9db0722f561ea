"""The phase-profile library (lib/libpnr_sm90_prof.so, built by __graft_entry__.build) on the H100: at a C2 frame its
outputs are bit-equal to the production library's, and its phase counters are filled and consistent (every phase
non-zero, none above the kernel total).  Each library runs in its own process (PNR_LIB is read at import)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pixel-nerf_b200", "lib")


def _run(lib, dump):
    cmd = [sys.executable, os.path.join(ROOT, "scripts", "tc_phase_profile.py"), "--lib", lib, "--workloads", "c2",
           "--engines", "tc", "--frames", "1", "--dump", dump]
    res = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    return [json.loads(l) for l in res.stdout.splitlines() if l.startswith("{") and '"engine"' in l][0]


def test_profile_library_matches_production_and_fills_counters(tmp_path):
    prof_lib = os.path.join(LIB, "libpnr_sm90_prof.so")
    assert os.path.isfile(prof_lib), "build() makes lib/libpnr_sm90_prof.so (make -C pixel-nerf_b200/csrc prof)"
    prod = _run(os.path.join(LIB, "libpnr_sm90.so"), str(tmp_path / "prod"))
    prof = _run(prof_lib, str(tmp_path / "prof"))
    for f in ("c2_tc_rgb.npy", "c2_tc_depth.npy"):
        a, b = np.load(tmp_path / "prod" / f), np.load(tmp_path / "prof" / f)
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), f
    assert all(v == 0 for v in prod["counters"].values()), prod["counters"]
    cnt = prof["counters"]
    assert all(v > 0 for v in cnt.values()), cnt
    assert all(v <= cnt["total"] for v in cnt.values()), cnt
