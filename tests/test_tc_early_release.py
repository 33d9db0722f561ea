"""The tensor engine releases a weight step before it waits for the next one, read from the PTX of both kernels (CPU
only: needs nvcc, not a GPU).

Each step's wgmma are committed as one group and retired by the next step's acquire(): `wgmma.wait_group 0`, then the
release (the acq_rel add on the slot pair's count that may refill the slots with the step two ahead), and only then
the FULL wait for the next step.  So the copy of step s + 2 is in flight while the warpgroup waits for step s + 1.
Retiring a step with `wait_group 1` after the next commit would release it only once the next step had landed."""
import os
import re
import subprocess

import pytest

from test_tc_codegen import CSRC, KERNEL as EXACT, NVCC
from test_tc_fast_codegen import FAST

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")

EVENTS = {
    "wgmma.commit_group": "C",
    "wgmma.wait_group.sync.aligned 0": "W",
    "atom.acq_rel.cta.shared::cta.add": "A",
    "mbarrier.try_wait": "T",
}


@pytest.fixture(scope="module")
def ptx(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("tc_early_release") / "pnr_field_tc.ptx")
    cmd = [NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-ptx",
           os.path.join(CSRC, "pnr_field_tc.cu"), "-o", out]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    text = open(out).read()
    bodies = {}
    for k in (EXACT, FAST):
        start = text.index(f".entry {k}(")
        end = text.find(".entry ", start + 1)
        bodies[k] = text[start:] if end < 0 else text[start:end]
    return bodies


def _events(body):
    pat = "|".join(re.escape(e) for e in EVENTS)
    return "".join(EVENTS[m.group(0)] for m in re.finditer(pat, body))


@pytest.mark.parametrize("kernel", [EXACT, FAST])
def test_no_step_is_retired_one_behind(ptx, kernel):
    waits = re.findall(r"wgmma\.wait_group\.sync\.aligned\s+(\d+)", ptx[kernel])
    assert waits and set(waits) == {"0"}, sorted(set(waits))


@pytest.mark.parametrize("kernel", [EXACT, FAST])
def test_every_commit_is_retired_and_released_before_the_next_full_wait(ptx, kernel):
    ev = _events(ptx[kernel])
    assert ev.count("C") > 0, ev   # one commit group per step
    # after each commit: wait_group 0, the release, and only then (if at all) another FULL wait
    bad = [m.start() for m in re.finditer(r"C(?!WA)", ev)]
    assert not bad, (bad, ev)
    # the retire waits are at least one per step site, on top of the drains that end the MMA runs
    assert ev.count("W") > ev.count("C"), ev
