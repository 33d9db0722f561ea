"""The tensor engine's weight-ring refill, read from the PTX of both kernels (CPU only: needs
nvcc, not a GPU).

The last of a warpgroup's 4 warps to release a step refills the ring (an acq_rel atomic add on a release count in
shared memory), so no thread waits on a barrier to refill: the only mbarrier waits left are the FULL waits of each
step (two slots per step in the exact kernel, the W_hi slot in the single-pass one), and the only arrivals are the
transaction arrivals that arm a FULL barrier for a bulk copy."""
import os
import re
import subprocess

import pytest

from test_tc_codegen import CSRC, KERNEL as EXACT, NVCC
from test_tc_fast_codegen import FAST

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def ptx(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("tc_refill") / "pnr_field_tc.ptx")
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


@pytest.mark.parametrize("kernel", [EXACT, FAST])
def test_refill_is_triggered_by_an_atomic_release_count(ptx, kernel):
    assert "atom.acq_rel.cta.shared::cta.add.u32" in ptx[kernel]


@pytest.mark.parametrize("kernel", [EXACT, FAST])
def test_only_transaction_arrivals(ptx, kernel):
    arrivals = re.findall(r"mbarrier\.arrive[\w:.]*", ptx[kernel])
    assert arrivals, "the FULL barriers are armed with mbarrier.arrive.expect_tx"
    assert all(".expect_tx" in a for a in arrivals), sorted(set(arrivals))


def test_only_full_waits_remain(ptx):
    # each acquire waits on the step's two slots (exact) or its W_hi slot (single pass); a wait on the refill path
    # would add the same number of waits to both kernels
    waits = {k: len(re.findall(r"mbarrier\.try_wait", ptx[k])) for k in (EXACT, FAST)}
    assert waits[FAST] > 0 and waits[EXACT] == 2 * waits[FAST], waits

