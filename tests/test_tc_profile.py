"""The phase-profile build of the tensor engine (-DPNR_TC_PROFILE, lib/libpnr_sm90_prof.so) against the production
build (CPU only: needs nvcc, not a GPU).  The profile hooks read clock64() around every ring wait, wgmma wait, barrier
and phase; the production kernels must not carry them.  The only clock reads a production kernel has are the two of
the fine pass's `ready` poll timeout (t0 and the check inside the back-off loop)."""
import os
import re
import subprocess

import pytest

from test_tc_codegen import CSRC, KERNEL as EXACT, NVCC, _tool
from test_tc_fast_codegen import FAST

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def _clock_reads(sass):
    return len(re.findall(r"\bS2U?R\b.*SR_CLOCK|\bCS2R\b.*SR_CLOCK", sass))


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    out = tmp_path_factory.mktemp("tc_profile")
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    procs, res = {}, {}
    for name, extra in (("prod", []), ("prof", ["-DPNR_TC_PROFILE"])):
        cubin = str(out / f"{name}.cubin")
        cmd = [NVCC, "-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", *extra, "-cubin",
               os.path.join(CSRC, "pnr_field_tc.cu"), "-o", cubin]
        procs[name] = (cubin, subprocess.Popen(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                                               text=True))
    for name, (cubin, p) in procs.items():
        _, err = p.communicate()
        assert p.returncode == 0, err[-4000:]
        res[name] = {k: subprocess.run([cuobjdump, "-sass", "-fun", k, cubin], capture_output=True, text=True,
                                       check=True).stdout for k in (EXACT, FAST)}
    return res


@pytest.mark.parametrize("kernel", [EXACT, FAST])
def test_production_kernel_has_no_profile_clock_reads(sass, kernel):
    assert "HGMMA" in sass["prod"][kernel]
    assert _clock_reads(sass["prod"][kernel]) <= 4, _clock_reads(sass["prod"][kernel])


@pytest.mark.parametrize("kernel", [EXACT, FAST])
def test_profile_kernel_reads_the_clock_in_every_phase(sass, kernel):
    # per-step hooks (FULL, EMPTY, wgmma_wait) are inlined at every step of every MMA run: hundreds of reads
    assert _clock_reads(sass["prof"][kernel]) >= 100, _clock_reads(sass["prof"][kernel])
