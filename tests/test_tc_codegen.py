"""Codegen guard for the fused tensor-engine kernel (CPU only: needs nvcc, not a GPU).

k_field_tc keeps 160 fp32 accumulators per thread in registers (the residual stream X and the hidden chunk H_c).  If a
later edit leaves ptxas short of registers, it silently serialises the wgmma: every HGMMA gets its own
WARPGROUP.ARRIVE / WARPGROUP.DEPBAR pair, the tensor pipe holds one m64n64k16 per warpgroup, and the kernel runs
several times slower with the same results.  These tests compile pnr_field_tc.cu with the Makefile's flags and check
that this has not happened."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pixel-nerf_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
KERNEL = "_ZN3pnr2tc10k_field_tcENS0_6ParamsE"

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def _tool(name):
    path = os.path.join(os.path.dirname(NVCC), name)
    return path if os.path.exists(path) else shutil.which(name)


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("tc_codegen")
    cubin = str(out / "pnr_field_tc.cubin")
    cmd = [NVCC, "-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
           "-cubin", os.path.join(CSRC, "pnr_field_tc.cu"), "-o", cubin]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", "-fun", KERNEL, cubin], capture_output=True, text=True, check=True)
    return {"ptxas": res.stderr + res.stdout, "sass": sass.stdout}


def _kernel_ptxas_block(log):
    # ptxas prints "Compiling entry function '<name>'", the function's properties, then the next function
    lines = log.splitlines()
    start = next(i for i, l in enumerate(lines) if f"Compiling entry function '{KERNEL}'" in l)
    end = next((i for i in range(start + 1, len(lines)) if "Compiling entry function" in lines[i]), len(lines))
    return "\n".join(lines[start:end])


def test_no_wgmma_serialisation_warning(compiled):
    bad = [l for l in compiled["ptxas"].splitlines() if "C7512" in l and KERNEL in l]
    assert not bad, "\n".join(bad)


def test_spills_stay_small(compiled):
    block = _kernel_ptxas_block(compiled["ptxas"])
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
    assert m, block
    stores, loads = int(m.group(1)), int(m.group(2))
    # today 164 / 228 (geometry and ray finishing, outside the MMA loops); a register shortage costs kilobytes
    assert stores <= 512 and loads <= 768, block


def _sass_ops(sass):
    ops = []
    for line in sass.splitlines():
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)(.*?);", line)
        if m:
            ops.append((m.group(1), m.group(2)))
    return ops


def test_wgmma_issued_in_groups(compiled):
    ops = _sass_ops(compiled["sass"])
    hgmma = sum(op.startswith("HGMMA") for op, _ in ops)
    sync = sum(op.startswith(("WARPGROUP.ARRIVE", "WARPGROUP.DEPBAR")) for op, _ in ops)
    assert hgmma >= 200, hgmma   # 9-HGMMA lin_in steps and 12-HGMMA fc steps
    # serialised: one ARRIVE and one DEPBAR per HGMMA (432 for 216); grouped: one pair per step of 9-12 HGMMA
    assert sync * 4 < hgmma, (sync, hgmma)


def test_steps_issue_back_to_back(compiled):
    """A step's wgmma (one commit group: 9 HGMMA for lin_in, 12 for an fc step) form one group in SASS, from a
    WARPGROUP.ARRIVE to the HGMMA that carries the gsb0 (group-complete) flag, with no wait and no local-memory access
    inside.  A serialised kernel closes a group after every HGMMA."""
    ops = _sass_ops(compiled["sass"])
    groups, bad = [], []
    cur = None
    for idx, (op, args) in enumerate(ops):
        if op.startswith("WARPGROUP.ARRIVE"):
            cur = {"start": idx, "hgmma": 0}
        elif op.startswith("HGMMA"):
            assert cur is not None, f"HGMMA without a preceding ARRIVE at op {idx}"
            cur["hgmma"] += 1
            if "gsb0" in args:
                groups.append(cur["hgmma"])
                cur = None
        elif cur is not None and (op.startswith(("LDL", "STL", "WARPGROUP.DEPBAR")) or op == "BAR.SYNC"):
            bad.append((idx, op, args))
    assert not bad, bad[:10]
    assert groups and min(groups) >= 9, groups
