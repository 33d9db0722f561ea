"""Codegen guard for the single-pass tensor-engine kernel k_field_tc_fast (CPU only: needs nvcc, not a GPU).

The single-pass kernel is the exact kernel's body compiled with one wgmma per k-step instead of three.  It must keep
the exact kernel's register health (no C7512 serialisation, small spills outside the MMA loops, each step issued as
one commit group) and must really issue a third of the exact kernel's HGMMA.  The exact kernel must stay in the same
unit under its own name (tests/test_tc_codegen.py checks its codegen)."""
import os
import re
import subprocess

import pytest

from test_tc_codegen import CSRC, KERNEL as EXACT, NVCC, _sass_ops, _tool

FAST = "_ZN3pnr2tc15k_field_tc_fastENS0_6ParamsE"

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("tc_fast_codegen")
    cubin = str(out / "pnr_field_tc.cubin")
    cmd = [NVCC, "-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
           "-cubin", os.path.join(CSRC, "pnr_field_tc.cu"), "-o", cubin]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    sass = {k: subprocess.run([cuobjdump, "-sass", "-fun", k, cubin], capture_output=True, text=True,
                              check=True).stdout for k in (FAST, EXACT)}
    return {"ptxas": res.stderr + res.stdout, "sass": sass}


def _ptxas_block(log, kernel):
    lines = log.splitlines()
    start = next(i for i, l in enumerate(lines) if f"Compiling entry function '{kernel}'" in l)
    end = next((i for i in range(start + 1, len(lines)) if "Compiling entry function" in lines[i]), len(lines))
    return "\n".join(lines[start:end])


def test_exact_kernel_keeps_its_symbol(compiled):
    assert f"Compiling entry function '{EXACT}'" in compiled["ptxas"]
    assert f"Compiling entry function '{FAST}'" in compiled["ptxas"]


def test_no_wgmma_serialisation_warning(compiled):
    bad = [l for l in compiled["ptxas"].splitlines() if "C7512" in l and FAST in l]
    assert not bad, "\n".join(bad)


def test_spills_stay_small(compiled):
    block = _ptxas_block(compiled["ptxas"], FAST)
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
    assert m, block
    assert int(m.group(1)) <= 512 and int(m.group(2)) <= 768, block   # the exact kernel's bound


def test_a_third_of_the_exact_hgmma(compiled):
    count = lambda k: sum(op.startswith("HGMMA") for op, _ in _sass_ops(compiled["sass"][k]))
    fast, exact = count(FAST), count(EXACT)
    assert fast >= 64, fast          # 3-HGMMA lin_in steps and 4-HGMMA fc steps
    assert 3 * fast == exact, (fast, exact)


def test_steps_issue_back_to_back(compiled):
    """Each step's wgmma (3 for lin_in, 4 for an fc step) form one group from a WARPGROUP.ARRIVE to the HGMMA with
    the gsb0 flag, with no wait, barrier or local-memory access inside, as in the exact kernel."""
    ops = _sass_ops(compiled["sass"][FAST])
    hgmma = sum(op.startswith("HGMMA") for op, _ in ops)
    sync = sum(op.startswith(("WARPGROUP.ARRIVE", "WARPGROUP.DEPBAR")) for op, _ in ops)
    assert sync < hgmma, (sync, hgmma)   # serialised: one ARRIVE and one DEPBAR per HGMMA (2 x hgmma)
    groups, bad, cur = [], [], None
    for idx, (op, args) in enumerate(ops):
        if op.startswith("WARPGROUP.ARRIVE"):
            cur = {"hgmma": 0}
        elif op.startswith("HGMMA"):
            assert cur is not None, f"HGMMA without a preceding ARRIVE at op {idx}"
            cur["hgmma"] += 1
            if "gsb0" in args:
                groups.append(cur["hgmma"])
                cur = None
        elif cur is not None and (op.startswith(("LDL", "STL", "WARPGROUP.DEPBAR")) or op == "BAR.SYNC"):
            bad.append((idx, op, args))
    assert not bad, bad[:10]
    assert groups and min(groups) >= 3, groups
