"""The tensor engine's producer warpgroup, read from the compiled PTX and SASS of both kernels (CPU only: needs nvcc,
not a GPU).

Each kernel runs 384 threads: two consumer warpgroups that issue the wgmma and one producer warpgroup whose lanes refill
the weight rings.  setmaxnreg moves registers from the producer to the consumers, so the consumers keep the 160
accumulator registers of a step in registers although the launch grants 65536 / 384 per thread.  The budgets must fit
the register file, and the producer's code, everything the thread can reach after its setmaxnreg.dec, must not issue
wgmma or join the consumers' named barrier (tests/test_tc_refill.py: it does not wait on an mbarrier either)."""
import os
import re
import subprocess

import pytest

from test_tc_codegen import CSRC, KERNEL as EXACT, NVCC, _tool
from test_tc_fast_codegen import FAST

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")

KERNELS = [EXACT, FAST]


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("tc_producer")
    src = os.path.join(CSRC, "pnr_field_tc.cu")
    arch = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a"]
    ptx, cubin = str(out / "pnr_field_tc.ptx"), str(out / "pnr_field_tc.cubin")
    for flag, dst in (("-ptx", ptx), ("-cubin", cubin)):
        res = subprocess.run([NVCC, *arch, flag, src, "-o", dst], cwd=CSRC, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-4000:]
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    text = open(ptx).read()
    res = {}
    for k in KERNELS:
        start = text.index(f".entry {k}(")
        end = text.find(".entry ", start + 1)
        sass = subprocess.run([cuobjdump, "-sass", "-fun", k, cubin], capture_output=True, text=True, check=True).stdout
        res[k] = {"ptx": text[start:] if end < 0 else text[start:end], "sass": sass}
    return res


def _budgets(ptx):
    dec = re.findall(r"setmaxnreg\.dec\.sync\.aligned\.u32\s+(\d+)", ptx)
    inc = re.findall(r"setmaxnreg\.inc\.sync\.aligned\.u32\s+(\d+)", ptx)
    return dec, inc


@pytest.mark.parametrize("kernel", KERNELS)
def test_three_warpgroups(compiled, kernel):
    m = re.search(r"\.maxntid\s+(\d+)", compiled[kernel]["ptx"])
    assert m and int(m.group(1)) == 384, m and m.group(0)


@pytest.mark.parametrize("kernel", KERNELS)
def test_register_budgets_fit_the_register_file(compiled, kernel):
    dec, inc = _budgets(compiled[kernel]["ptx"])
    assert len(set(dec)) == 1 and len(set(inc)) == 1, (dec, inc)
    producer, consumer = int(dec[0]), int(inc[0])
    assert producer < 168 < consumer, (producer, consumer)
    assert 128 * producer + 256 * consumer <= 65536, (producer, consumer)
    # ptxas kept both: the SASS moves the warpgroups to the same budgets
    sass = compiled[kernel]["sass"]
    assert re.search(rf"USETMAXREG\.DEALLOC\S*\s+{hex(producer)}\b", sass), "producer budget missing from the SASS"
    assert re.search(rf"USETMAXREG\.TRY_ALLOC\S*\s+(?:\w+,\s*)?{hex(consumer)}\b", sass), "consumer budget missing"


def _instructions(sass):
    """(address, predicate, opcode, operands) of every SASS instruction."""
    out = []
    for line in sass.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);", line)
        if m:
            out.append((int(m.group(1), 16), m.group(2), m.group(3), m.group(4)))
    return out


def _reachable_from(ins, start):
    """Indices of the instructions a thread can execute from ins[start] on: branches, calls and fall-through, up to
    an unconditional EXIT or a RET (the fall-through of every call site is followed as well)."""
    index = {addr: i for i, (addr, _, _, _) in enumerate(ins)}
    seen, todo = set(), [start]
    while todo:
        i = todo.pop()
        if i in seen or i >= len(ins):
            continue
        seen.add(i)
        _, pred, op, args = ins[i]
        assert not op.startswith(("BRX", "JMX", "JMP")), f"indirect branch at {ins[i]}"
        if op.startswith(("BRA", "CALL")):
            target = re.search(r"0x([0-9a-f]+)", args)
            assert target and int(target.group(1), 16) in index, ins[i]
            todo.append(index[int(target.group(1), 16)])
            if op.startswith("BRA") and pred is None and ".ANY" not in op:
                continue
        elif op.startswith(("EXIT", "RET")) and pred is None:
            continue
        todo.append(i + 1)
    return seen


@pytest.mark.parametrize("kernel", KERNELS)
def test_producer_issues_no_wgmma_and_never_waits_with_the_consumers(compiled, kernel):
    ins = _instructions(compiled[kernel]["sass"])
    starts = [i for i, (_, _, op, _) in enumerate(ins) if op.startswith("USETMAXREG.DEALLOC")]
    assert len(starts) == 1, starts
    ops = [ins[i][2] for i in _reachable_from(ins, starts[0])]
    assert any(op.startswith("UBLKCP") for op in ops), "the producer issues the ring's bulk copies"
    forbidden = [op for op in ops if op.startswith(("HGMMA", "WARPGROUP", "BAR.", "USETMAXREG.TRY"))]
    assert not forbidden, sorted(set(forbidden))
    # and the consumers' code is where the wgmma are
    assert sum(op.startswith("HGMMA") for _, _, op, _ in ins) > 0
