"""Static guards on the machine code of the flagship step kernel, hp1_step_kernel<4, true, true, 241> (the chained position-task step
of base_quadrotor + lee_attitude_control; 241 = hp_spec_id(AGX_CTRL_ATTITUDE, USE_RPS | MOTOR_RK4 | DISCRETE_MIX | GYROSCOPIC)).

hp1.cu is compiled for sm_90a with _build.py's flags; no GPU is needed.
- No register spills: at __launch_bounds__(64, 8) the kernel has 128 registers, and a spill slot lives in local memory.  The stack
  frame that remains belongs to sincosf's large-argument reduction, a cold path; ptxas counts it as stack, not as spills.
- The chain handshake invalidates L1 at most twice per step and never once per poll.  On sm_90a every acquire becomes CCTL.IVALL,
  which invalidates the SM's whole L1, the stack lines of every warp on the SM included.  So the waits poll with relaxed loads and
  acquire once with a fence afterwards: once after the prologue's waits, once after the rare arrival wait."""
import os
import re
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aerial_gym_simulator_b200 import _build  # noqa: E402

FLAGSHIP = "hp1_step_kernelILi4ELb1ELb1ELi241E"


@pytest.fixture(scope="module")
def flagship():
    """(ptxas -v report of the flagship, its SASS instructions as (address, text))"""
    extra = dict(_build.UNITS)["hp1.cu"]
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "hp1.o")
        cmd = [_build._nvcc()] + _build.NVCC_FLAGS + extra + ["-Xptxas", "-v", "-c", os.path.join(_build.CSRC, "hp1.cu"), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        sass = subprocess.run([_build.cuda_tool("cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    reports = [b for b in re.split(r"ptxas info\s+: Compiling entry function ", r.stdout + r.stderr) if FLAGSHIP in b.split("\n")[0]]
    assert len(reports) == 1, "the flagship instantiation is not in hp1.cu's ptxas report"
    funcs = [f for f in re.split(r"\n\s*Function : ", sass) if FLAGSHIP in f.split("\n")[0]]
    assert len(funcs) == 1, "the flagship instantiation is not in hp1.o"
    ins = [(int(m.group(1), 16), m.group(2)) for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", funcs[0])]
    return reports[0], ins


def test_flagship_has_no_register_spills(flagship):
    report, _ = flagship
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    regs = re.search(r"Used (\d+) registers", report)
    assert m and regs, report
    assert (int(m.group(1)), int(m.group(2))) == (0, 0), f"spills in the flagship step kernel: {m.group(0)}"
    assert int(regs.group(1)) <= 128, f"{regs.group(1)} registers: 8 CTAs of 64 threads per SM no longer fit"


def test_flagship_invalidates_l1_at_most_twice_and_never_in_a_poll_loop(flagship):
    _, ins = flagship
    cctl = [a for a, t in ins if "CCTL.IVALL" in t]
    # a loop is the range from a backward branch's target to the branch; a poll loop is an innermost one (it contains no other loop).
    # The blocks after the last EXIT (out-of-line paths for a diverged warp) branch back into the body without forming a loop.
    last_exit = max(a for a, t in ins if re.search(r"\bEXIT\b", t))
    loops = []
    for a, t in ins:
        m = re.search(r"\bBRA\S*\s+(?:[^,]*,\s*)?(0x[0-9a-f]+)\s*$", t)
        if m and int(m.group(1), 16) <= a < last_exit:
            loops.append((int(m.group(1), 16), a))
    assert loops, "no loop found in the flagship's SASS: the parser no longer matches cuobjdump's output"
    innermost = [(lo, hi) for lo, hi in loops if not any((lo, hi) != (l2, h2) and lo <= l2 and h2 <= hi for l2, h2 in loops)]
    in_loop = [hex(a) for a in cctl if any(lo <= a <= hi for lo, hi in innermost)]
    assert not in_loop, f"CCTL.IVALL (whole-L1 invalidation) inside a poll loop at {in_loop}"
    assert len(cctl) <= 2, f"{len(cctl)} CCTL.IVALL in the flagship step kernel: the handshake acquires more than once per wait"
