"""Machine code of articulated.cu (CUDA 12.9, _build.NVCC_FLAGS, sm_90a), no GPU needed: every kernel is free of spills, keeps its
registers and stack frame, and keeps its SASS bit for bit.  The unit is compiled once for the module."""
import hashlib
import os
import re
import subprocess
import tempfile

import pytest

from aerial_gym_simulator_b200 import _build

# kernel (a substring of its mangled name) -> (registers per thread, stack frame in bytes, md5 of the normalised SASS).  The stack
# frame of the step kernels is the per-body arrays of the ABA, in local memory by design (articulated.cu): 3,312 B at NB = 9, 5,856 B
# at NB = 16.  The body-state kernel builds its rows in shared memory and has none.
KERNELS = {
    "articulated_body_state_kernelILi16E": (62, 0, "49fabc56648bbeedb676825c9dfce8b7"),
    "articulated_body_state_kernelILi9E": (62, 0, "d6ab5ca7ca0215f6f63b3496123fa2d8"),
    "articulated_step_effort_kernelILi4ELi16ELb0E": (158, 5856, "09c0d3e7332544ce33a23224720c7ea1"),
    "articulated_step_effort_kernelILi4ELi16ELb1E": (158, 5856, "9579cc186f99b4fd0882a770a5f271e5"),
    "articulated_step_effort_kernelILi4ELi9ELb0E": (158, 3312, "abd31654971564ffba13ba49beb4fec6"),
    "articulated_step_effort_kernelILi4ELi9ELb1E": (158, 3312, "f6b6f80c1bcce608057bcdea4b8ec6cb"),
    "articulated_step_effort_kernelILi8ELi16ELb0E": (167, 5856, "3460f725d21829e0b968c1d33a994119"),
    "articulated_step_effort_kernelILi8ELi16ELb1E": (167, 5856, "1574c81ff97a7ac7fc0231afe3a3f2a2"),
    "articulated_step_effort_kernelILi8ELi9ELb0E": (167, 3312, "c3c8b9d43a5e98e00d872969082d91ee"),
    "articulated_step_effort_kernelILi8ELi9ELb1E": (167, 3312, "a32e11ab74110bf4d33d9e436db96c31"),
    "articulated_step_imu_kernelILi4ELi16E": (158, 5856, "126c2d9df2119902e827c3866d83e9fb"),
    "articulated_step_imu_kernelILi4ELi9E": (158, 3312, "2b321c922eed32aa91bc91d3594f5433"),
    "articulated_step_imu_kernelILi8ELi16E": (166, 5856, "f4eb229df3dcb4a243ca0d7daecea392"),
    "articulated_step_imu_kernelILi8ELi9E": (166, 3312, "8418465ed540f9c3753c25a8ffefbfff"),
    "articulated_step_joint_force_kernelILi4ELi16E": (165, 5856, "af65bddf37f1db054b1e694fba9562d9"),
    "articulated_step_joint_force_kernelILi4ELi9E": (165, 3312, "1a7e9a4c0a120dfb00aab10ea025e6f1"),
    "articulated_step_joint_force_kernelILi8ELi16E": (168, 5856, "567db4425f577673774188977c700cdf"),
    "articulated_step_joint_force_kernelILi8ELi9E": (168, 3312, "7ff9f015576a0cc3d10fea1495b172a4"),
    "articulated_step_kernelILi4ELi16E": (160, 5856, "61f12510a9b31d109fae04dc1a814d87"),
    "articulated_step_kernelILi4ELi9E": (160, 3312, "efbd4a3c22e2ad0447001440b6c8ac27"),
    "articulated_step_kernelILi8ELi16E": (167, 5856, "4d833f5c266d542fe19e29d2b82ef233"),
    "articulated_step_kernelILi8ELi9E": (167, 3312, "c2086c00bb11078baa2a0b9cc19015ce"),
}


@pytest.fixture(scope="module")
def articulated_unit():
    """(-Xptxas -v report, cuobjdump -sass listing) of articulated.cu"""
    src = os.path.join(_build.CSRC, "articulated.cu")
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "articulated.o")
        r = subprocess.run([_build._nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        sass = subprocess.run([_build.cuda_tool("cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def sass_functions(txt):
    """md5 of each function's SASS, normalised: comment lines and addresses dropped, encodings kept, the anonymous namespace's
    per-file hash masked"""
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__\w+?_cu_\w{8}", "ANON", m.group(1))
            out[cur] = []
            continue
        s = line.strip()
        if cur is None or not s or s.startswith(("//", "...", ".")):
            continue
        out[cur].append(re.sub(r"/\*[0-9a-f]{4,}\*/", "", s))
    return {k: hashlib.md5("\n".join(v).encode()).hexdigest() for k, v in out.items()}


def _reports(log):
    """mangled kernel name -> (stack frame bytes, spill text, registers), from the -Xptxas -v report"""
    blocks = re.findall(r"Compiling entry function '(\S+)'.*?\n.*?(\d+) bytes stack frame, (.*?spill loads)\n.*?Used (\d+) registers", log,
                        re.S)
    return {f: (int(stack), info, int(regs)) for f, stack, info, regs in blocks}


def _family(kernel):
    """the KERNELS keys of one kernel template"""
    keys = [k for k in KERNELS if k.startswith(kernel + "I")]
    assert keys, kernel
    return keys


def _check_resources(unit, kernel):
    """every instantiation of the template: its registers and stack frame, and no spills"""
    reports = _reports(unit[0])
    for key in _family(kernel):
        regs, stack, _ = KERNELS[key]
        found = [v for f, v in reports.items() if key in f]
        assert found == [(stack, "0 bytes spill stores, 0 bytes spill loads", regs)], (key, found)


def _check_sass(unit, kernel):
    """every instantiation of the template: its normalised SASS"""
    h = sass_functions(unit[1])
    for key in _family(kernel):
        hits = [v for k, v in h.items() if key in k]
        assert hits == [KERNELS[key][2]], (key, hits)


def test_every_kernel_is_pinned(articulated_unit):
    """the unit's kernels are those of KERNELS, each name holding exactly one key"""
    names = list(_reports(articulated_unit[0]))
    assert sorted(k for f in names for k in KERNELS if k in f) == sorted(KERNELS) and len(names) == len(KERNELS), names


def test_step_kernels_have_no_spills(articulated_unit):
    _check_resources(articulated_unit, "articulated_step_kernel")


def test_body_state_kernels_have_no_spills_and_no_stack(articulated_unit):
    _check_resources(articulated_unit, "articulated_body_state_kernel")


def test_imu_kernels_have_no_spills(articulated_unit):
    _check_resources(articulated_unit, "articulated_step_imu_kernel")


def test_effort_kernels_have_no_spills(articulated_unit):
    _check_resources(articulated_unit, "articulated_step_effort_kernel")


def test_joint_force_kernels_have_no_spills(articulated_unit):
    _check_resources(articulated_unit, "articulated_step_joint_force_kernel")


def test_step_kernels_keep_their_sass(articulated_unit):
    _check_sass(articulated_unit, "articulated_step_kernel")


def test_body_state_kernels_keep_their_sass(articulated_unit):
    _check_sass(articulated_unit, "articulated_body_state_kernel")


def test_imu_kernels_keep_their_sass(articulated_unit):
    _check_sass(articulated_unit, "articulated_step_imu_kernel")


def test_effort_kernels_keep_their_sass(articulated_unit):
    _check_sass(articulated_unit, "articulated_step_effort_kernel")


def test_joint_force_kernels_keep_their_sass(articulated_unit):
    _check_sass(articulated_unit, "articulated_step_joint_force_kernel")
