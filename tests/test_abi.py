"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a (H100), loads, exports
every symbol include/aerial_gym_b200.h declares, and the ctypes structs match its layout.
No compute call is made (no GPU here)."""
import ctypes
import os
import subprocess

import pytest

from aerial_gym_simulator_b200 import _build, _lib


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _lib.load()


def test_library_loads_and_versions(lib):
    assert lib.agx_abi_version() == 1
    assert lib.agx_last_error() is not None


def test_exports_every_declared_symbol(lib):
    names = _lib.declared_symbols()
    assert "agx_hp1_position_task_step" in names and "agx_hp1_physics_step" in names
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/aerial_gym_b200.h but not exported"


def test_struct_layout_matches(lib):
    assert lib.agx_sizeof(0) == ctypes.sizeof(_lib.AgxHp1Config)
    assert lib.agx_sizeof(1) == ctypes.sizeof(_lib.AgxHp1Buffers)
    assert lib.agx_sizeof(2) == ctypes.sizeof(_lib.AgxHp1ResetDraws)


def test_built_for_sm90a_only():
    out = subprocess.run([_build.cuda_tool("cuobjdump"), "--list-elf", _build.LIB], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert all("sm_90a" in line for line in out.splitlines() if "sm_" in line)


def test_argument_validation_without_gpu(lib):
    """NULL / invalid arguments are rejected before any CUDA call."""
    assert lib.agx_hp1_physics_step(None, None, None) == -3
    assert b"NULL" in lib.agx_last_error()
    cfg, buf = _lib.AgxHp1Config(), _lib.AgxHp1Buffers()
    cfg.num_motors = 5
    assert lib.agx_hp1_physics_step(ctypes.byref(cfg), ctypes.byref(buf), None) == -1
    assert b"num_motors" in lib.agx_last_error()


def test_product_never_imports_oracle():
    """The product package must not reach into oracle/ (tier rule 3)."""
    root = os.path.dirname(_build.PKG)
    for dp, _, files in os.walk(_build.PKG):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, os.path.join(dp, f)
    assert os.path.isdir(os.path.join(root, "oracle"))


def _header_prototypes():
    import re
    hdr = os.path.join(os.path.dirname(_build.PKG), "include", "aerial_gym_b200.h")
    txt = re.sub(r"/\*.*?\*/", "", open(hdr).read(), flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(?:int|uint64_t|const char\*)\s+(agx_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt):
        params = [p.strip() for p in m.group(2).split(",")]
        protos[m.group(1)] = [] if params == ["void"] else params
    return protos


def test_ctypes_argtypes_match_the_header(lib):
    """Every prototype in include/aerial_gym_b200.h against the argtypes _lib.load() declared: same arity, and
    pointer / float / integer in the same positions (a miscounted c_void_p run would shift every later argument)."""
    protos = _header_prototypes()
    assert len(protos) >= 18
    for name, params in protos.items():
        fn = getattr(lib, name)
        if fn.argtypes is None:
            assert not params or name in ("agx_last_error", "agx_abi_version"), f"{name}: no argtypes declared in _lib.py"
            continue
        assert len(fn.argtypes) == len(params), f"{name}: header has {len(params)} parameters, _lib.py declares {len(fn.argtypes)}"
        for i, (p, t) in enumerate(zip(params, fn.argtypes)):
            if "*" in p:
                ok = t in (ctypes.c_void_p, ctypes.c_char_p) or hasattr(t, "_type_") and isinstance(t._type_, type)
            elif p.startswith("float"):
                ok = t is ctypes.c_float
            else:
                ok = t in (ctypes.c_int, ctypes.c_int32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int64)
                if "uint64_t" in p:
                    ok = t is ctypes.c_uint64
            assert ok, f"{name}: parameter {i} `{p}` declared as {t}"
