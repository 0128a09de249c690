"""Build a VARIANT of libaerial_gym_b200.so (never shipped; A/B experiments on a GPU box through AGX_LIB_PATH):

    python tools/build_variant.py <name> [--hp1 "<extra nvcc flags for hp1.cu>"] [--hp2 "<... for hp2_raycast.cu>"] [-v]
    AGX_LIB_PATH=tools/dbg/libagx_<name>.so python bench.py --steps 200

All translation units of aerial_gym_simulator_b200/_build.py are compiled (same flags), so the variant exports the full ABI.
Round-2 candidates for the latency / instruction-fetch bound HP1 step (DESIGN 11; numerically identical to the default build --
the CPU shadow tests run the same text with the same macro: AGX_SHADOW_FLAGS="-DAGX_HP1_ROLL_MOTORS" python -m pytest tests -m "not gpu"):
    --hp1 "-DAGX_HP1_ROLL_MOTORS"     motor / allocation loops rolled (#pragma unroll 1): ~4x less straight-line code to fetch
    --hp1 "-DAGX_HP1_NOINLINE_TRIG"   one shared copy of sincosf instead of seven inlined ones
    --hp1 "-maxrregcount=96"          (or __launch_bounds__ experiments)"""
import os
import shlex
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aerial_gym_simulator_b200 import _build  # noqa: E402


def main(argv):
    name = argv[0]
    extra = {"hp1.cu": [], "hp2_raycast.cu": []}
    verbose = "-v" in argv
    for flag, unit in (("--hp1", "hp1.cu"), ("--hp2", "hp2_raycast.cu")):
        if flag in argv:
            extra[unit] = shlex.split(argv[argv.index(flag) + 1])
    out_dir = os.path.join(ROOT, "tools", "dbg", f"build_{name}")
    os.makedirs(out_dir, exist_ok=True)
    objs = []
    for unit, flags in _build.UNITS:
        obj = os.path.join(out_dir, unit.replace(".cu", ".o"))
        cmd = [_build._nvcc()] + _build.NVCC_FLAGS + flags + extra.get(unit, []) + (["-Xptxas", "-v"] if verbose else []) + \
              ["-c", os.path.join(_build.CSRC, unit), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            sys.stderr.write(r.stdout + r.stderr)
            raise SystemExit(f"nvcc failed for {unit}")
        if verbose and unit in extra and extra[unit]:
            for line in (r.stdout + r.stderr).splitlines():
                if "Used" in line or "spill" in line:
                    print(unit, line.strip())
        objs.append(obj)
    lib = os.path.join(ROOT, "tools", "dbg", f"libagx_{name}.so")
    subprocess.run([_build._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", lib] + objs, check=True)
    print("built", lib)


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    main(sys.argv[1:])
