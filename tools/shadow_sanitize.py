#!/usr/bin/env python
"""Run the CPU suite against an AddressSanitizer + UBSan build of the host shadow (tests/csrc/host_shadow.cu: the per-env / per-lane
device functions of csrc/*_core.cuh compiled for the host).  An out-of-bounds index, a misaligned vector access or signed overflow
in that text shows up here without a GPU; compute-sanitizer on the real kernels covers the thread mapping (profiles/sanitizer_*).

    python tools/shadow_sanitize.py [-k EXPR]          # writes profiles/shadow_sanitizers_<tag>.log (tag: --tag, default local; git-ignored)
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = "-Xcompiler -fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer -g"


def gcc_file(name):
    return subprocess.run(["gcc", f"-print-file-name={name}"], capture_output=True, text=True, check=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-k", default="shadow or cpu or host_stack")
    ap.add_argument("--tag", default="local")
    a = ap.parse_args()
    env = dict(os.environ, AGX_SHADOW_FLAGS=FLAGS)
    # build WITHOUT the preload (nvcc itself must not run under ASan)
    subprocess.run([sys.executable, "-c", "from tests import _shadow; _shadow.build(force=True)"], cwd=ROOT, env=env, check=True)
    env.update(LD_PRELOAD=gcc_file("libasan.so") + ":" + gcc_file("libubsan.so"), ASAN_OPTIONS="detect_leaks=0:halt_on_error=1",
               UBSAN_OPTIONS="print_stacktrace=1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/", "-q", "-s", "-m", "not gpu", "-k", a.k, "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True)
    out = r.stdout + r.stderr
    hits = [l for l in out.splitlines() if "runtime error" in l or "AddressSanitizer" in l]
    tail = [l for l in out.splitlines() if " passed" in l or " failed" in l]
    log = os.path.join(ROOT, "profiles", f"shadow_sanitizers_{a.tag}.log")
    with open(log, "w") as f:
        f.write(f"# python tools/shadow_sanitize.py -k '{a.k}'\n# shadow flags: {FLAGS}\n")
        f.write("\n".join(tail) + "\n")
        f.write(f"sanitizer reports: {len(hits)}\n" + "\n".join(hits[:200]) + ("\n" if hits else ""))
    print(open(log).read())
    # back to the plain shadow for the next normal test run
    subprocess.run([sys.executable, "-c", "from tests import _shadow; _shadow.build(force=True)"], cwd=ROOT,
                   env={k: v for k, v in os.environ.items() if k != "AGX_SHADOW_FLAGS"}, check=True)
    return 1 if (hits or r.returncode) else 0


if __name__ == "__main__":
    sys.exit(main())
