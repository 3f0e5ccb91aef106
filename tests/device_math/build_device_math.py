"""Builds tests/device_math/_build/libdevicemath.so: tests/device_math/device_math.cu with the product's nvcc and
codegen flags (imported from taichi_mpm_b200.build, so the two cannot drift apart)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(HERE, "device_math.cu")
LIB = os.path.join(HERE, "_build", "libdevicemath.so")


def build(force=False):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from taichi_mpm_b200 import build as B
    deps = [SRC, os.path.join(ROOT, "taichi_mpm_b200", "csrc", "mpmb_math.cuh"), os.path.abspath(B.__file__), os.path.abspath(__file__)]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    env = dict(os.environ)
    env.pop("CC", None)   # as taichi_mpm_b200.build: nvcc takes the system g++
    env.pop("CXX", None)
    cmd = [B.nvcc_path()] + B.NVCC_FLAGS + ["-I" + os.path.join(ROOT, "taichi_mpm_b200", "csrc"), "-o", LIB, SRC]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc failed building " + os.path.basename(LIB))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
