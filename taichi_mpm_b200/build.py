"""In-tree build of libmpmb.so (hand-written sm_90a CUDA for the H100 + the C-ABI of include/mpmb.h).

nvcc cross-compiles without a GPU; the built .so is git-ignored.
"""
import os
import subprocess
import sys

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
SRC = [os.path.join(_PKG, "csrc", "mpmb_engine.cu")]
# this file is a dependency too: a change of NVCC_FLAGS (e.g. the target architecture) rebuilds the library
DEPS = SRC + [os.path.join(_PKG, "csrc", "mpmb_math.cuh"), os.path.join(_PKG, "csrc", "mpmb_math2d.cuh"), os.path.join(_ROOT, "include", "mpmb.h"), os.path.abspath(__file__)]
LIB = os.path.join(_PKG, "lib", "libmpmb.so")
# the bounds-checked variant (-DMPMB_CHECKED): an index that would leave its array is recorded and skipped
CHECKED_LIB = os.path.join(_PKG, "lib", "libmpmb_checked.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-shared",
]


def nvcc_path():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if p and (os.path.isabs(p) and os.path.exists(p) or not os.path.isabs(p)):
            return p
    return "nvcc"


def needs_build(lib=None):
    lib = lib or LIB
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False, defines=(), out=None):
    """Compile libmpmb.so for sm_90a if it is missing or stale.  Returns the path.

    `defines` / `out` build an A/B variant next to the product (e.g. defines=["MPMB_EXP_TILE_XYZ"],
    out=".../lib/libmpmb_tile_xyz.so"; load it with MPMB_LIB=<path>); the default library is only
    ever built without defines."""
    lib = out or LIB
    if not force and not needs_build(lib):   # a variant's file name encodes its defines
        return lib
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    cmd = [nvcc_path()] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", lib] + SRC
    env = dict(os.environ)
    # this image exports CC/CXX pointing at a wrapper without OpenMP specs; nvcc should use the system g++
    env.pop("CC", None)
    env.pop("CXX", None)
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc failed building " + os.path.basename(lib))
    if verbose:
        sys.stderr.write(r.stdout)
    return lib


if __name__ == "__main__":
    # python -m taichi_mpm_b200.build [--force] [-v] [--define NAME ... --out PATH]
    argv = sys.argv[1:]
    defs = [argv[i + 1] for i, a in enumerate(argv) if a == "--define" and i + 1 < len(argv)]
    outp = next((argv[i + 1] for i, a in enumerate(argv) if a == "--out" and i + 1 < len(argv)), None)
    if defs and not outp:
        outp = os.path.join(_PKG, "lib", "libmpmb_" + "_".join(d.lower().replace("mpmb_exp_", "") for d in defs) + ".so")
    print(build(force="--force" in argv, verbose="-v" in argv, defines=defs, out=outp))
