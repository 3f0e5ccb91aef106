"""Builds tests/simt/_build/libmpmb_simt.so: the engine's CUDA source compiled for the HOST on top of the SIMT
emulator (simt.h).  The product source is not modified; two kinds of sites are rewritten in a temporary copy:
  * kernel launches   name<<<grid, block, smem, stream>>>(args)  ->  SIMT_LAUNCH((name), grid, block, smem, stream)(args)
  * inline PTX        cp.async copies / commit / wait, the system-scope release store and acquire load; the mbarrier /
                      TMA bulk-copy helpers carry their own emulator twins behind `#ifndef MPMB_SIMT_HOST ... #else`
Everything else — kernels, device math, the C-ABI host code — is compiled as it stands, with <cuda_runtime.h> and
<cub/...> resolving to the emulator's headers."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(ROOT, "taichi_mpm_b200", "csrc", "mpmb_engine.cu")
MATH = os.path.join(ROOT, "taichi_mpm_b200", "csrc", "mpmb_math.cuh")
MATH2 = os.path.join(ROOT, "taichi_mpm_b200", "csrc", "mpmb_math2d.cuh")   # the 2-D material math, included by SRC
OUT_DIR = os.path.join(HERE, "_build")
LIB = os.path.join(OUT_DIR, "libmpmb_simt.so")

RULES = [
    (re.compile(r'\b([A-Za-z_]\w*(?:<[^<>;]*>)?)<<<(.*?)>>>\('), r'SIMT_LAUNCH((\1), \2)('),
    (re.compile(r'asm volatile\("cp\.async\.c[ag]\.shared\.global \[%0\], \[%1\], (\d+);\\n" ::"r"\((\w+)\), "l"\((.*)\)\);'), r'simt::cp_async(\2, \3, \1);'),
    (re.compile(r'asm volatile\("" ::: "memory"\);'), ';'),   # compiler-only barrier
    (re.compile(r'asm volatile\("cp\.async\.commit_group;\\n" ::\);'), ';'),
    (re.compile(r'asm volatile\("cp\.async\.wait_group \d+;\\n" ::: "memory"\);'), ';'),
    (re.compile(r'asm volatile\("st\.release\.sys\.global\.s32 \[%0\], %1;" ::"l"\((.*?)\), "r"\((.*?)\) : "memory"\);'), r'*(\1) = (\2);'),
    (re.compile(r'asm volatile\("ld\.acquire\.sys\.global\.s32 %0, \[%1\];" : "=r"\((\w+)\) : "l"\((.*?)\) : "memory"\);'), r'\1 = *(\2);'),
]


def drop_device_only(text):
    """`#ifndef MPMB_SIMT_HOST ... #else` regions hold device-only inline PTX (mbarrier / TMA bulk copies) whose emulator
    twins follow the #else: the device half is cut out before the rewrite rules and the leftover-asm check run."""
    out, skip = [], False
    for line in text.split("\n"):
        st = line.strip()
        if st == "#ifndef MPMB_SIMT_HOST":
            skip = True
            out.append("#if 1  // MPMB_SIMT_HOST: device half removed by build_simt.py")
            continue
        if skip:
            if st == "#else":
                skip = False
            out.append("")      # keep line numbers
            continue
        out.append(line)
    return "\n".join(out)


def transform(text):
    text = drop_device_only(text)
    for rx, rep in RULES:
        text = rx.sub(rep, text)
    left = [l for l in text.splitlines() if "<<<" in l or re.search(r"\basm\b", l)]
    left = [l for l in left if not l.strip().startswith("//")]
    if left:
        raise RuntimeError("unrewritten launch / asm sites:\n" + "\n".join(left[:10]))
    return text


def build(defines=(), force=False, asan=None):
    """asan (default: env MPMB_SIMT_ASAN=1): AddressSanitizer build — device memory is malloc'd host memory and
    shared memory is static storage, so out-of-bounds global / shared accesses of the kernels are reported; run with
    LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 (a memory checker without a GPU)."""
    if asan is None:
        asan = os.environ.get("MPMB_SIMT_ASAN", "") == "1"
    ubsan = os.environ.get("MPMB_SIMT_UBSAN", "") == "1"   # UndefinedBehaviorSanitizer (LD_PRELOAD libubsan.so)
    deps = [SRC, MATH, MATH2, os.path.join(HERE, "simt.h"), os.path.join(HERE, "simt.cpp"), os.path.join(HERE, "stub", "cub", "simt_cub.h"), __file__]
    tag = "_".join([d.lower().replace("mpmb_exp_", "") for d in defines] + (["asan"] if asan else []) + (["ubsan"] if ubsan else []))
    lib = LIB if not tag else LIB.replace(".so", "_" + tag + ".so")
    if not force and os.path.exists(lib) and all(os.path.getmtime(d) <= os.path.getmtime(lib) for d in deps):
        return lib
    os.makedirs(OUT_DIR, exist_ok=True)
    gen = os.path.join(OUT_DIR, "mpmb_engine_simt" + ("_" + tag if tag else "") + ".cpp")
    with open(gen, "w") as f:
        f.write('#line 1 "%s"\n' % SRC)
        f.write(transform(open(SRC).read()))
    cmd = ["/usr/bin/g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-march=x86-64-v3", "-mfma", "-w",
           "-I" + os.path.join(HERE, "stub"), "-I" + os.path.dirname(SRC), "-I" + os.path.join(ROOT, "include")] + ["-D" + d for d in defines] + (
           ["-fsanitize=address", "-fno-omit-frame-pointer"] if asan else []) + (
           ["-fsanitize=undefined", "-fno-sanitize-recover=undefined"] if ubsan else []) + [
           gen, os.path.join(HERE, "simt.cpp"), "-o", lib]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        raise RuntimeError("g++ failed building " + os.path.basename(lib))
    return lib


if __name__ == "__main__":
    defs = [sys.argv[i + 1] for i, a in enumerate(sys.argv) if a == "--define" and i + 1 < len(sys.argv)]
    print(build(defs, force=True))
