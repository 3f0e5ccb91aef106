"""Device-advanced rigid bodies (tests/test_gpu_rigid_motion.py) and examples/rigid_paddle.py on the SIMT emulator build of the
engine (see tests/test_simt_emulated.py), so that the CPU suite covers the advance / level-set collision kernels and their host
code.  The emulator has no CUDA graphs: graph replay itself is only exercised on a GPU."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _env():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    return env


def test_rigid_motion_suite_passes_on_the_simt_emulator():
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_rigid_motion.py"],
                       cwd=ROOT, env=_env(), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


_EXAMPLE = r"""
import os, sys, importlib.util
sys.path.insert(0, %r)
from tests.simt import build_simt
os.environ["MPMB_LIB"] = build_simt.build()
spec = importlib.util.spec_from_file_location("rigid_paddle", os.path.join(%r, "examples", "rigid_paddle.py"))
m = importlib.util.module_from_spec(spec)
spec.loader.exec_module(m)
mpm = m.main(2, 32)
print("paddle at x=%%.6f" %% mpm.rigids[0].position[0])
"""


def test_rigid_paddle_example_runs_on_the_emulator():
    r = subprocess.run([sys.executable, "-c", _EXAMPLE % (ROOT, ROOT)], cwd=ROOT, env=_env(), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    # two frames of 2e-3 at base_delta_t 1e-4 are 39 substeps on the float32 clock (as in the reference)
    assert "frame 2: t=0.0039" in r.stdout, r.stdout[-500:]
    # the paddle follows its script: x = 0.35 + 0.8 t at the end of the second frame
    assert "paddle at x=0.353120" in r.stdout, r.stdout[-500:]
