"""The z-slab re-cut (tests/test_gpu_slab_recut.py) on the SIMT emulator build of the engine (see tests/test_simt_emulated.py),
so that the CPU suite covers the layer histogram, the pack, the re-slicing apply and the substeps after it.  The two-GPU
spawn tests need a real device and report as skipped there."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_slab_recut_suite_passes_on_the_simt_emulator():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_slab_recut.py"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "10 passed" in tail and "failed" not in tail, tail
