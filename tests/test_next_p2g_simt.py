"""The next-P2G parity tests (tests/test_gpu_next_p2g.py) on the SIMT emulator build of the engine (see
tests/test_simt_emulated.py), so that the CPU suite checks the affine matrix every writer caches for the next rasterize."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_next_p2g_suite_passes_on_the_simt_emulator():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_next_p2g.py"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail
