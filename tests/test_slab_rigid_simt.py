"""The rigid-coupled z-slab suite (tests/test_gpu_slab_rigid.py) on the SIMT emulator build of the engine (see
tests/test_simt_emulated.py), so that the CPU suite covers the slab rigid transfers, both impulse transports, the colour state in
the migration and re-cut records and the chained-oracle runs.  The two-GPU spawn tests need real devices and report as skipped.
About 100 s."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_slab_rigid_suite_passes_on_the_simt_emulator():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_slab_rigid.py"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "13 passed, 2 skipped" in tail and "failed" not in tail, tail
