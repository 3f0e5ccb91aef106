"""The rigid-coupled parity tests (tests/test_gpu_rigid_parity.py) on the SIMT emulator build of the engine (see
tests/test_simt_emulated.py), in index order and in the reversed and shuffled CTA / thread orders, so that the CPU suite checks
k_p2g_rigid, k_g2p_rigid and the affine matrix the latter caches against the fp64 oracle.  About 30 s per order."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("order", ["0", "1", "2"], ids=["index", "reversed", "shuffled"])
def test_rigid_parity_suite_passes_on_the_simt_emulator(order):
    env = dict(os.environ, MPMB_SIMT="1", MPMB_SIMT_ORDER=order)
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_rigid_parity.py"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail
