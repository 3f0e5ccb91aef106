"""The edge-state tests of the engine's kernels (tests/test_gpu_material_edges.py: rotated, large, degenerate,
near-singular and inverted deformation gradients, every kind) on the SIMT emulator build of the engine (see
tests/test_simt_emulated.py), so that the CPU suite runs them too."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_material_edges_suite_passes_on_the_simt_emulator():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_material_edges.py"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    print("\n".join(l for l in r.stdout.splitlines() if " pg=" in l))
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail
