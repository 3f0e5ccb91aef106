"""The resident-set edits (tests/test_gpu_resident_edit.py) and examples/water_source.py on the SIMT emulator build of the
engine (see tests/test_simt_emulated.py), so that the CPU suite covers the append / delete kernels and host code."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _env():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    return env


def test_resident_edit_suite_passes_on_the_simt_emulator():
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_resident_edit.py"],
                       cwd=ROOT, env=_env(), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


_EXAMPLE = r"""
import os, sys, importlib.util
sys.path.insert(0, %r)
from tests.simt import build_simt
os.environ["MPMB_LIB"] = build_simt.build()
spec = importlib.util.spec_from_file_location("water_source", os.path.join(%r, "examples", "water_source.py"))
m = importlib.util.module_from_spec(spec)
spec.loader.exec_module(m)
m.main(3)
"""


def test_water_source_example_runs_on_the_emulator():
    r = subprocess.run([sys.executable, "-c", _EXAMPLE % (ROOT, ROOT)], cwd=ROOT, env=_env(), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    assert "frame 3: 768 particles, ids 0..767, earlier ids unchanged" in r.stdout, r.stdout[-500:]
