"""The 2-D engine's GPU suite (tests/test_gpu_mpm2d.py) on the SIMT emulator build of the engine (see
tests/test_simt_emulated.py), so that the CPU suite covers the 2-D kernels and their host code; and one multi-tile scene
in the reversed and shuffled CTA and thread orders (MPMB_SIMT_ORDER), which must reproduce the index-order run bit for
bit (the 2-D substep has no atomics on its results)."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _env(order):
    env = dict(os.environ, MPMB_SIMT="1", MPMB_SIMT_ORDER=order)
    env.pop("MPMB_LIB", None)
    return env


def test_mpm2d_suite_passes_on_the_simt_emulator():
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_mpm2d.py"],
                       cwd=ROOT, env=_env("0"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


def test_mpm2d_bench_cases_pass_on_the_simt_emulator():
    # tests/test_gpu_zz_mpm2d_bench.py's cases the emulator runs (about 90 s on 8 host threads): the 64^2 collapse after
    # 0.05 s and every large grid; the full-size states and the longer collapses carry needs_cuda and are deselected here,
    # so that "skipped" still means a selected case did not run
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_zz_mpm2d_bench.py",
                        "-k", "64-0.05s or test_large_grids"], cwd=ROOT, env=_env("0"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "8 passed" in tail and "failed" not in tail and "skipped" not in tail, tail


_SCRIPT = r"""
import os, sys
import numpy as np
sys.path.insert(0, %r)
from tests.simt import build_simt
os.environ["MPMB_LIB"] = build_simt.build()
from taichi_mpm_b200 import scenes
from tests import test_gpu_mpm2d as M
res = (80, 72)
scene, st = M.scene2d(scenes.MAT_SAND, res=res, blocks=[((8, 8), (72, 64))], levelset=("shapes", [(1, 0, (40.0, 12.0, 0.0, 6.0))]),
                      seed=21, vel=0.0, dt=2e-4)
X = st["x"] * res[0]
st["v"] = (np.stack([np.sin(X[:, 1] * 0.3), np.cos(X[:, 0] * 0.2)], 1) * 0.9 / res[0] / 2e-4).astype(np.float32)
e = M.make_engine2d(scene, st)
e.substep(4)
np.savez(sys.argv[1], **e.download())
"""


@pytest.mark.parametrize("order", ["1", "2"], ids=["reversed", "shuffled"])
def test_multi_tile_scene_is_independent_of_the_scheduling_order(tmp_path, order):
    outs = []
    for o in ("0", order):
        out = str(tmp_path / ("order%s.npz" % o))
        r = subprocess.run([sys.executable, "-c", _SCRIPT % ROOT, out], cwd=ROOT, env=_env(o), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True)
        assert r.returncode == 0, r.stdout[-2000:]
        outs.append(np.load(out))
    assert len(outs[0]["id"]) > 4000
    for k in outs[0].files:
        assert np.array_equal(outs[0][k], outs[1][k]), k


_EXAMPLE = r"""
import os, sys, importlib.util, tempfile
sys.path.insert(0, %r)
from tests.simt import build_simt
os.environ["MPMB_LIB"] = build_simt.build()
spec = importlib.util.spec_from_file_location("sand_column_2d", os.path.join(%r, "examples", "sand_column_2d.py"))
m = importlib.util.module_from_spec(spec)
spec.loader.exec_module(m)
d = tempfile.mkdtemp()
m.main(4, 48, d)
print(sorted(os.listdir(d)))
"""


def test_2d_example_runs_on_the_emulator():
    # examples/sand_column_2d.py through the mirror: MPM2D(res=(48, 48)), a floor and a circle, an add between frames, frames
    r = subprocess.run([sys.executable, "-c", _EXAMPLE % (ROOT, ROOT)], cwd=ROOT, env=_env("0"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    assert "frame 4:" in r.stdout and "'0004.bgeo'" in r.stdout, r.stdout[-500:]
