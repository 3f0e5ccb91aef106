"""The drop-in for pools that mix particle types (tests/test_gpu_dropin_mixed.py) on the SIMT-emulator build of the engine
(tests/simt): the byte round trip and the refusals through the C-ABI, the reference's own MPM<3> object stepping a pool of all
eight types through it, and its AsyncMPM<3> scheduler routed through one engine on two-type pools."""
import os
import subprocess
import sys

import pytest

from oracle import pyoracle_mixed as M
from taichi_mpm_b200 import scenes
from tests import test_gpu_dropin_mixed as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not M.ref_available(), reason="reference build (oracle/_ref) not available")


@needs_ref
def test_round_trip_and_refusals_on_the_emulator():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_dropin_mixed.py",
                        "-k", "round_trips or defaults or refused"], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "3 passed" in tail and "failed" not in tail and "skipped" not in tail, tail


@needs_ref
def test_reference_solver_steps_a_mixed_pool_through_the_c_abi_on_the_emulator(tmp_path):
    from tests.simt import build_simt
    G.run_dropin_mixed(build_simt.build(), tmp_path)


@needs_ref
@pytest.mark.parametrize("pair", [(scenes.MAT_SAND, scenes.MAT_ELASTIC), (scenes.MAT_SNOW, scenes.MAT_WATER)], ids=["sand_elastic", "snow_water"])
def test_reference_asyncmpm_routes_a_mixed_pool_on_the_emulator(pair):
    from tests.simt import build_simt
    G.run_async_mixed(build_simt.build(), pair)
