"""The 2-D drop-in (tests/test_gpu_dropin_2d.py) on the SIMT-emulator build of the engine (tests/simt): the byte round trips,
the bit-identity with the field-wise upload, the refusals, and the reference's own MPM<2> object stepping every material and a
mixed pool through mpmb_upload_aos / mpmb_download_aos on a 2-D handle."""
import os
import subprocess
import sys

import pytest

from oracle import pyoracle2d_aos as A
from taichi_mpm_b200 import scenes
from tests import test_gpu_dropin_2d as G
from tests.test_gpu_mpm2d import KINDS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not A.ref_available(), reason="reference build (oracle/_ref) not available")


@needs_ref
def test_aos_calls_on_the_emulator():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_dropin_2d.py",
                        "-k", "round_trip or write_only or bit_identical or refusals or inplace_layout"], cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "12 passed" in tail and "failed" not in tail and "skipped" not in tail, tail


@needs_ref
@pytest.mark.parametrize("name,kind", KINDS, ids=[k[0] for k in KINDS])
def test_reference_solver_steps_through_the_c_abi_on_the_emulator(name, kind, tmp_path):
    from tests.simt import build_simt
    G.run_dropin2d(build_simt.build(), kind, tmp_path)


@needs_ref
def test_reference_solver_steps_a_mixed_pool_through_the_c_abi_on_the_emulator(tmp_path):
    from tests.simt import build_simt
    G.run_dropin2d(build_simt.build(), None, tmp_path, mixed=True)
