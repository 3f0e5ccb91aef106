"""The tile-walk tests (tests/test_gpu_tile_walk.py) on the SIMT emulator build of the engine, in index order and in the
reversed and shuffled CTA orders: the chained oracle comparison with the launches sized for one SM, and the bitwise
comparison across grid sizes of the tile-scene, seed and AsyncMPM legs (the sequence and slab legs take minutes on the
emulator and run on the GPU only).  (The emulator performs bulk copies when their mbarrier is first waited on, so
a read racing an in-flight copy shows only on hardware.)"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("order", ["0", "1", "2"], ids=["index", "reversed", "shuffled"])
def test_tile_walk_suite_passes_on_the_simt_emulator(order):
    env = dict(os.environ, MPMB_SIMT="1", MPMB_SIMT_ORDER=order)
    env.pop("MPMB_LIB", None)
    env.pop("MPMB_NUM_SMS", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "sms1 or tile_scene or seed or async_device",
                        "tests/test_gpu_tile_walk.py"], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "4 passed" in tail and "failed" not in tail and "skipped" not in tail, tail
