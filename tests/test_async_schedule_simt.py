"""AsyncMPM's block scheduler on the device (tests/test_gpu_async_schedule.py) on the SIMT emulator build of the engine (see
tests/test_simt_emulated.py), so that the CPU suite covers the mpmb_async_schedule / mpmb_async_advance_level kernels and
host code."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_async_schedule_suite_passes_on_the_simt_emulator():
    env = dict(os.environ, MPMB_SIMT="1")
    env.pop("MPMB_LIB", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_async_schedule.py"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail
