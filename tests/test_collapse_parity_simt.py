"""The port-settled column of tests/test_gpu_zz_collapse_parity.py on the SIMT emulator build of the engine, in index and
shuffled CTA order: a 32^3 sand column settled onto its floor by 2 000 substeps of the fp32 port, uploaded, 4 substeps,
then three chained substeps and one substep on three windows against the fp64 oracle.  Each order runs in its own
process and settles the column again.  Run time: 50 s for both orders together on an idle 8-core x86 host, with the
emulator library already built; most of it is the port's 2 000 substeps."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("order", ["0", "2"], ids=["index", "shuffled"])
def test_collapse_parity_passes_on_the_simt_emulator(order):
    env = dict(os.environ, MPMB_SIMT="1", MPMB_SIMT_ORDER=order)
    env.pop("MPMB_LIB", None)
    env.pop("MPMB_NUM_SMS", None)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider", "-k", "port_settled",
                        "tests/test_gpu_zz_collapse_parity.py"], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    print("\n".join(l for l in r.stdout.splitlines() if "port-settled" in l or "window" in l))
    tail = "\n".join(r.stdout.strip().splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "1 passed" in tail and "failed" not in tail and "skipped" not in tail, tail
