"""k_p2g and k_g2p hand tiles out from per-launch device counters (claimed in slot order, zeroed by the ordering): which
CTA processes a tile must not change a bit of the result, and every path that launches the two kernels — whole
substeps, CUDA-graph replay of substep pairs (odd and even counts), the z-slab `_part` stages, and substeps after an
append — must find its counter at zero."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("id", "x", "v", "F", "b", "ps")


def run_sequence(no_graph=False):
    """A fast-moving sand block (dozens of movers per substep) through every launch path; the states after each leg."""
    from tests import common as T
    from tests.test_gpu_slab import _scene
    scene, st = _scene()
    e = T.make_engine(scene, st, no_graph=no_graph)
    out = []

    def snap():
        d = e.download()
        out.append({k: d[k] for k in KEYS})

    e.substep(1)          # odd: host launches
    e.substep(4)          # even: substep pairs (graph replay where graphs are on)
    e.substep(3)          # odd again: pairs + one
    snap()
    # one substep through the z-slab stages: part 1 (boundary layers; none on one engine) claims past every tile,
    # part 2 must still start from its own zeroed counter
    e.sort_particles_and_populate_grid()
    e.rasterize_part(1)
    e.rasterize_part(2)
    e.resample_part(2)
    e.resample_part(1)
    snap()
    rng = np.random.default_rng(11)
    x = (np.array([0.45, 0.45, 0.9]) + 0.1 * rng.random((300, 3))).astype(np.float32)
    e.append(x, np.zeros_like(x), np.full(300, st["mass"][0], np.float32), np.full(300, st["vol"][0], np.float32), group=np.zeros(300, np.int32))
    e.substep(2)
    snap()
    e.close()
    return out


def run_reference_sequence():
    """The same substeps with the `_part` substep replaced by a whole one: the states must be the same bits."""
    from tests import common as T
    from tests.test_gpu_slab import _scene
    scene, st = _scene()
    e = T.make_engine(scene, st, no_graph=True)
    out = []
    for n in (8, 1):
        e.substep(n)
        d = e.download()
        out.append({k: d[k] for k in KEYS})
    rng = np.random.default_rng(11)
    x = (np.array([0.45, 0.45, 0.9]) + 0.1 * rng.random((300, 3))).astype(np.float32)
    e.append(x, np.zeros_like(x), np.full(300, st["mass"][0], np.float32), np.full(300, st["vol"][0], np.float32), group=np.zeros(300, np.int32))
    e.substep(2)
    d = e.download()
    out.append({k: d[k] for k in KEYS})
    e.close()
    return out


def assert_same(a, b, what):
    assert len(a) == len(b)
    for i, (sa, sb) in enumerate(zip(a, b)):
        for k in KEYS:
            assert sa[k].shape == sb[k].shape and np.array_equal(sa[k], sb[k]), "%s: leg %d, %s" % (what, i, k)


@pytest.mark.gpu
def test_claimed_tiles_give_the_same_bits_with_graphs_parts_and_appends():
    graph = run_sequence(no_graph=False)
    host = run_sequence(no_graph=True)
    assert_same(graph, host, "graph replay vs host launches")
    assert_same(host, run_reference_sequence(), "_part stages vs whole substep")
    assert len(graph[-1]["id"]) > len(graph[0]["id"])  # the append landed


_ORDER_SCRIPT = r"""
import os, sys, pickle
sys.path.insert(0, %r)
from tests.simt import build_simt
os.environ["MPMB_LIB"] = build_simt.build()
from tests import test_tile_claims as M
pickle.dump((M.run_sequence(), M.run_reference_sequence()), open(sys.argv[1], "wb"))
"""


def test_claimed_tiles_do_not_depend_on_cta_order_on_the_emulator(tmp_path):
    # the emulator runs CTAs in index order, reversed, or shuffled per launch (MPMB_SIMT_ORDER), so each order hands the
    # tiles to different CTAs; every leg of the sequence must come out the same bits, and equal to the whole-substep path
    import pickle
    runs = []
    for order in ("0", "1", "2"):
        out = str(tmp_path / ("order%s.pkl" % order))
        env = dict(os.environ, MPMB_SIMT="1", MPMB_SIMT_ORDER=order)
        env.pop("MPMB_LIB", None)
        r = subprocess.run([sys.executable, "-c", _ORDER_SCRIPT % ROOT, out], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout[-2000:]
        with open(out, "rb") as f:
            runs.append(pickle.load(f))
    for seq, ref in runs:
        assert_same(seq, ref, "_part stages vs whole substep")
    for order, (seq, _) in zip("12", runs[1:]):
        assert_same(runs[0][0], seq, "CTA order 0 vs %s" % order)
    assert len(runs[0][0][-1]["id"]) > len(runs[0][0][0]["id"])
